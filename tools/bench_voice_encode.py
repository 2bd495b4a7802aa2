"""Voice-prompt encoder (a-9): `vv_voice_encode` against the PyTorch fp32 formulation it replaced.

The PyTorch side is `oracle.vv_oracle.voice_prompt_embeds` on CUDA tensors with fp32 weights and TF32 off (cuDNN convolutions, cuBLAS
linears), which is what the former PyTorch voice-prompt path computed.  Both sides get the same explicit noise.  The `-l2` presets have
the shipped acoustic encoder and connector shapes (H = 1536 / 3584); only the LM depth, which this benchmark does not touch, is cut.

Prints one JSON line per (preset, voices, seconds): median ms of each path over the repeats (CUDA events), TFLOP/s from the FLOP count of
the encoder + connector computed from shapes below, and the rel-L2 between the two outputs.  The card name and its power limit are read in
the same run.

    python tools/bench_voice_encode.py [--presets 1.5b-l2 7b-l2] [--voices 1 4] [--seconds 10 30] [--repeats 5] [--warmup 2]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import vv_oracle as O  # noqa: E402
from vibevoice_b200.configuration import preset_config  # noqa: E402
from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference  # noqa: E402
from vibevoice_b200.synth import SynthTokenizer, synth_state_dict  # noqa: E402

ENC = "model.acoustic_tokenizer.encoder"


def encoder_flops(cfg, n: int, T: int) -> int:
    """Multiply-adds x 2 of the non-streaming encoder + acoustic connector for n voices of T samples."""
    tc, H = cfg.acoustic_tokenizer_config, cfg.decoder_config.hidden_size
    nf, depths, ratios = tc.encoder_n_filters, tc.encoder_depth_list, list(reversed(tc.encoder_ratios))
    f, t, cin = 0, T, 1
    for i, d in enumerate(depths):
        c = nf << i
        k, s = (7, 1) if i == 0 else (2 * ratios[i - 1], ratios[i - 1])
        t = -(-t // s)
        f += 2 * t * c * k * cin                      # stem / downsample conv
        f += d * (2 * t * c * 7 + 2 * 2 * t * c * 4 * c)   # depthwise mixer + FFN of every Block1D
        cin = c
    f += 2 * t * tc.vae_dim * 7 * cin                 # head conv (t = frames)
    f += 2 * t * (tc.vae_dim * H + H * H)             # connector fc1, fc2
    return n * f


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def timed(fn, warmup, repeats):
    for _ in range(warmup):
        out = fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--presets", nargs="+", default=["1.5b-l2", "7b-l2"])
    ap.add_argument("--voices", nargs="+", type=int, default=[1, 4])
    ap.add_argument("--seconds", nargs="+", type=float, default=[10, 30])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_voice_encode needs a CUDA device")
    name, power = card()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    for preset in args.presets:
        cfg = preset_config(preset)
        tok = SynthTokenizer(cfg.decoder_config.vocab_size)
        sd = synth_state_dict(cfg, 1234, torch.bfloat16)
        m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=1)
        m.load_state_dict(sd, tok)
        eng = m.engine
        w = {k: v.to("cuda", torch.float32) for k, v in sd.items() if k.startswith(("model.acoustic_", "model.speech_"))}
        del sd
        for n in args.voices:
            for sec in args.seconds:
                T = int(sec * 24000)
                F = eng.voice_frames(T)
                g = torch.Generator().manual_seed(n * 1000 + T)
                wavs = (torch.randn(n, T, generator=g) * 0.05).cuda()
                std_n, eps = torch.randn(n, generator=g).cuda(), torch.randn(n, F, 64, generator=g).cuda()
                sigma = std_n * (cfg.acoustic_tokenizer_config.fix_std / 0.8)
                masks = torch.ones(n, F, dtype=torch.bool, device="cuda")
                with torch.no_grad():
                    ms_native, got = timed(lambda: eng.voice_encode(wavs, sigma, eps), args.warmup, args.repeats)
                    ms_torch, want = timed(lambda: O.voice_prompt_embeds(w, cfg, wavs, masks, noise=(std_n, eps)), args.warmup, args.repeats)
                flops = encoder_flops(cfg, n, T)
                print(json.dumps(dict(preset=preset, voices=n, seconds=sec, frames=F, gflop=round(flops / 1e9, 1),
                                      native_ms=round(ms_native, 3), torch_fp32_ms=round(ms_torch, 3),
                                      native_tflops=round(flops / ms_native / 1e9, 2), torch_tflops=round(flops / ms_torch / 1e9, 2),
                                      speedup=round(ms_torch / ms_native, 2), rel_l2=float((got.reshape(-1, got.shape[-1]) - want).norm() / want.norm()),
                                      gpu=name, power_limit_and_max_sm_clock=power)), flush=True)
                del got, want
                torch.cuda.empty_cache()
        eng.close()


if __name__ == "__main__":
    main()
