"""Throughput of the request queue (`vibevoice_b200.serving.RequestQueue`) against static `generate()` batches of B over the same requests.

A static batch runs until its longest row ends, so its useful share of the work is mean length / max length; the queue refills a finished
row at once.  The request set spreads its lengths (frames of speech per request) over a wide range; each request is scripted to exactly
its length on both paths (diffusion tokens, then EOS: `ForcedTokenScript` for `generate()`, the same tokens put in place of the decoded ones
for the queue), so both produce the same audio seconds.  Synthetic VibeVoice-1.5B weights, native prompt prefill, every request prefilled
from its own prompt.  Times are CUDA events on the engine stream around a whole pass; each figure is the median of --runs passes after one
warm-up pass.  A second queue pass mixes step counts (5 / 10 / 20) to measure what the per-row sampler's N_max steps per frame cost.

    python tools/bench_queue.py [--preset 1.5b] [--batch 4] [--requests 12] [--prompt 512] [--runs 3]

Prints one JSON line: audio-s/s of the queue and of the static batches, their ratio, the ideal ratio sum(max of each static batch) /
sum(lengths) * B ... and the GPU's name, power limit and clocks.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SR, HOP = 24000, 3200


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [v.strip() for v in r.stdout.splitlines()[0].split(",")]))
    except Exception as e:          # the measurement still stands; the reader sees the machine is unknown
        return {"error": str(e)}


def timed(eng, fn):
    """fn() between two CUDA events on the engine stream; returns (ms, result)."""
    torch.cuda.synchronize(eng.device)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(eng.stream)
    out = fn()
    b.record(eng.stream)
    b.synchronize()
    return a.elapsed_time(b), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preset", default="1.5b")
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--requests", type=int, default=12)
    ap.add_argument("--prompt", type=int, default=512)
    ap.add_argument("--frames", default="8,96,16,64,24,128,12,48,32,80,20,40", help="speech frames per request (cycled)")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_queue.py measures the GPU: no CUDA device")
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.modeling import ForcedTokenScript, VibeVoiceForConditionalGenerationInference
    from vibevoice_b200.serving import RequestQueue
    from vibevoice_b200.synth import SynthTokenizer, iter_synth_state_dict_fast

    dev = torch.device("cuda", 0)
    cfg = preset_config(args.preset)
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    B = args.batch
    model = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=B, prefill_impl="native")
    parts = ("lm", "head", "acoustic_decoder", "semantic", "connectors", "lm_head")
    model.load_state_dict(iter_synth_state_dict_fast(cfg, 1234, device=dev, parts=parts), tok)
    eng = model.engine
    d, eos = tok.speech_diffusion_id, tok.eos_token_id
    frames_cycle = [int(x) for x in args.frames.split(",")]
    frames = [frames_cycle[i % len(frames_cycle)] for i in range(args.requests)]
    g = torch.Generator().manual_seed(0)
    prompts = []
    for _ in range(args.requests):
        ids = torch.randint(0, min(cfg.decoder_config.vocab_size, 151643), (1, args.prompt), generator=g)
        ids[0, -1] = tok.speech_start_id
        prompts.append(ids)
    max_new = max(frames) + 2
    audio_s = sum(frames) * HOP / SR

    def static_pass():
        out_s = 0.0
        model.set_ddpm_inference_steps(args.steps)
        for b0 in range(0, args.requests, B):
            idx = list(range(b0, min(b0 + B, args.requests)))
            ids = torch.cat([prompts[i] for i in idx])
            scripts = [[d] * frames[i] + [eos] for i in idx]
            torch.manual_seed(b0)
            out = model.generate(input_ids=ids, tokenizer=tok, cfg_scale=1.3, max_new_tokens=max_new, max_length_times=1e9,
                                 logits_processor=[ForcedTokenScript(scripts)], show_progress_bar=False)
            out_s += sum(a.shape[-1] for a in out.speech_outputs if a is not None) / SR
        return out_s

    def queue_pass(steps_of):
        q = RequestQueue(model, max_total_tokens=B * (args.prompt + max_new + 8) + B * (max_new + 8))
        for i in range(args.requests):
            q.submit(dict(input_ids=prompts[i]), cfg_scale=1.3, steps=steps_of(i), max_new_tokens=max_new, max_length_times=1e9, seed=i)
        read = eng.read_tokens
        rid_frames = dict(enumerate(frames))

        def scripted():                      # each request: diffusion tokens for its frames, then EOS (what ForcedTokenScript does)
            t, lg = read()
            t = t.copy()
            for r, row in enumerate(q._rows):
                if row is not None and row.step >= 0:
                    t[r] = d if row.step < rid_frames[row.req.rid] else eos
            return t, lg
        eng.read_tokens = scripted
        try:
            outs = list(q.run())
        finally:
            del eng.read_tokens
        return sum(o.speech_outputs[0].shape[-1] for _, o in outs if o.speech_outputs[0] is not None) / SR

    res = {}
    for name, fn in [("static", static_pass), ("queue", lambda: queue_pass(lambda i: args.steps)),
                     ("queue_mixed_steps", lambda: queue_pass(lambda i: [5, 10, 20][i % 3]))]:
        fn()                                  # warm-up: programs built, graphs captured
        ms = []
        for _ in range(args.runs):
            t, out_s = timed(eng, fn)
            assert abs(out_s - audio_s) < 1e-6, (name, out_s, audio_s)
            ms.append(t)
        res[name] = dict(ms_median=statistics.median(ms), ms_all=[round(x, 1) for x in ms], audio_s_per_s=audio_s / (statistics.median(ms) / 1e3))
    # the useful share of a static batch is mean / max length: the queue can gain up to sum(max per batch * batch size) / sum(lengths)
    bound = sum(max(frames[b0:b0 + B]) * len(frames[b0:b0 + B]) for b0 in range(0, args.requests, B)) / sum(frames)
    print(json.dumps(dict(tool="bench_queue", preset=args.preset, batch=B, requests=args.requests, prompt_tokens=args.prompt, frames=frames,
                          steps=args.steps, audio_s=audio_s, static=res["static"], queue=res["queue"],
                          queue_mixed_steps_5_10_20=res["queue_mixed_steps"],
                          queue_over_static=res["queue"]["audio_s_per_s"] / res["static"]["audio_s_per_s"],
                          static_padding_bound=bound, gpu=gpu_info())))


if __name__ == "__main__":
    main()
