"""Prompt prefill: the native kernels (`vv_lm_prefill`, csrc/vv_prefill.cuh) against the PyTorch prefill (`TorchPrefill`: cuBLAS + SDPA in
bf16 on a second bf16 copy of the LM).

Full 28-layer 1.5B at L = 4 096 / 16 384 / 63 488 and 7B at L = 30 720, synthetic weights from the seed.  Both sides prefill the same
embeddings into the paged pool of the same engine.  Prints one JSON line per (model, L): median ms over the repeats (CUDA events, after
warm-up), tokens/s and TFLOP/s of each side (FLOPs of the linears + causal attention, from shapes below), the rel-L2 between the two last
hidden states, and device memory: resident after load (engine weights, plus the bf16 copy for TorchPrefill) and the peak during the
prefill.  With --profile, one more native run per model at its longest L is traced with torch.profiler and split into GEMM / attention /
other kernel time, each GEMM / attention share turned into TFLOP/s.  The card name, power limit and max SM clock are read in the same run.

    python tools/bench_prefill.py [--models 1.5b 7b] [--lens 4096 16384 63488] [--lens7b 30720] [--repeats 5] [--warmup 1] [--profile]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from vibevoice_b200.configuration import preset_config  # noqa: E402
from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference  # noqa: E402
from vibevoice_b200.prefill import TorchPrefill  # noqa: E402
from vibevoice_b200.synth import SynthTokenizer, iter_synth_state_dict_fast  # noqa: E402

PARTS = ("lm", "head", "acoustic_decoder", "semantic", "connectors", "lm_head")


def flops(dc, L: int):
    """(linear, attention) FLOPs of one prefill of L tokens: 2 per multiply-add; causal attention counts the L (L + 1) / 2 visible pairs
    for Q K^T and for P V."""
    H, I, nh, nkv, hd = dc.hidden_size, dc.intermediate_size, dc.num_attention_heads, dc.num_key_value_heads, dc.head_dim
    lin = 2 * L * (H * (nh + 2 * nkv) * hd + nh * hd * H + H * 2 * I + I * H)
    att = 2 * 2 * nh * hd * (L * (L + 1) // 2)
    return lin * dc.num_hidden_layers, att * dc.num_hidden_layers


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def used():
    free, total = torch.cuda.mem_get_info()
    return total - free


def timed(fn, warmup, repeats):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms), out


def rel_l2(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def run_model(name, lens, args, cname, power):
    cfg = preset_config(name)
    dc = cfg.decoder_config
    tok = SynthTokenizer(dc.vocab_size)
    torch.cuda.synchronize()
    base = used()
    m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=1, prefill_impl="native")
    m.load_state_dict(iter_synth_state_dict_fast(cfg, 1234, device="cuda", parts=PARTS), tok)
    eng = m.engine
    eng.kv_init(max(lens) + 256)
    torch.cuda.synchronize()
    res_native = used() - base
    # the bf16 LM copy a model loaded with torch_prefill=True keeps
    lm = {k: v for k, v in iter_synth_state_dict_fast(cfg, 1234, device="cuda", parts=("lm",))}
    tp = TorchPrefill(cfg, lm, eng.device)
    del lm
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    res_torch = used() - base
    g = torch.Generator(device="cuda").manual_seed(7)
    for L in lens:
        e = torch.randn(L, dc.hidden_size, generator=g, device="cuda") * 0.5
        lin, att = flops(dc, L)
        out = {}
        for impl in ("native", "torch"):
            def fn():
                eng.kv_set_len(0, 0)
                if impl == "native":
                    return eng.lm_prefill(0, e)
                with torch.cuda.stream(eng.stream):
                    h = tp.run(eng, 0, e)
                torch.cuda.current_stream().wait_stream(eng.stream)
                return h
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            a0 = torch.cuda.memory_allocated()
            ms, h = timed(fn, args.warmup, args.repeats)
            peak = torch.cuda.max_memory_allocated() - a0
            out[impl] = dict(ms=round(ms, 2), tok_s=round(L / ms * 1e3), tflops=round((lin + att) / ms / 1e9, 1),
                             resident_gb=round((res_native if impl == "native" else res_torch) / 2 ** 30, 2),
                             peak_gb=round(((res_native if impl == "native" else res_torch) + peak) / 2 ** 30, 2), hidden=h.float().cpu())
        rec = dict(model=name, L=L, gpu=cname, power_limit_max_sm_clock=power, linear_tflop=round(lin / 1e12, 2), attention_tflop=round(att / 1e12, 2),
                   hidden_rel_l2=rel_l2(out["native"].pop("hidden"), out["torch"].pop("hidden")), native=out["native"], torch_prefill=out["torch"],
                   speedup=round(out["torch"]["ms"] / out["native"]["ms"], 3))
        print(json.dumps(rec), flush=True)
    if args.profile:
        L = max(lens)
        e = torch.randn(L, dc.hidden_size, generator=g, device="cuda") * 0.5
        eng.kv_set_len(0, 0)
        eng.lm_prefill(0, e)
        torch.cuda.synchronize()
        from torch.profiler import ProfilerActivity, profile
        eng.kv_set_len(0, 0)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.lm_prefill(0, e)
            torch.cuda.synchronize()
        t = {"gemm": 0.0, "attention": 0.0, "other": 0.0}
        for ev in prof.key_averages():
            us = ev.self_device_time_total if hasattr(ev, "self_device_time_total") else ev.self_cuda_time_total
            k = "gemm" if "pf_gemm_kernel" in ev.key else "attention" if "pf_attn_kernel" in ev.key else "other"
            t[k] += us
        lin, att = flops(dc, L)
        print(json.dumps(dict(model=name, L=L, profile_ms={k: round(v / 1e3, 2) for k, v in t.items()},
                              gemm_tflops=round(lin / (t["gemm"] * 1e6), 1) if t["gemm"] else None,
                              attention_tflops=round(att / (t["attention"] * 1e6), 1) if t["attention"] else None, gpu=cname,
                              power_limit_max_sm_clock=power)), flush=True)
    del tp
    eng.close()
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=["1.5b", "7b"])
    ap.add_argument("--lens", nargs="+", type=int, default=[4096, 16384, 63488])
    ap.add_argument("--lens7b", nargs="+", type=int, default=[30720])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_prefill needs a CUDA device")
    cname, power = card()
    for name in args.models:
        run_model(name, args.lens7b if name == "7b" else args.lens, args, cname, power)


if __name__ == "__main__":
    main()
