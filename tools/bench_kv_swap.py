"""What moving a parked request's KV pages to host memory costs: `vv_kv_swap_out` / `vv_kv_swap_in` time and rate per record size, at
the KV page shapes of VibeVoice-1.5B (28 layers, 2 KV heads of 128) and 7B (28 layers, 4 KV heads of 128), against one
`cudaMemcpyAsync` of a contiguous pinned buffer of the same size in each direction (the DMA ceiling on the same machine).

The swap kernel touches only the KV pool, so the model is a narrow one with exactly those pool shapes (synthetic weights; hidden width
128).  A record of N private pages is made by writing N * 64 positions of one sequence and parking it.  Each size is warmed up once,
then timed over --reps round trips with CUDA events on the engine stream around each call; the median is reported, with GB/s as the
record's bytes over that time.  After the last round trip the sequence's layer-0 K/V is read back and compared bit for bit.  The GPU's
name, power limit and clocks are read in the same run.

    python tools/bench_kv_swap.py [--pages 1,8,32,33,470] [--reps 10]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_queue import gpu_info, timed      # noqa: E402

SHAPES = {"1.5b": 2, "7b": 4}                # KV heads; both models have 28 layers and head_dim 128


def make_engine(kv_heads):
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    from vibevoice_b200.synth import SynthTokenizer, synth_state_dict
    cfg = preset_config("tiny")
    dc = cfg.decoder_config
    dc.num_hidden_layers, dc.num_key_value_heads, dc.num_attention_heads, dc.head_dim = 28, kv_heads, 2 * kv_heads, 128
    tok = SynthTokenizer(dc.vocab_size)
    parts = ("lm", "head", "acoustic_decoder", "semantic", "connectors", "lm_head")
    m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=1, prefill_impl="native")
    m.load_state_dict(synth_state_dict(cfg, 1234, torch.bfloat16, parts=parts), tok)
    return m.engine


def one_shape(args, name):
    eng = make_engine(SHAPES[name])
    dc = eng.config.decoder_config
    out = []
    try:
        top = max(args.pages)
        eng.kv_init(64 * (top + 8))
        g = torch.Generator(device=eng.device).manual_seed(0)
        for n in args.pages:
            L = 64 * n
            k = torch.randn(L, dc.num_key_value_heads, dc.head_dim, generator=g, device=eng.device).to(torch.bfloat16)
            v = torch.randn(L, dc.num_key_value_heads, dc.head_dim, generator=g, device=eng.device).to(torch.bfloat16)
            eng.kv_write(0, 0, 0, k, v)
            eng.kv_set_len(0, L)
            h = eng.kv_park(0)
            nbytes = eng.kv_swap_bytes(h)
            assert nbytes == n * eng.kv_page_bytes
            t_out, t_in = [], []
            for rep in range(args.reps + 1):
                ms, buf = timed(eng, lambda: eng.kv_swap_out(h))
                ms2, _ = timed(eng, lambda: eng.kv_swap_in(h, buf))
                if rep:                                   # rep 0 warms up
                    t_out.append(ms)
                    t_in.append(ms2)
                eng.sync()                                # the engine lets go of the buffer: the pinned cache takes it back
            eng.kv_unpark(h, 0)
            k2, v2 = eng.kv_read(0, 0, 0, L)
            assert torch.equal(k2, k) and torch.equal(v2, v), "swap round trip changed the K/V"
            eng.kv_set_len(0, 0)
            # the ceiling: one contiguous copy of the same size each way
            host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
            dev = torch.empty(nbytes, dtype=torch.uint8, device=eng.device)
            d2h, h2d = [], []
            for rep in range(args.reps + 1):
                with torch.cuda.stream(eng.stream):
                    a, _ = timed(eng, lambda: host.copy_(dev, non_blocking=True))
                    b, _ = timed(eng, lambda: dev.copy_(host, non_blocking=True))
                if rep:
                    d2h.append(a)
                    h2d.append(b)
            eng.sync()
            med = statistics.median
            gbs = lambda ms: round(nbytes / (ms * 1e6), 2)
            row = dict(model=name, pages=n, bytes=nbytes, swap_out_us=round(med(t_out) * 1e3, 1), swap_out_GBs=gbs(med(t_out)),
                       swap_in_us=round(med(t_in) * 1e3, 1), swap_in_GBs=gbs(med(t_in)), memcpy_d2h_us=round(med(d2h) * 1e3, 1),
                       memcpy_d2h_GBs=gbs(med(d2h)), memcpy_h2d_us=round(med(h2d) * 1e3, 1), memcpy_h2d_GBs=gbs(med(h2d)))
            print(json.dumps(row), flush=True)
            out.append(row)
    finally:
        eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1.5b,7b")
    ap.add_argument("--pages", default="1,8,32,33,470")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the rows as JSON here")
    args = ap.parse_args()
    args.pages = [int(x) for x in args.pages.split(",")]
    if not torch.cuda.is_available():
        raise SystemExit("bench_kv_swap.py measures on a CUDA device; there is none")
    info = gpu_info()
    print(json.dumps({"gpu": info}), flush=True)
    rows = []
    for name in args.shapes.split(","):
        rows += one_shape(args, name)
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(gpu=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
