"""What request priorities buy a mixed service: latency of short interactive requests behind a backlog of long ones, with and without
priorities (`RequestQueue.submit(priority=)`), and the throughput and per-preemption cost it takes.

Workload per model (synthetic weights, native prompt prefill, --batch rows): a backlog of --backlog priority-0 requests scripted to
256-512 speech frames each, and --interactive requests of 8-16 frames submitted from inside the `run()` loop after fixed frame counts
(deterministic arrivals).  Every request is scripted to its length (diffusion tokens, then EOS, put in place of the decoded tokens as
tools/bench_queue.py does), so both passes make the same audio.  In the "fifo" pass every request has priority 0 (today's
first-in-first-out queue); in the "priority" pass the interactive requests have priority 1 and preempt backlog rows.

The pool holds the worst case of B live rows and B parked ones by default (`--pool live+parked`), so parking never waits for pages.
`--pool live` sizes it for the B live rows alone: then a preempting request does not fit beside the rows it preempts unless their
pages move to host memory, and `--swap-gib X` adds a "priority_swap" pass with `RequestQueue(host_swap_bytes=X GiB)`.

Reported per model and pass: the interactive requests' latency from submit to result (p50 / p90, in frames and host ms; results leave
`run()` after a device synchronisation), total audio-s/s (CUDA events around the whole run), and in the priority pass the number of parks
and the cost of one park plus its resume in us (CUDA events on the engine stream around each call), with the GPU's name, power limit
and clocks read in the same run.  With swapping, also the number of swap-outs and the median cost of one swap-out and one swap-in
(`Engine.kv_swap_out` / `kv_swap_in`, CUDA events around each call, the pinned-buffer allocation included).

    python tools/bench_priority.py [--presets 1.5b,7b] [--batch 8] [--backlog 24] [--interactive 12] [--prompt 256]
                                   [--pool live+parked|live] [--swap-gib X]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_queue import SR, HOP, gpu_info, timed      # noqa: E402


def pct(xs, p):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(round(p / 100 * (len(xs) - 1))))]


def one_model(args, preset):
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    from vibevoice_b200.serving import RequestQueue
    from vibevoice_b200.synth import SynthTokenizer, iter_synth_state_dict_fast

    dev = torch.device("cuda", 0)
    cfg = preset_config(preset)
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    B = args.batch
    model = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=B, prefill_impl="native")
    parts = ("lm", "head", "acoustic_decoder", "semantic", "connectors", "lm_head")
    model.load_state_dict(iter_synth_state_dict_fast(cfg, 1234, device=dev, parts=parts), tok)
    eng = model.engine
    d, eos = tok.speech_diffusion_id, tok.eos_token_id
    g = torch.Generator().manual_seed(0)
    n_all = args.backlog + args.interactive
    prompts = []
    for _ in range(n_all):
        ids = torch.randint(0, min(cfg.decoder_config.vocab_size, 151643), (1, args.prompt), generator=g)
        ids[0, -1] = tok.speech_start_id
        prompts.append(ids)
    long = [int(x) for x in torch.randint(256, 513, (args.backlog,), generator=g)]
    short = [int(x) for x in torch.randint(8, 17, (args.interactive,), generator=g)]
    frames = long + short
    # arrivals spread over the backlog's span: after frame `at[i]` interactive request i is submitted
    span = sum(long) // B
    at = [args.first_arrival + i * (span - args.first_arrival) // (args.interactive + 1) for i in range(args.interactive)]
    max_new = max(frames) + 2

    def run_pass(prio, scale=1, swap_bytes=0):
        fr = [max(1, f // scale) for f in frames]
        pages = (args.prompt + max_new + 2 + 63) // 64 + (max_new + 2 + 63) // 64      # a request's worst case (RequestQueue.submit)
        held = B if args.pool == "live" else 2 * B                                       # B live rows (and up to B parked ones)
        q = RequestQueue(model, max_total_tokens=held * pages * 64, host_swap_bytes=swap_bytes)
        sub = lambda i, p: q.submit(dict(input_ids=prompts[i]), cfg_scale=1.3, steps=args.steps, max_new_tokens=max_new,
                                    max_length_times=1e9, seed=i, priority=p)
        rid_frames = {sub(i, 0): fr[i] for i in range(args.backlog)}
        read, frame, park, resume = eng.read_tokens, q._frame, q._park, q._resume
        n_frame, submitted, costs = [0], {}, []
        arrive = {}
        for i, f in enumerate(at):
            arrive.setdefault(max(1, f // scale), []).append(args.backlog + i)

        def scripted():
            t, lg = read()
            t = t.copy()
            for r, row in enumerate(q._rows):
                if row is not None and row.step >= 0:
                    t[r] = d if row.step < rid_frames[row.req.rid] else eos
            return t, lg

        def counted():
            done = frame()
            n_frame[0] += 1
            for i in arrive.get(n_frame[0], []):
                rid = sub(i, prio)
                rid_frames[rid] = fr[i]
                submitted[rid] = (n_frame[0], time.perf_counter())
            return done

        def ev_timed(fn, key):
            def call(*a):
                ms, _ = timed(eng, lambda: fn(*a))
                costs.append((key, ms))
            return call
        eng.read_tokens, q._frame = scripted, counted
        q._park, q._resume = ev_timed(park, "park"), ev_timed(resume, "resume")
        q._swap_out = ev_timed(q._swap_out, "swap_out")
        eng.kv_swap_in = ev_timed(eng.kv_swap_in, "swap_in")
        lat_f, lat_ms, audio = [], [], 0.0
        try:
            ms, outs = timed(eng, lambda: [(rid, out, n_frame[0], time.perf_counter()) for rid, out in q.run()])
        finally:
            del eng.read_tokens, eng.kv_swap_in
        for rid, out, nf, t in outs:
            audio += out.speech_outputs[0].shape[-1] / SR
            if rid in submitted:
                lat_f.append(nf - submitted[rid][0])
                lat_ms.append((t - submitted[rid][1]) * 1e3)
        want = sum(fr) * HOP / SR
        assert abs(audio - want) < 1e-6, (audio, want)
        parks = [c for k, c in costs if k == "park"]
        resumes = [c for k, c in costs if k == "resume"]
        res = dict(wall_ms=round(ms, 1), audio_s=round(audio, 2), audio_s_per_s=round(audio / (ms / 1e3), 3), frames_run=n_frame[0],
                   interactive_latency_frames=dict(p50=pct(lat_f, 50), p90=pct(lat_f, 90)),
                   interactive_latency_ms=dict(p50=round(pct(lat_ms, 50), 1), p90=round(pct(lat_ms, 90), 1)), parks=q.parks)
        if parks:
            res["park_us_median"] = round(statistics.median(parks) * 1e3, 1)
            res["resume_us_median"] = round(statistics.median(resumes) * 1e3, 1)
            res["park_plus_resume_us"] = round((statistics.median(parks) + statistics.median(resumes)) * 1e3, 1)
        if swap_bytes:
            res["swaps"] = q.swaps
            for k in ("swap_out", "swap_in"):
                c = [ms for key, ms in costs if key == k]
                if c:
                    res[k + "_us_median"] = round(statistics.median(c) * 1e3, 1)
        return res

    swap = int(args.swap_gib * (1 << 30))
    run_pass(1, scale=32, swap_bytes=swap)     # warm-up: programs built, graphs captured, a park and a resume (and a swap) taken
    out = dict(fifo=run_pass(0), priority=run_pass(1))
    if swap:
        out["priority_swap"] = run_pass(1, swap_bytes=swap)
    eng.close()
    del model
    torch.cuda.empty_cache()
    return dict(backlog_frames=long, interactive_frames=short, arrivals_after_frame=at, **out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--presets", default="1.5b,7b")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--backlog", type=int, default=24)
    ap.add_argument("--interactive", type=int, default=12)
    ap.add_argument("--prompt", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--first-arrival", type=int, default=50)
    ap.add_argument("--pool", default="live+parked", choices=["live+parked", "live"],
                    help="KV pool sized for B live rows and B parked ones, or for the live rows alone")
    ap.add_argument("--swap-gib", type=float, default=0.0, help="host memory for swapped KV pages; > 0 adds a priority_swap pass")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_priority.py measures the GPU: no CUDA device")
    res = dict(tool="bench_priority", batch=args.batch, backlog=args.backlog, interactive=args.interactive, prompt_tokens=args.prompt,
               steps=args.steps, gpu=gpu_info())
    if args.pool != "live+parked" or args.swap_gib:
        res.update(pool=args.pool, swap_gib=args.swap_gib)
    for p in args.presets.split(","):
        res[p] = one_model(args, p)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
