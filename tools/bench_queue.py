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

With `--voices K` every request also carries voice samples, as a service with a fixed voice library sees them: K speaker combinations of
1-4 speakers with 10-30 s synthetic wavs each, given to the requests in round robin, the voice section in front of the --prompt script
tokens.  Then only the queue is measured: each request's voices are encoded and prefilled at admission, or, with `--presets`, each
combination is a `VoicePreset` made once before the passes and the requests attach its shared KV pages (every pass starts a new queue,
so each pass prefills each preset once).  The JSON line adds the time the queue spent admitting (CUDA events around admission and
prompt prefill, per pass) and the KV pages the pool held after each frame (peak and mean).

    python tools/bench_queue.py --preset 1.5b --batch 8 --requests 48 --voices 6 [--presets]
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
    ap.add_argument("--voices", type=int, default=0, help="voice library size K (0: requests without voices)")
    ap.add_argument("--presets", action="store_true", help="with --voices: serve the library as voice presets")
    args = ap.parse_args()
    if args.presets and not args.voices:
        sys.exit("--presets needs --voices K")
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
    parts = ("lm", "head", "acoustic_decoder", "semantic", "connectors", "lm_head") + (("acoustic_encoder",) if args.voices else ())
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

    if args.voices:
        voice_queue(args, model, tok, eng, prompts, frames, audio_s, max_new, timed)
        return
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


def voice_library(k, cfg, tok, seed=0):
    """k voice prompt prefixes (system prompt ids + " Speaker s:" <speech_start> <speech_diffusion> x frames <speech_end> per speaker) in
    `VibeVoiceProcessor.voice_prefix`'s format: combination j has 1 + j % 4 speakers of 10-30 s of synthetic audio."""
    g = torch.Generator().manual_seed(seed)
    V = min(cfg.decoder_config.vocab_size, 151643)
    rnd = lambda n: torch.randint(0, V, (n,), generator=g).tolist()
    lib = []
    for j in range(k):
        secs = [10 + (7 * j + 11 * s) % 21 for s in range(1 + j % 4)]
        wavs = torch.zeros(len(secs), max(secs) * SR)
        ids, sim = rnd(30), [False] * 30
        for s, sec in enumerate(secs):
            wavs[s, :sec * SR] = torch.randn(sec * SR, generator=g) * 0.1
            n = -(-sec * SR // HOP)                  # ceil, as the processor counts a voice's frames
            ids += rnd(4) + [tok.speech_start_id] + [tok.speech_diffusion_id] * n + [tok.speech_end_id] + rnd(1)
            sim += [False] * 5 + [True] * n + [False] * 2
        masks = torch.zeros(len(secs), -(-max(secs) * SR // HOP), dtype=torch.bool)
        for s, sec in enumerate(secs):
            masks[s, :-(-sec * SR // HOP)] = True
        lib.append(dict(input_ids=torch.tensor([ids]), speech_input_mask=torch.tensor([sim]), speech_tensors=wavs, speech_masks=masks))
    return lib


def voice_queue(args, model, tok, eng, prompts, frames, audio_s, max_new, timed):
    from vibevoice_b200.serving import RequestQueue
    lib = voice_library(args.voices, model.config, tok)
    presets = [model.voice_preset(p, seed=j) for j, p in enumerate(lib)] if args.presets else None
    reqs = []
    for i, pr in enumerate(prompts):
        j = i % args.voices
        ids = torch.cat([lib[j]["input_ids"], pr], dim=1)
        sim = torch.cat([lib[j]["speech_input_mask"], torch.zeros_like(pr, dtype=torch.bool)], dim=1)
        reqs.append((dict(input_ids=ids, speech_input_mask=sim, speech_tensors=lib[j]["speech_tensors"], speech_masks=lib[j]["speech_masks"]),
                     None if presets is None else presets[j]))
    Lmax = max(r["input_ids"].shape[1] for r, _ in reqs)
    d, eos = tok.speech_diffusion_id, tok.eos_token_id
    B = args.batch
    stats = {}

    def queue_pass():
        q = RequestQueue(model, max_total_tokens=B * (Lmax + max_new + 8) + B * (max_new + 8))
        for i, (inp, p) in enumerate(reqs):
            q.submit(inp, cfg_scale=1.3, steps=args.steps, max_new_tokens=max_new, max_length_times=1e9, seed=i, voice_preset=p)
        read, admit, prefill, frame = eng.read_tokens, q._admit, q._prefill_progress, q._frame
        ev, pages = [], []

        def on_events(fn):                    # admission and prompt prefill between two CUDA events on the engine stream
            def run(*a):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(eng.stream)
                out = fn(*a)
                e1.record(eng.stream)
                ev.append((e0, e1))
                return out
            return run

        def scripted():
            t, lg = read()
            t = t.copy()
            for r, row in enumerate(q._rows):
                if row is not None and row.step >= 0:
                    t[r] = d if row.step < frames[row.req.rid] else eos
            return t, lg

        def framed():
            out = frame()
            pages.append(eng.kv_pages - eng.kv_pages_free())
            return out
        eng.read_tokens, q._admit, q._prefill_progress, q._frame = scripted, on_events(admit), on_events(prefill), framed
        try:
            outs = list(q.run())
        finally:
            del eng.read_tokens
        eng.sync()
        stats["admit_ms"] = sum(a.elapsed_time(b) for a, b in ev)
        stats["pages_peak"], stats["pages_mean"] = max(pages), sum(pages) / len(pages)
        return sum(o.speech_outputs[0].shape[-1] for _, o in outs if o.speech_outputs[0] is not None) / SR

    queue_pass()                              # warm-up: programs built, graphs captured
    ms, admit, peak, mean = [], [], [], []
    for _ in range(args.runs):
        t, out_s = timed(eng, queue_pass)
        assert abs(out_s - audio_s) < 1e-6, (out_s, audio_s)
        ms.append(t)
        admit.append(stats["admit_ms"])
        peak.append(stats["pages_peak"])
        mean.append(stats["pages_mean"])
    print(json.dumps(dict(tool="bench_queue", preset=args.preset, batch=B, requests=args.requests, prompt_tokens=args.prompt, frames=frames,
                          steps=args.steps, audio_s=audio_s, voices=args.voices, presets=bool(args.presets),
                          voice_prefix_tokens=[int(p["input_ids"].shape[1]) for p in lib],
                          queue=dict(ms_median=statistics.median(ms), ms_all=[round(x, 1) for x in ms],
                                     audio_s_per_s=audio_s / (statistics.median(ms) / 1e3)),
                          admit_ms_median=statistics.median(admit), admit_ms_all=[round(x, 1) for x in admit],
                          kv_pages_peak=max(peak), kv_pages_mean=statistics.median(mean), kv_pages_total=eng.kv_pages, gpu=gpu_info())))


if __name__ == "__main__":
    main()
