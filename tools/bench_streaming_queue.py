"""Serving throughput and latency of the streaming-0.5B request queue (`vibevoice_b200.serving.StreamingRequestQueue`) against serial
solo `generate()` calls of the same requests.

Workload: the streaming-0.5B shapes (24 layers split 4 / 20, H 896, 14 / 2 heads of 64) with synthetic weights; every request starts from
a cached-prompt preset (random K/V in the reference's `all_prefilled_outputs` format, --prompt-lm / --prompt-tts positions) and has 20..200
text tokens; its max_new_tokens covers its text windows, their speech windows and 0..3 more speech windows.  The EOS classifier is biased
off, so every request ends at its own limit and both paths make the same audio.  5 diffusion steps and CFG 1.5 (the streaming CLI's
defaults).  All requests are submitted at t = 0 (the queue) or called one after another from t = 0 (serial).

Reported per path: aggregate audio-s/s; first-audio latency from submit (p50 / p90); each request's real-time margin = min over its later
chunks of (audio delivered after its first chunk) / (wall time since its first chunk), worst and p10 over requests (>= 1: playback that
starts at the first chunk never stalls); and for the queue the per-tick time by tick mix (text only / speech only / mixed), from CUDA
events on the engine stream.  The card's name, power limit and max SM clock are read in the same run.

    python tools/bench_streaming_queue.py [--requests 16] [--slots 1,2,4] [--prompt-lm 256] [--prompt-tts 512] [--warmup 2]
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SR, HOP = 24000, 3200
FRAME_S = HOP / SR


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [v.strip() for v in r.stdout.splitlines()[0].split(",")]))
    except Exception as e:          # the measurement still stands; the reader sees the machine is unknown
        return {"error": str(e)}


def build(slots, dev):
    from vibevoice_b200 import streaming as S
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.synth import iter_synth_state_dict_fast
    cfg = preset_config("streaming-0.5b")
    H = cfg.decoder_config.hidden_size
    g = torch.Generator(device=dev).manual_seed(7)

    def items():
        for name, t in iter_synth_state_dict_fast(cfg, 1234, device=dev, parts=("lm", "head", "acoustic_decoder", "connectors")):
            if not name.startswith("model.semantic"):
                yield name, t
        yield "model.tts_input_types.weight", torch.randn(2, H, device=dev, generator=g) * 0.05
        yield "tts_eos_classifier.fc1.weight", torch.randn(H, H, device=dev, generator=g) * 0.05
        yield "tts_eos_classifier.fc1.bias", torch.zeros(H, device=dev)
        yield "tts_eos_classifier.fc2.weight", torch.randn(1, H, device=dev, generator=g) * 0.05
        yield "tts_eos_classifier.fc2.bias", torch.full((1,), -8.0, device=dev)       # off: every request ends at its limit
    m = S.VibeVoiceStreamingForConditionalGenerationInference(cfg, tts_backbone_num_hidden_layers=20, max_slots=slots)
    m.load_state_dict(items())
    m.set_ddpm_inference_steps(5)
    return m


def preset(cfg, lm_len, tts_len, dev):
    dc = cfg.decoder_config
    H, low = dc.hidden_size, dc.num_hidden_layers - 20
    g = torch.Generator(device=dev).manual_seed(11)

    def cache(n, L):
        return tuple((torch.randn(1, dc.num_key_value_heads, L, dc.head_dim, device=dev, generator=g).to(torch.bfloat16) * 0.5,
                      torch.randn(1, dc.num_key_value_heads, L, dc.head_dim, device=dev, generator=g).to(torch.bfloat16) * 0.5) for _ in range(n))
    out = lambda n, L: SimpleNamespace(past_key_values=cache(n, L), last_hidden_state=torch.randn(1, L, H, device=dev, generator=g) * 0.1)
    return {"lm": out(low, lm_len), "tts_lm": out(20, tts_len), "neg_lm": out(low, 1), "neg_tts_lm": out(20, 1)}


def requests(n, seed, tts_len):
    rnd = random.Random(seed)
    reqs = []
    for i in range(n):
        n_text = rnd.randint(20, 200)
        windows = -(-n_text // 5)
        reqs.append(dict(text=torch.randint(0, 150000, (n_text,)), max_new_tokens=n_text + 6 * (windows + rnd.randint(0, 3)),
                         seed=rnd.randint(0, 10 ** 6), tts_ids=torch.zeros(1, tts_len, dtype=torch.long)))
    return reqs


class Clocked:
    """AudioStreamer(1) that keeps the wall time of every chunk."""

    def __init__(self):
        from vibevoice_b200.streamer import AudioStreamer
        self.st, self.t = AudioStreamer(1), []

    @property
    def batch_size(self):
        return 1

    def put(self, a, idx):
        self.t.append(time.perf_counter())
        self.st.put(a, idx)

    def end(self, idx=None):
        self.st.end(idx)


def stats(t0, clocks, audio_s, wall):
    first = [(c.t[0] - t0) * 1e3 for c in clocks if c.t]
    margins = []
    for c in clocks:
        r = [k * FRAME_S / (t - c.t[0]) for k, t in enumerate(c.t) if k > 0]
        if r:
            margins.append(min(r))
    return {"audio_s": round(audio_s, 2), "wall_s": round(wall, 3), "audio_s_per_s": round(audio_s / wall, 2),
            "first_audio_ms_p50": round(float(np.percentile(first, 50)), 2), "first_audio_ms_p90": round(float(np.percentile(first, 90)), 2),
            "realtime_margin_worst": round(min(margins), 3), "realtime_margin_p10": round(float(np.percentile(margins, 10)), 3)}


def kw(r, pre):
    return dict(input_ids=r["tts_ids"], tts_lm_input_ids=r["tts_ids"], tts_text_ids=r["text"][None], neg_text_input_id=151655,
                all_prefilled_outputs=pre, max_new_tokens=r["max_new_tokens"])


def serial(m, reqs, pre, max_total_tokens):
    m.engine.kv_init(max_total_tokens)                  # generate() sizes the pool for its first request only
    clocks, audio = [], 0.0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for r in reqs:
        c = Clocked()
        torch.manual_seed(r["seed"])
        out = m.generate(cfg_scale=1.5, audio_streamer=c, **kw(r, pre))
        audio += out.speech_outputs[0].shape[-1] / SR
        clocks.append(c)
    torch.cuda.synchronize()
    return stats(t0, clocks, audio, time.perf_counter() - t0)


def queued(m, reqs, pre, max_total_tokens):
    from vibevoice_b200 import serving
    eng = m.engine
    q = serving.StreamingRequestQueue(m, max_total_tokens=max_total_tokens)
    clocks, ticks = [], []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for r in reqs:
        c = Clocked()
        q.submit(cfg_scale=1.5, steps=5, seed=r["seed"], audio_streamer=c, **kw(r, pre))
        clocks.append(c)
    audio = 0.0
    while q._waiting or any(s is not None for s in q._slots):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(eng.stream)
        done = q.step()
        e1.record(eng.stream)
        ticks.append((q.last_tick, e0, e1))
        for _, out in done:
            audio += out.speech_outputs[0].shape[-1] / SR
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    res = stats(t0, clocks, audio, wall)
    mix = {}
    for (n_text, n_speech), e0, e1 in ticks:
        kind = "idle" if not n_text and not n_speech else "text_only" if not n_speech else "speech_only" if not n_text else "mixed"
        mix.setdefault(kind, []).append(e0.elapsed_time(e1))
    res["tick_ms_median"] = {k: round(statistics.median(v), 3) for k, v in mix.items()}
    res["ticks"] = {k: len(v) for k, v in mix.items()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--slots", default="1,2,4")
    ap.add_argument("--prompt-lm", type=int, default=256)
    ap.add_argument("--prompt-tts", type=int, default=512)
    ap.add_argument("--warmup", type=int, default=2, help="requests served before each timed pass")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: there is nothing to measure without one")
    dev = torch.device("cuda", 0)
    reqs = requests(args.requests, args.seed, args.prompt_tts)
    warm = requests(args.warmup, args.seed + 1, args.prompt_tts)
    line = {"bench": "streaming_queue", "gpu": gpu_info(), "requests": args.requests, "steps": 5, "cfg_scale": 1.5,
            "prompt_lm": args.prompt_lm, "prompt_tts": args.prompt_tts, "text_tokens": [int(r["text"].numel()) for r in reqs]}
    per_seq = max(args.prompt_lm, args.prompt_tts) + max(r["max_new_tokens"] for r in reqs + warm) + 130     # tokens, with page slack
    for slots in [int(s) for s in args.slots.split(",")]:
        m = build(slots, dev)
        pre = preset(m.config, args.prompt_lm, args.prompt_tts, dev)
        try:
            if slots == 1:
                serial(m, warm, pre, 3 * per_seq)
                line["serial"] = serial(m, reqs, pre, 3 * per_seq)
                print(json.dumps({"serial": line["serial"]}), flush=True)
            queued(m, warm, pre, 3 * slots * per_seq)
            line["queue_slots_%d" % slots] = queued(m, reqs, pre, 3 * slots * per_seq)
            print(json.dumps({"queue_slots_%d" % slots: line["queue_slots_%d" % slots]}), flush=True)
        finally:
            m.engine.close()
            del m
            torch.cuda.empty_cache()
    line["gpu_after"] = gpu_info()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
