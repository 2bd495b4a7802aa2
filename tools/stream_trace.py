"""Per-stage time breakdown inside the persistent weight-stream kernel (csrc/vv_stream.cuh) for one CTA:
    VV_STREAM_TRACE=<cta> python tools/stream_trace.py [--model 1.5b --steps 30 --batch 1 --prog samp]
Stamps (SM clock): worker thread: stage start, barrier passed, row statistics done, B operand staged, accumulators complete, epilogue
issued; MMA thread: saw b_ready, saw the last tile, committed; producer: issued the last tile of the stage."""
import argparse
import ctypes as C
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vibevoice_b200 import _native as N
from vibevoice_b200.configuration import preset_config
from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
from vibevoice_b200.synth import SynthTokenizer, iter_synth_state_dict_fast

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="1.5b")
ap.add_argument("--steps", type=int, default=30)
ap.add_argument("--batch", type=int, default=1)
ap.add_argument("--prog", default="samp")
ap.add_argument("--ctx", type=int, default=61440)
ap.add_argument("--mhz", type=float, default=1965.0)
a = ap.parse_args()
os.environ.setdefault("VV_STREAM_TRACE", "5")
cfg = preset_config(a.model)
tok = SynthTokenizer(cfg.decoder_config.vocab_size)
B = a.batch
m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=B)
m.load_state_dict(iter_synth_state_dict_fast(cfg, 1234, device="cuda", parts=("lm", "head", "acoustic_decoder", "semantic", "connectors", "lm_head")), tok)
eng = m.engine
eng.kv_init(B * 1024)
eng.set_diffusion_steps(a.steps)
with torch.cuda.stream(eng.stream):
    eng.active.fill_(1)
    eng.noise.normal_()
    eng.hidden.normal_()
if a.prog.startswith("lm"):
    ctx = a.ctx
    eng.kv_init(B * (ctx + 64) + B * 64)
    for r in range(B):
        N.check(eng.lib.vv_kv_reserve(eng.h, r, ctx + 16, eng.s))
        eng.kv_set_len(r, ctx)
        eng.kv_set_len(B + r, 0)
    eng.embed_tokens([tok.speech_start_id] * (2 * B), eng.embeds)
    for _ in range(5):
        eng.lm_decode()
        eng.kv_commit([1] * (2 * B))
elif a.prog.startswith("decf"):
    for _ in range(5):
        eng.codec_decode()
elif a.prog.startswith("encb"):
    for _ in range(5):
        eng.semantic_encode()
else:
    for _ in range(5):
        eng.diffusion_sample(1.3)
eng.sync()
MAXO = 4096
out = np.zeros((MAXO, 12), dtype=np.int64)
meta = np.zeros((MAXO, 4), dtype=np.int32)
n = eng.lib.vv_stream_trace_read(eng.h, out.ctypes.data_as(C.c_void_p), meta.ctypes.data_as(C.c_void_p), MAXO, a.prog.encode())
print("stages traced:", n)
us = lambda cyc: cyc / a.mhz
rows = {}
for i in range(n):
    t = out[i]
    kind, Nn, K, pro = meta[i]
    if kind == 2 and t[5]:
        rows.setdefault(("attention", 0, 0), []).append([us(t[1] - t[0]), us(t[2] - t[1]), us(t[3] - t[2]), us(t[4] - t[3]), us(t[5] - t[4]), us(t[5] - t[0]),
                                                         0, 0, 0, us(t[9] - t[0])])
        continue
    if kind != 0 or t[5] == 0:
        continue
    key = (int(Nn), int(K), int(pro))
    rows.setdefault(key, []).append([us(t[1] - t[0]), us(t[2] - t[1]), us(t[3] - t[2]), us(t[4] - t[3]), us(t[5] - t[4]), us(t[5] - t[0]),
                                     us(t[6] - t[3]), us(t[7] - t[6]), us(t[8] - t[7]), us(t[9] - t[0])])
print("%-22s %5s | %8s %8s %8s %8s %8s | %8s | %9s %9s %9s | %12s" % ("stage (N,K,pro)", "n", "barrier", "stats", "stageB", "mma-wait", "epilog", "total",
                                                                  "b->mma", "mma-loop", "commit", "prod-ahead"))
for key, v in rows.items():
    v = np.array(v)
    med = np.median(v, axis=0)
    print("%-22s %5d | %8.2f %8.2f %8.2f %8.2f %8.2f | %8.2f | %9.2f %9.2f %9.2f | %12.2f" % (str(key), len(v), *med))
print("inside 'stats' (norm stages): loads issued %.2f us, first row pair reduced %.2f us after the barrier" % (
    np.median([us(out[i][10] - out[i][1]) for i in range(n) if meta[i][3] in (1, 2) and out[i][10]]),
    np.median([us(out[i][11] - out[i][1]) for i in range(n) if meta[i][3] in (1, 2) and out[i][11]])))
G = torch.cuda.get_device_properties(0).multi_processor_count     # one stream-kernel CTA per SM
t2 = np.zeros((MAXO, G, 2), dtype=np.int64)
G = eng.lib.vv_stream_trace_read2(eng.h, t2.ctypes.data_as(C.c_void_p), MAXO)
if G:
    t2 = t2.reshape(-1)[: MAXO * G * 2].reshape(MAXO, G, 2)[:n]
    spread, mech, late = [], [], np.zeros(G)
    for i in range(1, n):
        arr, rel = t2[i, :, 0], t2[i, :, 1]
        if arr.min() == 0:
            continue
        spread.append((arr.max() - arr.min()) / 1e3)
        mech.append((rel.max() - arr.max()) / 1e3)
        late[np.argmax(arr)] += 1
    print("grid barrier over %d CTAs: arrival spread median %.2f us (p90 %.2f), last arrival -> last release median %.2f us (p90 %.2f)" % (
        G, np.median(spread), np.percentile(spread, 90), np.median(mech), np.percentile(mech, 90)))
    order = np.argsort(-late)[:8]
    print("CTAs arriving last most often:", [(int(c), int(late[c])) for c in order])
    # per-CTA mean lateness relative to the median arrival
    lat = np.array([t2[i, :, 0] - np.median(t2[i, :, 0]) for i in range(1, n) if t2[i, :, 0].min() > 0]) / 1e3
    m = lat.mean(axis=0)
    print("mean lateness (us) by CTA: min %.2f max %.2f; worst CTAs %s" % (m.min(), m.max(), [(int(c), round(float(m[c]), 2)) for c in np.argsort(-m)[:8]]))
    # wall-clock span of the kernel's stages (globaltimer, ns) against the SM-cycle stamps -> the SM clock the run really had
    rel_ok = [i for i in range(1, n) if t2[i, :, 0].min() > 0]
    if len(rel_ok) > 2:
        i0, i1 = rel_ok[0], rel_ok[-1]
        span_ns = float(t2[i1, :, 1].max() - t2[i0, :, 0].min())
        cyc = float(out[i1][1] - out[i0][0]) if out[i1][1] and out[i0][0] else 0.0
        print("stages %d..%d: %.1f us by globaltimer, %.0f SM cycles on the traced CTA -> effective SM clock %.0f MHz (stamps above assume %.0f)" % (
            i0, i1, span_ns / 1e3, cyc, cyc / (span_ns / 1e3) if span_ns else 0.0, a.mhz))
print("(attention rows: barrier | Q staged | first segment's pages | merge + partial | remaining segments)")
tot = sum(us(out[i][5] - out[i][0]) for i in range(n) if meta[i][0] in (0, 2) and out[i][5])
print("sum of traced stage totals: %.1f us; first->last stamp: %.1f us" % (tot, us(out[:n, 5].max() - out[:n, 0][out[:n, 0] > 0].min())))

# the same program by CUDA events, as bench.py times it (graph replays queued back to back)
fn = {"lm": lambda: (eng.lm_decode(), eng.kv_commit([1] * (2 * B))), "de": eng.codec_decode, "en": eng.semantic_encode}.get(a.prog[:2], lambda: eng.diffusion_sample(1.3))
for label, f in (("program call", fn),) + ((("lm_decode without kv_commit", eng.lm_decode),) if a.prog.startswith("lm") else ()):
    for _ in range(3):
        f()
    eng.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(eng.stream)
    for _ in range(16):
        f()
    e1.record(eng.stream)
    eng.sync()
    print("%s by CUDA events (tracing on): %.1f us" % (label, e0.elapsed_time(e1) * 1e3 / 16))
