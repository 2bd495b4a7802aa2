"""Micro-benchmark of the weight-streaming GEMV through the C ABI (vv_debug_gemv2): achieved HBM GB/s per shape, from the
kernel's device time (torch.profiler; every vv_debug_gemv2 call synchronises, so events around the calls would time the host too)
over launches that rotate through ~400 MB of weight copies, far more than the H100's 50 MB L2."""
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from vibevoice_b200 import _native as NV
from vibevoice_b200.configuration import preset_config
from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
from vibevoice_b200.synth import SynthTokenizer, synth_state_dict

cfg = preset_config("tiny")
tok = SynthTokenizer(cfg.decoder_config.vocab_size)
m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=1)
m.load_state_dict(synth_state_dict(cfg, 1, torch.bfloat16), tok)      # vv_debug_gemv2 needs finalized weights
eng = m.engine
P = lambda t: C.c_void_p(t.data_ptr())
shapes = [(2, 1536, 4608, 0, 2), (2, 1536, 8960, 0, 2), (2, 9216, 1536, 1, 5), (2, 17920, 1536, 1, 5), (2, 2048, 1536, 1, 0)] if os.environ.get("VV_SHORT") else [(2, 2048, 1536, 1, 0), (2, 1536, 1536, 0, 2), (2, 17920, 1536, 1, 5), (2, 1536, 8960, 0, 2), (2, 21504, 1536, 0, 0),
          (2, 9216, 1536, 2, 5), (2, 1536, 4608, 0, 3), (1, 8192, 2048, 1, 6), (1, 2048, 8192, 0, 4),
          (2, 4608, 3584, 1, 0), (2, 37888, 3584, 1, 5), (2, 3584, 18944, 0, 2), (8, 17920, 1536, 1, 5), (4, 17920, 1536, 1, 5)]
out = []
for M, N, K, pro, epi in shapes:
    wbytes = N * K * 2
    ncopy = max(2, int(400e6 // wbytes) + 1)
    W = torch.randn(ncopy, N, K, device="cuda", dtype=torch.bfloat16) * 0.02
    x = torch.randn(M, K, device="cuda")
    nw = torch.rand(K, device="cuda") + 0.5
    gam = torch.rand(N, device="cuda") + 0.5
    y = torch.zeros(M, N, device="cuda")
    # some shapes name LM / diffusion-head kinds linear() does not have; each runs as the nearest kind it has:
    # AdaLN (2) -> RMSNorm (1), gated residual (3) -> gamma residual (4), SwiGLU (5) -> SiLU (7)
    pro_ = pro if pro != 2 else 1
    epi_ = {3: 4, 5: 7}.get(epi, epi)
    res = P(y) if epi_ in (2, 4) else None
    info = np.zeros(2, dtype=np.int32)
    iters = 200

    def run(n):
        for i in range(n):
            NV.check(eng.lib.vv_debug_gemv2(eng.h, P(W[i % ncopy]), None, P(x), K, 0, 0, P(y), N, res, N, M, N, K, pro_, P(nw), 1e-6,
                                            epi_, P(gam), 0, NV.iptr(info), eng.s), "vv_debug_gemv2")
    run(20)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run(iters)
    kern = [e for e in prof.key_averages() if "gemv_kernel" in e.key]
    assert kern and sum(e.count for e in kern) == iters, [(e.key, e.count) for e in prof.key_averages()]
    us = sum(e.device_time_total for e in kern) / iters
    rec = dict(M=M, N=N, K=K, pro=pro_, epi=epi_, MB=round(wbytes / 1e6, 1), us=round(us, 2), GBps=round(wbytes / us / 1e3, 1))
    out.append(rec)
    print(rec, flush=True)
    del W
os.makedirs(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "reports"), exist_ok=True)
json.dump(out, open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "reports", "gemv_bench.json"), "w"))
