"""Micro-benchmark of the weight-streaming GEMV through the C ABI (vv_debug_gemv): achieved HBM GB/s per shape,
timed with CUDA events over back-to-back launches that rotate through ~400 MB of weight copies,
far more than the H100's 50 MB L2."""
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vibevoice_b200 import _native as NV
from vibevoice_b200.configuration import preset_config
from vibevoice_b200.engine import Engine

cfg = preset_config("tiny")
eng = Engine(cfg, [1, 2, 3, 4], max_batch=1)
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
    y = torch.zeros(M, N, device="cuda")
    pro_ = pro if pro != 2 else 1      # debug entry has no adaLN operands; RMSNORM has the same cost profile
    epi_ = epi if epi in (0, 2, 5, 6, 7) else 2
    iters = 200

    def run(n):
        for i in range(n):
            NV.check(eng.lib.vv_debug_gemv(eng.h, P(W[i % ncopy]), None, P(x), P(y), M, N, K, pro_, P(nw), 1e-6, epi_, eng.s))
    run(20)
    eng.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(eng.stream)
    run(iters)
    e1.record(eng.stream)
    eng.sync()
    us = e0.elapsed_time(e1) * 1e3 / iters
    rec = dict(M=M, N=N, K=K, pro=pro_, epi=epi_, MB=round(wbytes / 1e6, 1), us=round(us, 2), GBps=round(wbytes / us / 1e3, 1))
    out.append(rec)
    print(rec, flush=True)
    del W
os.makedirs(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "reports"), exist_ok=True)
json.dump(out, open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "reports",
                                 "gemv_bench_%s.json" % ("notma" if os.environ.get("VV_NO_TMA") == "1" else "tma")), "w"))
