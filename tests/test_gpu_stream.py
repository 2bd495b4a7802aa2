"""`-m gpu`: the persistent weight-stream kernel (wgmma with register accumulators, weight tiles by TMA through a ring that runs across
grid barriers; csrc/vv_stream.cuh) against a plain PyTorch fp32 reference of the same op.  Activations are split into bf16 hi + lo
inside the kernel, weights are bf16 on both sides -> agreement to ~1e-5 (summation order, 2^-17 relative activation rounding)."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from vibevoice_b200 import _native as NV

from test_gpu_parity import rel_l2, report, tiny2  # noqa: F401  (fixture)

SP_NONE, SP_RMSNORM, SP_SWIGLU, SP_GELU, SP_SILU = 0, 1, 3, 4, 6
SA_ONE, SA_GAMMA = 0, 2

SHAPES = [(2, 1536, 1536), (2, 2048, 1536), (2, 17920, 1536), (2, 1536, 8960), (2, 64, 1536), (2, 1536, 64), (1, 100, 264),
          (8, 1536, 1536), (4, 3584, 3584), (2, 37888, 3584), (3, 130, 72), (5, 4608, 896), (16, 512, 1024), (30, 2048, 512),
          (2, 9216, 4608), (8, 8192, 2048)]


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_stream_gemv_matches_torch(tiny2, M, N, K):
    eng = tiny2[0].engine
    g = torch.Generator().manual_seed(M * 1000003 + N * 101 + K)
    W = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    bias = torch.randn(N, generator=g) * 0.1
    nw = torch.rand(K, generator=g) + 0.5
    gam = torch.rand(N, generator=g) + 0.5
    Wd, bd, nwd, gamd = W.cuda(), bias.cuda(), nw.cuda(), gam.cuda()
    P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    cases = [(SP_NONE, SA_ONE, False, True), (SP_RMSNORM, SA_ONE, False, False), (SP_SWIGLU, SA_ONE, True, False),
             (SP_GELU, SA_GAMMA, True, True), (SP_SILU, SA_ONE, False, True)]
    for pro, ak, accumulate, with_bias in cases:
        x = torch.randn(M, 2 * K if pro == SP_SWIGLU else K, generator=g)
        xd = x.cuda()
        y = torch.full((M, N), 0.25, device="cuda")
        torch.cuda.synchronize()
        NV.check(eng.lib.vv_debug_stream_gemv(eng.h, P(Wd), P(bd) if with_bias else None, P(xd), P(y), M, N, K, pro, P(nwd), 1e-5, ak,
                                              P(gamd) if ak == SA_GAMMA else None, int(accumulate), eng.s), "vv_debug_stream_gemv")
        xt = x
        if pro == SP_RMSNORM:
            xt = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-5) * nw
        elif pro == SP_SWIGLU:
            xt = torch.nn.functional.silu(x[:, 0::2]) * x[:, 1::2]
        elif pro == SP_GELU:
            xt = torch.nn.functional.gelu(x)
        elif pro == SP_SILU:
            xt = torch.nn.functional.silu(x)
        ref = xt @ W.float().T
        if with_bias:
            ref = ref + bias
        if ak == SA_GAMMA:
            ref = ref * gam
        if accumulate:
            ref = ref + 0.25
        e = rel_l2(y, ref)
        report("stream_gemv", M=M, N=N, K=K, pro=pro, alpha=ak, accumulate=accumulate, rel_l2=e)
        assert e < 2e-5, (M, N, K, pro, ak, accumulate, e)
