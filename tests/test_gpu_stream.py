"""`-m gpu`: the persistent weight-stream kernel (wgmma with register accumulators, weight tiles by TMA through a ring that runs across
grid barriers; csrc/vv_stream.cuh) against a plain PyTorch fp32 reference of the same op.  Activations are split into bf16 hi + lo
inside the kernel, weights are bf16 on both sides -> agreement to ~1e-5 (summation order, 2^-17 relative activation rounding)."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from vibevoice_b200 import _native as NV

from test_gpu_parity import rel_l2, report, tiny2  # noqa: F401  (fixture)

SP_NONE, SP_RMSNORM, SP_ADALN, SP_SWIGLU, SP_GELU, SP_SILU = 0, 1, 2, 3, 4, 6
SA_ONE, SA_GATE, SA_GAMMA = 0, 1, 2

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


# ---- every stage feature of a linear stage through vv_debug_stream_gemv2, against a float64 reference ------------------------------
SENTINEL = 12345.0
G_SM = None


def _sm_count():
    global G_SM
    if G_SM is None:
        G_SM = torch.cuda.get_device_properties(0).multi_processor_count
    return G_SM


def _max_segments(N, K, G):
    """Largest number of (row tile, k range) segments any CTA owns (the kernel's stream-K split, vv_stream.cuh st_part)."""
    KB, R = (K + 63) // 64, (N + 127) // 128
    U = R * KB
    best = 0
    for c in range(G):
        u0, u1 = U * c // G, U * (c + 1) // G
        best = max(best, len({u // KB for u in range(u0, u1)}))
    return best


def _stream_case(eng, g, M, N, K, pro, ak, with_nw=True, with_bias=True, store=False, cap=0):
    """One linear with guard bands: x rows ldx > K (SwiGLU: > 2K) with NaN in the padding, AdaLN scale / shift and gate rows with NaN
    padding, y rows ldy > N plus extra rows, padding and extra rows holding a sentinel.  Returns (error, stages run): rel-L2 against a
    float64 reference, elementwise relative to the terms' magnitude for outputs of fewer than 16 elements."""
    Kx = 2 * K if pro == SP_SWIGLU else K
    ldx, pld, lda, ldy = Kx + 4, K + 8, N + 3, N + 5
    W = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    bias = torch.randn(N, generator=g) * 0.1
    nw = torch.rand(K, generator=g) + 0.5
    x = torch.full((M, ldx), float("nan"))
    x[:, :Kx] = torch.randn(M, Kx, generator=g) * 2.0
    shift, scale = torch.full((M, pld), float("nan")), torch.full((M, pld), float("nan"))
    shift[:, :K], scale[:, :K] = torch.randn(M, K, generator=g) * 0.3, torch.randn(M, K, generator=g) * 0.3
    alpha = torch.full((M, lda), float("nan"))
    alpha[:, :N] = torch.rand(M, N, generator=g) + 0.5
    gam = torch.rand(N, generator=g) + 0.5
    y = torch.full((M + 3, ldy), SENTINEL)
    y[:M, :N] = float("nan") if store else 0.25
    d = {k: v.cuda() for k, v in dict(W=W, bias=bias, nw=nw, x=x, shift=shift, scale=scale, alpha=alpha, gam=gam, y=y).items()}
    P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    torch.cuda.synchronize()
    al = d["alpha"] if ak == SA_GATE else (d["gam"] if ak == SA_GAMMA else None)
    adaln = pro == SP_ADALN
    n_st = NV.check(eng.lib.vv_debug_stream_gemv2(
        eng.h, P(d["W"]), P(d["bias"]) if with_bias else None, P(d["x"]), ldx, P(d["y"]), ldy, M, N, K, pro,
        P(d["nw"]) if with_nw else None, 1e-5, P(d["shift"]) if adaln else None, P(d["scale"]) if adaln else None, pld if adaln else 0,
        ak, P(al), lda, int(store), cap, eng.s), "vv_debug_stream_gemv2")
    got = d["y"].cpu()
    # float64 reference of the same op
    xd = x[:, :Kx].double()
    if pro in (SP_RMSNORM, SP_ADALN):
        xt = xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-5)
        if with_nw:
            xt = xt * nw.double()
        if adaln:
            xt = xt * (1 + scale[:, :K].double()) + shift[:, :K].double()
    elif pro == SP_SWIGLU:
        xt = torch.nn.functional.silu(xd[:, 0::2]) * xd[:, 1::2]
    elif pro == SP_GELU:
        xt = torch.nn.functional.gelu(xd)
    elif pro == SP_SILU:
        xt = torch.nn.functional.silu(xd)
    else:
        xt = xd
    ref, mag = xt @ W.double().T, xt.abs() @ W.double().abs().T          # mag: size of the summed terms, for outputs too small to average
    if with_bias:
        ref, mag = ref + bias.double(), mag + bias.double().abs()
    if ak == SA_GATE:
        ref, mag = ref * alpha[:, :N].double(), mag * alpha[:, :N].double()
    elif ak == SA_GAMMA:
        ref, mag = ref * gam.double(), mag * gam.double()
    if not store:
        ref, mag = ref + 0.25, mag + 0.25
    out = got[:M, :N]
    assert not torch.isnan(out).any(), "NaN in the output (padding read or store missed an element)"
    assert torch.equal(got[:M, N:], torch.full_like(got[:M, N:], SENTINEL)), "write past N into the row padding of y"
    assert torch.equal(got[M:], torch.full_like(got[M:], SENTINEL)), "write past M into the rows after y"
    if out.numel() < 16:
        # a lone output may be a cancelled sum, whose rel-L2 measures fp32 rounding of the terms, not the kernel: hold every element to
        # the same 2e-5 relative to the size of its terms instead
        return float(((out.double() - ref).abs() / mag).max()), n_st
    return rel_l2(out, ref), n_st


GEMV2_CASES = [  # (prologue, alpha, norm weight, store): the sampler's gate/up + gated down, the final layer, the noisy projection
    (SP_ADALN, SA_GATE, True, False), (SP_ADALN, SA_GATE, False, False), (SP_SWIGLU, SA_GATE, True, False),
    (SP_RMSNORM, SA_GAMMA, True, True)]


@pytest.mark.parametrize("K", [8, 56, 72])
@pytest.mark.parametrize("N", [1, 63, 129])
@pytest.mark.parametrize("M", [1, 8, 9, 16, 17, 32])
def test_stream_gemv2_features_vs_float64(tiny2, M, N, K):
    """AdaLN (with / without a norm weight) and SwiGLU prologues with the gated epilogue, and the store epilogue, at both sides of every
    MMA-height switch (M = 8 | 9, 16 | 17), with strided, NaN-padded inputs and sentinel-guarded outputs."""
    eng = tiny2[0].engine
    g = torch.Generator().manual_seed(M * 7919 + N * 31 + K)
    for pro, ak, with_nw, store in GEMV2_CASES:
        if store and K > 64:
            continue
        e, n_st = _stream_case(eng, g, M, N, K, pro, ak, with_nw=with_nw, store=store)
        report("stream_gemv2", M=M, N=N, K=K, pro=pro, alpha=ak, norm_w=with_nw, store=store, rel_l2=e)
        assert n_st == 1 and e < 2e-5, (M, N, K, pro, ak, with_nw, store, n_st, e)


def _expected_slices(M, N, K, cap, G):
    """The K-split rule of finish_stream for a linear without the attention merge: the fewest equal k-block slices whose operand
    (k-blocks a CTA touches x MMA height x 128 bytes) fits the cap; one k-block per slice if none does."""
    KB, R, nB = (K + 63) // 64, (N + 127) // 128, 16 if M <= 8 else (32 if M <= 16 else 64)
    fits = lambda kbs: min(-(-R * kbs // G), kbs) * nB * 128 <= cap
    kbs = KB
    if not fits(KB):
        for s in range(2, KB + 1):
            kbs = -(-KB // s)
            if fits(kbs) or kbs <= 1:
                break
    return -(-KB // kbs)


@pytest.mark.parametrize("shape", ["max_segments", "idle_ctas"])
def test_stream_gemv2_work_split_extremes(tiny2, shape):
    """max_segments: 7 G - 1 row tiles of 2 k-blocks -- the busiest CTAs own 8 (row tile, k range) segments, the most the host accepts.
    idle_ctas: one row tile of 64 k-blocks, fewer units than CTAs (most CTAs idle, the others one k-block each)."""
    eng = tiny2[0].engine
    G = _sm_count()
    M, N, K = (3, (7 * G - 1) * 128 - 5, 72) if shape == "max_segments" else (17, 100, 4096)
    if shape == "max_segments":
        assert _max_segments(N, K, G) == 8, _max_segments(N, K, G)
    else:
        assert (N + 127) // 128 * ((K + 63) // 64) < G
    g = torch.Generator().manual_seed(N + K)
    for pro, ak, with_nw, store in GEMV2_CASES[:3]:
        e, n_st = _stream_case(eng, g, M, N, K, pro, ak, with_nw=with_nw)
        report("stream_gemv2_split_extremes", M=M, N=N, K=K, pro=pro, alpha=ak, rel_l2=e)
        assert n_st == 1 and e < 2e-5, (M, N, K, pro, e)


@pytest.mark.parametrize("M,N,K,cap", [(9, 129, 72, 1), (5, 300, 1000, 1), (17, 4096, 1024, 16384), (32, 257, 200, 1), (8, 2048, 3584, 8000)])
def test_stream_gemv2_k_split_vs_float64(tiny2, M, N, K, cap):
    """A stage whose operand exceeds the cap runs as consecutive K slices that sum into y: only the first adds the bias, RMSNorm / AdaLN
    statistics still cover the whole row, SwiGLU reads its interleaved pairs at 2 k0.  cap = 1 -> one k-block per slice."""
    eng = tiny2[0].engine
    slices = _expected_slices(M, N, K, cap, _sm_count())
    assert slices > 1
    g = torch.Generator().manual_seed(M * 13 + N + K)
    for pro, ak, with_nw in [(SP_ADALN, SA_GATE, True), (SP_ADALN, SA_GATE, False), (SP_RMSNORM, SA_ONE, True), (SP_SWIGLU, SA_GATE, True),
                             (SP_GELU, SA_GAMMA, True), (SP_NONE, SA_ONE, True)]:
        e, n_st = _stream_case(eng, g, M, N, K, pro, ak, with_nw=with_nw, cap=cap)
        report("stream_gemv2_k_split", M=M, N=N, K=K, cap=cap, pro=pro, alpha=ak, stages=n_st, rel_l2=e)
        assert n_st == slices and e < 2e-5, (M, N, K, pro, ak, n_st, slices, e)
