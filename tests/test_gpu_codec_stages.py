"""The codec passes stage by stage: every stage boundary of the kernel-per-stage path (`vv_debug_codec_taps`) against float64 stage
references written here, and the GEMM dispatch behind `linear()` (`vv_debug_gemv2`) case by case.

Every frame runs two codec passes, the acoustic decoder (one 7.5 Hz latent -> 3200 samples) and the semantic encoder (3200 samples -> one
feature row).  Stages with T <= 8 frames and B * T <= 32 rows run inside the weight-stream programs (`decf:` / `encb:`); every other stage
runs as a chain of small launches: assemble_window*, dwconv_res, rows_norm*, conv_naive / conv_warp, advance and the tensor-core GEMMs of
`linear()`.  End to end the passes are held to 2e-3 (test_gpu_parity.py); here each stage is held on its own.

  * Teacher forcing: each tap's float64 reference runs on the GPU's own input to that stage (the previous tap), with a history that was
    fed those same GPU inputs frame after frame.  Only active rows are compared, so the error of a tap belongs to its stage alone.
  * Bound: 2e-5 rel-L2 per active row (BOUND), the single-linear bound of test_gpu_stream.py: bf16 weights on both sides, activations
    split into bf16 hi + lo inside the kernels, fp32 accumulation.  The stream hand-off taps cover whole weight-stream programs (the
    decoder front: stem + up to 11 blocks; the encoder back: up to 11 blocks + head conv) and are held to 1e-4 (HANDOFF_BOUND).
  * Sensitivity: a kernel that kept only the bf16 hi half of a Block1D's FFN operands moves that block's output by 8e-5 .. 3e-4 and the
    audio by up to 1.6e-3 when every decoder block does it, which the 2e-3 end-to-end bound lets through.  At T = 40, 800 and 3200 the
    per-stage bound must be at most a third of that move (checked without a GPU).
  * `vv_debug_gemv2`: every kernel `linear()` can pick, at both sides of the M, K and split-K switches, through the codec's own row
    maps, with NaN in the input padding and sentinels around the output; held to 2e-5 against float64.

Every tap and unit case is appended to reports/parity_report.jsonl.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from vibevoice_b200 import _native as NV

from test_gpu_parity import tiny2  # noqa: F401  (fixture)

BOUND, HANDOFF_BOUND = 2e-5, 1e-4
TAP_CONV, TAP_BLOCK, TAP_HANDOFF, TAP_OUT = 0, 1, 2, 3
DEC, ENC = "model.acoustic_tokenizer.decoder", "model.semantic_tokenizer.encoder"


def _rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ---- float64 stage references (time-major [n, T, C], like the kernels' activations) -------------------------------------------------
def _rms(x, w, eps):
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * w


def conv_ref(x, w, b, hist, stride=1, groups=1):
    """Streaming causal Conv1d (SConv1d): x [n, T, Cin], hist [n, k - stride, Cin] -> y [n, T / stride, Cout], next history."""
    xin = torch.cat([hist, x], 1)
    y = F.conv1d(xin.transpose(1, 2), w, b, stride=stride, groups=groups).transpose(1, 2)
    return y, xin[:, xin.shape[1] - hist.shape[1]:]


def convtr_ref(x, w, b, hist, stride):
    """Streaming ConvTranspose1d (SConvTranspose1d) with the causal trim on the right: x [n, T, Cin], hist [n, k - 1, Cin] ->
    y [n, T * stride, Cout] (the last T * stride outputs), next history."""
    k = w.shape[-1]
    xin = torch.cat([hist, x], 1)
    y = F.conv_transpose1d(xin.transpose(1, 2), w, b, stride=stride)
    y = y[..., :y.shape[-1] - (k - stride)]
    return y[..., -x.shape[1] * stride:].transpose(1, 2), xin[:, xin.shape[1] - (k - 1):]


def block_ref(x, w, hist, eps, ffn_bf16=False):
    """Block1D: x + gamma * dwconv7(RMSNorm(x)), then + ffn_gamma * linear2(GELU(linear1(RMSNorm(.)))).  hist [n, 6, C] holds the normed
    rows of earlier frames.  ffn_bf16 rounds both FFN operands to bf16 (the sensitivity check)."""
    y, hist = conv_ref(_rms(x, w("norm.weight"), eps), w("mixer.conv.conv.conv.weight"), w("mixer.conv.conv.conv.bias"), hist,
                       groups=x.shape[-1])
    x = x + y * w("gamma")
    rb = (lambda t: t.to(torch.bfloat16).double()) if ffn_bf16 else (lambda t: t)
    u = F.gelu(rb(_rms(x, w("ffn_norm.weight"), eps)) @ w("ffn.linear1.weight").T + w("ffn.linear1.bias"))
    return x + (rb(u) @ w("ffn.linear2.weight").T + w("ffn.linear2.bias")) * w("ffn_gamma"), hist


class PassRef:
    """The float64 layers of one pass (0 = acoustic decoder, 1 = semantic encoder), each with its own history of all B rows."""

    def __init__(self, sd, cfg, which, B):
        tc = cfg.acoustic_tokenizer_config if which == 0 else cfg.semantic_tokenizer_config
        self.sd, self.which, self.B, self.eps, self.hist = sd, which, B, tc.layernorm_eps, {}
        self.p = DEC if which == 0 else ENC
        self.depths = tc.decoder_depth_list if which == 0 else tc.encoder_depth_list
        self.ratios = list(tc.decoder_ratios) if which == 0 else list(reversed(tc.encoder_ratios))
        self.ns = len(self.depths)

    def w(self, name):
        return self.sd[name].double()

    def _run(self, key, rows, ctx, x, fn, commit=True):
        if key not in self.hist:
            self.hist[key] = torch.zeros(self.B, ctx, x.shape[-1], dtype=torch.float64)
        y, h = fn(self.hist[key][rows])
        if commit:
            self.hist[key][rows] = h
        return y

    def conv(self, i, x, rows):
        """The convolution in front of stage i (i = n_stages: the head conv)."""
        if i == self.ns:
            name, kind, s = self.p + ".head.conv.conv", "conv", 1
        elif self.which == 0 and i > 0:
            name, kind, s = "%s.upsample_layers.%d.0.convtr.convtr" % (self.p, i), "convtr", self.ratios[i - 1]
        else:
            name = "%s.%s_layers.%d.0.conv.conv" % (self.p, "upsample" if self.which == 0 else "downsample", i)
            kind, s = "conv", (1 if i == 0 else self.ratios[i - 1])
        W, b = self.w(name + ".weight"), self.w(name + ".bias")
        k = W.shape[-1]
        if kind == "convtr":
            return self._run(name, rows, k - 1, x, lambda h: convtr_ref(x, W, b, h, s))
        return self._run(name, rows, k - s, x, lambda h: conv_ref(x, W, b, h, s))

    def block(self, i, j, x, rows, ffn_bf16=False, commit=True):
        p = "%s.stages.%d.%d" % (self.p, i, j)
        return self._run(p, rows, 6, x, lambda h: block_ref(x, lambda n: self.w(p + "." + n), h, self.eps, ffn_bf16), commit)

    def stages(self, first, last, x, rows):
        """Stages [first, last): conv + blocks each."""
        for i in range(first, last):
            x = self.conv(i, x, rows)
            for j in range(self.depths[i]):
                x = self.block(i, j, x, rows)
        return x

    def zero(self, rows):
        for h in self.hist.values():
            h[rows] = 0


def tap_reference(ref, meta, x_in, prev, rows, handoff):
    """Teacher-forced reference of one tap: its stage run on the previous tap (prev), or, for the stream hand-off taps, the stages of the
    weight-stream program they stand for.  handoff = the stage at which this pass's stream program meets the kernel-per-stage path."""
    kind, stage, idx = meta[:3]
    if kind == TAP_CONV:
        return ref.conv(stage, prev, rows)
    if kind == TAP_BLOCK:
        return ref.block(stage, idx, prev, rows)
    if kind == TAP_HANDOFF:
        return ref.stages(0, stage, x_in, rows) if ref.which == 0 else prev     # decoder: stem + front stages; encoder: its input
    if ref.which == 0:
        return ref.conv(ref.ns, prev, rows)
    return ref.conv(ref.ns, ref.stages(handoff, ref.ns, prev, rows), rows)   # encoder: back stages + head conv


def tap_bound(which, kind):
    """The decoder front's output and the encoder back's output stand for whole weight-stream programs; every other tap for one stage."""
    return HANDOFF_BOUND if (which, kind) in ((0, TAP_HANDOFF), (1, TAP_OUT)) else BOUND


def check_pass(ref, taps, x_in, rows, **report_kw):
    """Every tap of one pass against its teacher-forced reference: [(meta, worst rel-L2 over the active rows, bound)]."""
    from test_gpu_parity import report
    out, prev = [], x_in
    handoff = next(m[1] for m, _ in taps if m[0] == TAP_HANDOFF)
    for meta, t in taps:
        want = tap_reference(ref, meta, x_in[rows], prev[rows], rows, handoff)
        got = t[rows].double()
        assert got.shape == want.shape, (meta, got.shape, want.shape)
        err = max(_rel(got[r], want[r]) for r in range(len(rows)))
        bound = tap_bound(ref.which, meta[0])
        report("codec_stage_tap", which=ref.which, meta=list(meta), rows=list(rows), rel_l2=err, bound=bound, **report_kw)
        out.append((meta, err, bound))
        prev = t.double()
    return out


def decoder_T(cfg):
    """Frames per decoder stage for one latent frame (the semantic encoder's are the same, reversed)."""
    T = [1]
    for r in cfg.acoustic_tokenizer_config.decoder_ratios:
        T.append(T[-1] * r)
    return T


def stream_split(T, B, ns):
    """(decoder front stages, first encoder back stage) of the host's rule: a stage runs in a stream program iff T <= 8 and B * T <= 32."""
    ok = lambda t: t <= 8 and B * t <= 32
    nf = 1
    while nf < ns - 1 and ok(T[nf]):
        nf += 1
    f = ns - 1
    while f > 1 and ok(T[::-1][f - 1]):
        f -= 1
    return nf, f


# ---- CPU: the references against the oracle's pinned fp32 streaming functions, and the sensitivity of the bound ---------------------
def _oracle_layers(sd, cfg, which):
    """[(kind, stage, index, oracle function of (x [n, C, T], state, rows))] of one pass in order."""
    from oracle import vv_oracle as O
    tc = cfg.acoustic_tokenizer_config if which == 0 else cfg.semantic_tokenizer_config
    depths = tc.decoder_depth_list if which == 0 else tc.encoder_depth_list
    ratios = list(tc.decoder_ratios) if which == 0 else list(reversed(tc.encoder_ratios))
    p, ns, eps = (DEC if which == 0 else ENC), len(depths), tc.layernorm_eps
    out = []
    for i in range(ns):
        if which == 0 and i > 0:
            f = lambda x, st, r, i=i: O.sconvtr_stream(sd, "%s.upsample_layers.%d.0" % (p, i), x, st, r, ratios[i - 1])
        elif which == 0:
            f = lambda x, st, r: O.sconv1d_stream(sd, p + ".upsample_layers.0.0", x, st, r)
        else:
            f = lambda x, st, r, i=i: O.sconv1d_stream(sd, "%s.downsample_layers.%d.0" % (p, i), x, st, r, stride=1 if i == 0 else ratios[i - 1])
        out.append((TAP_CONV, i, 0, f))
        for j in range(depths[i]):
            out.append((TAP_BLOCK, i, j, lambda x, st, r, i=i, j=j: O.block1d_stream(sd, "%s.stages.%d.%d" % (p, i, j), x, st, r, eps)))
    out.append((TAP_CONV, ns, 0, lambda x, st, r: O.sconv1d_stream(sd, p + ".head", x, st, r)))
    return out


def test_stage_references_match_the_oracle():
    """Each float64 stage reference (conv, transposed conv, strided conv, Block1D, head) against the oracle's fp32 function on the same
    input and the same history, over ragged frames of the tiny preset's decoder and semantic encoder: <= 1e-6 rel-L2."""
    from oracle import vv_oracle as O
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.synth import synth_state_dict
    cfg = preset_config("tiny")
    sd = synth_state_dict(cfg, 1234, torch.bfloat16, parts=("acoustic_decoder", "semantic"))
    g = torch.Generator().manual_seed(7)
    B = 3
    for which in (0, 1):
        ref, st = PassRef(sd, cfg, which, B), O.StreamState(B)
        worst = 0.0
        for rows in ([0, 1, 2], [1], [0, 2], [0, 1, 2], [2, 0]):
            r = torch.tensor(rows)
            x = torch.randn(len(rows), 1, 64, generator=g) if which == 0 else torch.randn(len(rows), 3200, 1, generator=g) * 0.3
            for kind, i, j, f in _oracle_layers(sd, cfg, which):
                want = f(x.transpose(1, 2).contiguous(), st, r).transpose(1, 2)
                got = ref.conv(i, x.double(), rows) if kind == TAP_CONV else ref.block(i, j, x.double(), rows)
                e = _rel(got, want)
                assert e <= 1e-6, (which, rows, kind, i, j, e)
                worst = max(worst, e)
                x = want
        assert worst > 0


def test_stage_bound_catches_bf16_ffn_operands():
    """A Block1D whose FFN operands keep only their bf16 hi half (the kernels split activations into bf16 hi + lo) must move that block's
    output by at least 3x BOUND at T = 40, 800 and 3200 (1.5b-l2 decoder, real activations after 3 frames of history)."""
    from test_gpu_parity import report
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.synth import synth_state_dict
    cfg = preset_config("1.5b-l2")
    sd = synth_state_dict(cfg, 1234, torch.bfloat16, parts=("acoustic_decoder",))
    ref = PassRef(sd, cfg, 0, 1)
    scale, bias = float(sd["model.speech_scaling_factor"]), float(sd["model.speech_bias_factor"])
    g = torch.Generator().manual_seed(1234)
    moved = {}
    for f in range(4):
        x = (torch.randn(1, 1, 64, generator=g).double() / scale - bias)
        for i in range(ref.ns):
            x = ref.conv(i, x, [0])
            for j in range(ref.depths[i]):
                if f == 3 and j == 0 and x.shape[1] in (40, 800, 3200):
                    moved[x.shape[1]] = _rel(ref.block(i, j, x, [0], ffn_bf16=True, commit=False), ref.block(i, j, x, [0], commit=False))
                x = ref.block(i, j, x, [0])
    report("codec_stage_sensitivity", bound=BOUND, moved=moved)
    assert sorted(moved) == [40, 800, 3200]
    for T, m in moved.items():
        assert m >= 3 * BOUND, (T, m)


# ---- GPU: teacher-forced stage parity --------------------------------------------------------------------------------------------------
def _frame_rows(B, f):
    """The active sets of test_gpu_presets._codec_checks: every row, and every third frame a ragged half."""
    return list(range(B)) if f % 3 != 2 or B == 1 else [r for r in range(B) if (r + f) % 2 == 0]


def _set_latent(eng, lat):
    with torch.cuda.stream(eng.stream):
        eng.latent.copy_(lat.cuda())


def _tap_parity(model, cfg, sdf, B, tag, n_frames=12):
    """n_frames of both passes through the tap entry, with ragged active sets and a state zeroing in the middle (from frame 7 on the
    k = 7 histories hold only real frames).  The encoder is fed the decoder's GPU output."""
    from test_gpu_parity import report
    eng = model.engine
    eng.codec_state_reset()
    dec, enc = PassRef(sdf, cfg, 0, B), PassRef(sdf, cfg, 1, B)
    nf, f0 = stream_split(decoder_T(cfg), B, dec.ns)
    scale, bias = float(sdf["model.speech_scaling_factor"]), float(sdf["model.speech_bias_factor"])
    g = torch.Generator().manual_seed(50 + B)
    worst = {}
    for f in range(n_frames):
        rows = _frame_rows(B, f)
        if f == n_frames // 2:
            zr = [0] if B == 1 else [0, B - 1]
            eng.codec_state_zero(zr); dec.zero(zr); enc.zero(zr)
        lat = torch.randn(B, 64, generator=g)
        _set_latent(eng, lat)
        dt = eng.codec_taps(0, rows)
        et = eng.codec_taps(1, rows)
        assert dt[0][0][:2] == (TAP_HANDOFF, nf) and [m for m, _ in et if m[0] == TAP_HANDOFF][0][1] == f0, (dt[0][0], nf, f0)
        res = {"decoder": check_pass(dec, dt, (lat.double() / scale - bias)[:, None, :], rows, preset=tag, B=B, frame=f),
               "encoder": check_pass(enc, et, dt[-1][1].double(), rows, preset=tag, B=B, frame=f)}
        for name, rs in res.items():
            for meta, err, bound in rs:
                key = "%s kind %d" % (name, meta[0])
                worst[key] = max(worst.get(key, 0.0), err)
        bad = [(name, meta, err, bound) for name, rs in res.items() for meta, err, bound in rs if not err < bound]
        assert not bad, (tag, B, f, rows, bad)
    report("codec_stage_taps_worst", preset=tag, B=B, frames=n_frames, worst=worst)
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 4, 8])
@pytest.mark.parametrize("preset", ["tiny", "1.5b-l2"])
def test_codec_stage_taps_vs_float64(preset, B):
    """Every tap of 12 frames of both passes.  1.5b-l2 has the real codec widths (C up to 2048, T up to 3200); at B = 8 the T = 8 stage
    of both passes leaves the stream programs (64 rows > 32) and runs here with C = 1024 > MR_MAXK_NORM, through rows_norm_block and an
    unfused GEMM instead of the folded-norm ring."""
    from test_gpu_presets import _model
    model, cfg, tok, sdf = _model(preset, B)
    try:
        _tap_parity(model, cfg, sdf, B, preset)
    finally:
        model.engine.close()


@pytest.mark.gpu
def test_codec_stage_taps_on_wgmma(monkeypatch):
    """VV_WGMMA=2: every prologue-free codec GEMM with M > 8 (transposed convs, FFN down-projections, and the FFN up-projections behind
    their separate RMSNorm) runs through its row map on the wgmma kernel."""
    from test_gpu_presets import _model
    monkeypatch.setenv("VV_WGMMA", "2")
    model, cfg, tok, sdf = _model("1.5b-l2", 2)
    try:
        _tap_parity(model, cfg, sdf, 2, "1.5b-l2 VV_WGMMA=2", n_frames=4)
    finally:
        model.engine.close()


# ---- GPU: state -------------------------------------------------------------------------------------------------------------------------
# the same rows on the same state and inputs: split-K and the stream programs sum with fp32 atomics whose order is not reproducible, and
# the difference carries through the pass.  Two engines differ by up to 2.1e-5 per tap (H100 80GB HBM3, 1.5b-l2, B = 2); a history off by
# one frame moves the taps by orders of magnitude more.
SAME = 1e-4


def _both_passes(eng, lat, rows):
    _set_latent(eng, lat)
    return eng.codec_taps(0, rows) + eng.codec_taps(1, rows)


def _pass_outputs(taps):
    """(audio [B, 3200], features [B, semantic_vae_dim]) from the output taps of a decoder + encoder tap list."""
    audio, feat = [t for m, t in taps if m[0] == TAP_OUT]
    return audio[:, :, 0], feat[:, 0]


def _row_diff(ta, tb, r):
    assert [m for m, _ in ta] == [m for m, _ in tb]
    return max(_rel(a[r], b[r]) for (_, a), (_, b) in zip(ta, tb))


@pytest.mark.gpu
def test_codec_taps_keep_state_like_production():
    """1. a row's history does not move while it is inactive: when it becomes active again its taps equal those of a twin engine that
    never saw those frames; 2. a row zeroed by codec_state_zero gives the taps of a freshly reset engine; 3. tap calls and the production
    vv_codec_decode_frame / vv_semantic_encode_frame interleaved on one engine give the pass outputs of tap calls alone."""
    from test_gpu_parity import report
    from test_gpu_presets import _model
    ma, cfg, _, _ = _model("1.5b-l2", 2, oracle=False)
    mb, _, _, _ = _model("1.5b-l2", 2, oracle=False)
    a, b = ma.engine, mb.engine
    try:
        g = torch.Generator().manual_seed(99)
        lats = [torch.randn(2, 64, generator=g) for _ in range(12)]
        a.codec_state_reset(); b.codec_state_reset()
        for f in range(3):
            _both_passes(a, lats[f], [0, 1]); _both_passes(b, lats[f], [0, 1])
        for f in range(3, 6):                      # row 1 inactive on a; b never sees these frames
            _both_passes(a, lats[f], [0])
        e_inactive = _row_diff(_both_passes(a, lats[6], [0, 1]), _both_passes(b, lats[6], [1]), 1)
        a.codec_state_zero([1]); b.codec_state_reset()
        e_zeroed = _row_diff(_both_passes(a, lats[7], [0, 1]), _both_passes(b, lats[7], [0, 1]), 1)
        a.codec_state_reset(); b.codec_state_reset()
        e_mixed = 0.0
        for f in range(8, 12):
            tb = _both_passes(b, lats[f], [0, 1])
            if f % 2:
                got = _pass_outputs(_both_passes(a, lats[f], [0, 1]))
            else:
                _set_latent(a, lats[f])
                a.upload_frame_inputs(torch.zeros(2, 64), [0, 1])
                a.codec_decode(); a.semantic_encode(); a.sync()
                got = (a.audio.cpu(), a.feat.cpu())
            want = _pass_outputs(tb)
            e_mixed = max(e_mixed, *(_rel(x[r], y[r]) for x, y in zip(got, want) for r in range(2)))
        report("codec_taps_state", inactive_row=e_inactive, zeroed_row=e_zeroed, mixed_calls=e_mixed, bound=SAME)
        assert e_inactive < SAME and e_zeroed < SAME and e_mixed < SAME, (e_inactive, e_zeroed, e_mixed)
    finally:
        a.close(); b.close()


@pytest.mark.gpu
def test_codec_taps_errors():
    """Too little tap space or a bad `which`: VV_ERR_INVALID with nothing launched; before vv_finalize_weights: VV_ERR_STATE."""
    from test_gpu_presets import _model
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.engine import Engine
    cfg = preset_config("tiny")
    raw = Engine(cfg, [1, 2], max_batch=1)
    try:
        assert raw.lib.vv_debug_codec_taps(raw.h, 0, None, None, None, None, 0, None, None) == -3
    finally:
        raw.close()
    model, cfg, _, _ = _model("tiny", 2, oracle=False)
    eng = model.engine
    try:
        n = eng.lib.vv_debug_codec_taps(eng.h, 0, None, None, None, None, 0, None, None)
        meta = np.zeros((n, 5), dtype=np.int32)
        assert eng.lib.vv_debug_codec_taps(eng.h, 0, None, None, None, None, 0, NV.iptr(meta), None) == n
        need = 2 * int((meta[:, 3].astype("int64") * meta[:, 4]).sum())
        taps = torch.zeros(need, device="cuda")
        P = lambda t: C.c_void_p(t.data_ptr())
        before = eng.launch_count()
        for which, space in ((0, need - 1), (2, need), (-1, need)):
            rc = eng.lib.vv_debug_codec_taps(eng.h, which, P(eng.latent), P(eng.active), P(eng.audio), P(taps), space, None, eng.s)
            assert rc == -1, (which, space, rc)
        assert eng.launch_count() == before
        torch.cuda.synchronize()
        assert not taps.any()
        assert eng.lib.vv_debug_codec_taps(eng.h, 0, P(eng.latent), P(eng.active), P(eng.audio), P(taps), need, None, eng.s) == n
    finally:
        eng.close()


# ---- GPU: vv_debug_gemv2, the GEMM dispatch of the kernel-per-stage path -----------------------------------------------------------------
PRO_NONE, PRO_RMSNORM, PRO_SILU = 0, 1, 3
EPI_NONE, EPI_RESID, EPI_GATED_RESID, EPI_GAMMA_RESID, EPI_GELU, EPI_SILU = 0, 2, 3, 4, 6, 7
KERNELS = ["gemv", "ring<1,GELU>", "ring<1,NONE>", "ring<0,GAMMA_RESID>", "ring<0,NONE>", "ring<0,GELU>", "ring<0,RESID>", "ring<-1,-1>",
           "gemm_mma", "wgmma"]
SENTINEL = 12345.0


def convtr_map(B, Tin, Cin):
    """Transposed conv of the decoder: row (b, t) reads the window [frame t-1 | frame t] of a [1 + Tin, Cin] window per batch row."""
    return dict(M=B * Tin, K=2 * Cin, T=Tin, rs=Cin, win=(1 + Tin) * Cin)


def strided_map(B, Tout, s, Cin):
    """Strided conv of the encoder: row (b, t) reads window rows [t s, t s + 2 s) of a [s + Tout s, Cin] window."""
    return dict(M=B * Tout, K=2 * s * Cin, T=Tout, rs=s * Cin, win=(s + Tout * s) * Cin)


def ctx6_map(B, T, Cin):
    """7-tap stem / head conv: row (b, t) reads window rows [t, t + 7) of a [6 + T, Cin] window."""
    return dict(M=B * T, K=7 * Cin, T=T, rs=Cin, win=(6 + T) * Cin)


# name: (M, N, K or a row map, prologue, epilogue, residual: None / "inplace" / "separate", kernel)
GEMV2_CASES = {
    "gemv_m8_rms_gelu": (8, 200, 512, PRO_RMSNORM, EPI_GELU, None, "gemv"),
    "gemv_m8_gamma_inplace": (8, 96, 2048, PRO_NONE, EPI_GAMMA_RESID, "inplace", "gemv"),
    "ring_rms_gelu_m9_k512": (9, 200, 512, PRO_RMSNORM, EPI_GELU, None, "ring<1,GELU>"),
    "ring_rms_gelu_m33_k504": (33, 130, 504, PRO_RMSNORM, EPI_GELU, None, "ring<1,GELU>"),
    "ring_rms_none_m32": (32, 63, 264, PRO_RMSNORM, EPI_NONE, None, "ring<1,NONE>"),
    "mma_rms_gelu_k520": (33, 130, 520, PRO_RMSNORM, EPI_GELU, None, "gemm_mma"),
    "ring_gamma_inplace_split1": (32, 96, 448, PRO_NONE, EPI_GAMMA_RESID, "inplace", "ring<0,GAMMA_RESID>"),
    "ring_gamma_inplace_split2": (32, 6400, 512, PRO_NONE, EPI_GAMMA_RESID, "inplace", "ring<0,GAMMA_RESID>"),
    "ring_gamma_inplace_split16": (33, 256, 2056, PRO_NONE, EPI_GAMMA_RESID, "inplace", "ring<0,GAMMA_RESID>"),
    "ring_gamma_separate": (40, 300, 1024, PRO_NONE, EPI_GAMMA_RESID, "separate", "ring<0,GAMMA_RESID>"),
    "ring_none_m9": (9, 65, 72, PRO_NONE, EPI_NONE, None, "ring<0,NONE>"),
    "ring_gelu_m33": (33, 129, 264, PRO_NONE, EPI_GELU, None, "ring<0,GELU>"),
    "ring_gelu_c1024_m64": (64, 4096, 1024, PRO_NONE, EPI_GELU, None, "ring<0,GELU>"),
    "ring_resid_separate": (17, 70, 136, PRO_NONE, EPI_RESID, "separate", "ring<0,RESID>"),
    "ring_resid_inplace_split8": (32, 128, 1024, PRO_NONE, EPI_RESID, "inplace", "ring<0,RESID>"),
    "ring_generic_silu": (20, 100, 96, PRO_NONE, EPI_SILU, None, "ring<-1,-1>"),
    "ring_generic_rms_gamma": (24, 100, 256, PRO_RMSNORM, EPI_GAMMA_RESID, "separate", "ring<-1,-1>"),
    "ring_generic_gated": (24, 100, 128, PRO_NONE, EPI_GATED_RESID, "separate", "ring<-1,-1>"),
    "mma_silu": (12, 100, 128, PRO_SILU, EPI_NONE, None, "gemm_mma"),
    "mma_rms_gamma_inplace_split8": (32, 128, 1024, PRO_RMSNORM, EPI_GAMMA_RESID, "inplace", "gemm_mma"),
    "wgmma_gamma_inplace": (200, 4000, 520, PRO_NONE, EPI_GAMMA_RESID, "inplace", "wgmma"),
    "wgmma_none_m65": (65, 12300, 136, PRO_NONE, EPI_NONE, None, "wgmma"),
    "convtr_window": (None, 160, convtr_map(2, 40, 64), PRO_NONE, EPI_NONE, None, "ring<0,NONE>"),
    "convtr_window_gemv": (None, 256, convtr_map(2, 4, 128), PRO_NONE, EPI_NONE, None, "gemv"),
    "convtr_window_wgmma": (None, 1800, convtr_map(2, 200, 64), PRO_NONE, EPI_NONE, None, "wgmma"),
    "strided_window": (None, 128, strided_map(2, 200, 4, 64), PRO_NONE, EPI_NONE, None, "ring<0,NONE>"),
    "ctx6_window": (None, 50, ctx6_map(2, 40, 32), PRO_NONE, EPI_NONE, None, "ring<0,NONE>"),
    "ctx6_window_gemv": (None, 40, ctx6_map(2, 4, 8), PRO_NONE, EPI_NONE, None, "gemv"),
}


def expected_split(M, N, K, inplace, kernel, G):
    """The host's split-K rule: an in-place residual on a tensor-core GEMM grid smaller than the GPU splits K over up to 16 CTAs."""
    gx, gy, nk = -(-N // 64), -(-M // 32), -(-K // 64)
    if not inplace or kernel in ("gemv", "wgmma") or nk < 8 or gx * gy >= G:
        return 1
    return max(min(nk // 2, 16, 2 * G // (gx * gy)), 1)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(GEMV2_CASES))
def test_gemv2_vs_float64(tiny2, case):
    """One linear() through vv_debug_gemv2: the kernel and split-K factor it reached, no NaN read from the input padding, nothing written
    outside y, and the result within 2e-5 of float64 (residual epilogues: relative to the GEMM term, not to the residual)."""
    from test_gpu_parity import report
    eng = tiny2[0].engine
    M, N, K, pro, epi, resid, kernel = GEMV2_CASES[case]
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    if isinstance(K, dict):                                   # a codec row map; batch windows 8 floats apart, NaN in between
        mp = K
        M, K, T, ldx, bs = mp["M"], mp["K"], mp["T"], mp["rs"], mp["win"] + 8
        x = torch.full((M // T * bs + 8,), float("nan"))
        for b in range(M // T):
            x[b * bs:b * bs + mp["win"]] = torch.randn(mp["win"], generator=g)
        offs = torch.tensor([(m // T) * bs + (m % T) * ldx for m in range(M)])
    else:
        T, ldx, bs = 0, K + 4, 0
        x = torch.full((M, ldx), float("nan"))
        x[:, :K] = torch.randn(M, K, generator=g) * 2.0
        x = x.flatten()
        offs = torch.arange(M) * ldx
    W = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    bias, nw = torch.randn(N, generator=g) * 0.1, torch.rand(K, generator=g) + 0.5
    gam = torch.rand(N, generator=g) + 0.5
    ldy, lda = N + 5, N + 3
    gate = torch.full((M, lda), float("nan"))
    gate[:, :N] = torch.rand(M, N, generator=g) + 0.5
    res = torch.full((M, lda), float("nan"))
    res[:, :N] = torch.randn(M, N, generator=g)
    y = torch.full((M + 3, ldy), SENTINEL)
    y[:M, :N] = res[:, :N] if resid == "inplace" else float("nan")
    d = {k: v.cuda() for k, v in dict(W=W, bias=bias, nw=nw, gam=gam, gate=gate, res=res, x=x, y=y).items()}
    P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    rp, ldres = (d["y"], ldy) if resid == "inplace" else ((d["res"], lda) if resid else (None, 0))
    ea = d["gam"] if epi == EPI_GAMMA_RESID else (d["gate"] if epi == EPI_GATED_RESID else None)
    info = np.zeros(2, dtype=np.int32)
    torch.cuda.synchronize()
    NV.check(eng.lib.vv_debug_gemv2(eng.h, P(d["W"]), P(d["bias"]), P(d["x"]), ldx, T, bs, P(d["y"]), ldy, P(rp), ldres, M, N, K, pro,
                                    P(d["nw"]), 1e-5, epi, P(ea), lda, NV.iptr(info), eng.s), "vv_debug_gemv2")
    got = d["y"].cpu()
    # float64 reference
    xr = x.double()[offs[:, None] + torch.arange(K)[None, :]]
    if pro == PRO_RMSNORM:
        xr = _rms(xr, nw.double(), 1e-5)
    elif pro == PRO_SILU:
        xr = F.silu(xr)
    lin = xr @ W.double().T + bias.double()
    r0 = res[:, :N].double()
    ref = {EPI_NONE: lin, EPI_GELU: F.gelu(lin), EPI_SILU: F.silu(lin), EPI_RESID: r0 + lin, EPI_GAMMA_RESID: r0 + gam.double() * lin,
           EPI_GATED_RESID: r0 + gate[:, :N].double() * lin}[epi]
    out = got[:M, :N].double()
    assert not torch.isnan(out).any(), "NaN in the output (input padding read, or an element not written)"
    assert torch.equal(got[:M, N:], torch.full_like(got[:M, N:], SENTINEL)), "write past N into the row padding of y"
    assert torch.equal(got[M:], torch.full_like(got[M:], SENTINEL)), "write past M into the rows after y"
    e = float((out - ref).norm() / ((ref - r0).norm() if resid else ref.norm()))
    G = torch.cuda.get_device_properties(0).multi_processor_count
    split = expected_split(M, N, K, resid == "inplace", kernel, G)
    report("codec_gemv2", case=case, M=M, N=N, K=K, kernel=KERNELS[info[0]], split_k=int(info[1]), rel_l2=e)
    assert (KERNELS[info[0]], int(info[1])) == (kernel, split), (case, KERNELS[info[0]], int(info[1]), kernel, split)
    if case.endswith("split2") or case.endswith("split8") or case.endswith("split16"):
        assert split == int(case.rsplit("split", 1)[1]), (case, split, G)
    assert e < 2e-5, (case, e)
