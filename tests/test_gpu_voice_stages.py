"""The voice-prompt encoder (`vv_voice_encode`, csrc/vv_voice.cuh) stage by stage: every stage boundary (`vv_debug_voice_taps`) against
float64 stage references written here, the grouping and chunking the workspace selects, and the isolation of voices in one group.

`vv_voice_encode` runs the non-streaming acoustic encoder (stem conv, 6 strided convs, the Block1Ds of every stage, head conv), the
sampling step and the acoustic connector.  Every GEMM runs on gemm_wgmma_kernel with bf16 weights, hi + lo bf16 operands and fp32
accumulation.  Voices run in groups and GEMM rows in chunks, both sized from the caller's workspace.  End to end, test_gpu_voice.py holds
it to 1e-4 (1e-3 at full width); here each stage is held on its own.

  * Teacher forcing: each tap's float64 reference runs on the GPU's own input to that stage (the previous tap).  Error = rel-L2 per
    (voice, time row), the denominator floored at 1e-3 of the tap's RMS row norm, so that a wrong boundary row is not diluted by a long
    voice.  Bound 2e-5 (BOUND), the single-stage bound of the codec taps, widened for GEMMs with K > 6 667 to 3e-9 K (tap_bound).
  * The references chained without teacher forcing match the oracle (`encoder_full`, `voice_prompt_embeds`) on the CPU.
  * Sensitivity: each bug class below, applied to one stage's reference on that stage's input at the GPU cases' own shapes and inputs,
    must move its tap by at least 3x its bound in at least one case (checked without a GPU).
  * A Python replica of the host's plan (voice_plan / voice_chunk) gives the workspace minimum, the groups, the chunks and the launch
    count of every case; the GPU cases assert that launch count, so each case provably reached the grouping and chunking it names.
  * Bit-exactness: every output row is computed by the same instructions whatever the grouping, so taps, mean and embeddings do not
    depend on the workspace, and a voice does not depend on its neighbours in a group (NaN or +-1e4 neighbours included).

Every case is appended to reports/parity_report.jsonl.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from vibevoice_b200 import _native as NV

from test_gpu_codec_stages import _rms, conv_ref
from test_gpu_parity import report

BOUND = 2e-5
# The error of one wgmma chain grows about linearly with K (fp32 accumulation): the convolution taps measured 1.0e-5 at K = 4 096 (tiny's
# last downsample), 1.8e-5 at 8 192 (small's) and 3.85e-5 at 16 384 (1.5b / 7b's; their head conv, K = 14 336: 3.0e-5) on an H100 80GB
# HBM3 at 700 W, about 2.3e-9 K.  A tap whose GEMM has K > 6 667 is held to 3e-9 K (4.9e-5 at 16 384) instead of BOUND.
K_SLOPE = 3e-9
VT_CONV, VT_MIX, VT_BLOCK, VT_FC1, VT_EMBEDS = range(5)
KINDS = ["conv", "mixer", "block", "fc1", "embeds"]
ENC, CON = "model.acoustic_tokenizer.encoder", "model.acoustic_connector"
SEED = 1234
WG_BK = 64                                   # k-block of gemm_wgmma_kernel
VOICE_CHUNK_MAX = 65535 * 64                 # rows of one GEMM launch
HOP = 3200


# ---- the host's plan, restated (vv_runtime.cu: voice_plan, voice_act_bytes, voice_chunk, vv_voice_encode) ------------------------------
def _a256(b):
    return (b + 255) & ~255


class Plan:
    def __init__(self, cfg, T):
        tc = cfg.acoustic_tokenizer_config
        ns, nf, ratios = len(tc.encoder_depth_list), tc.encoder_n_filters, list(reversed(tc.encoder_ratios))
        self.H, self.D, self.depths = cfg.decoder_config.hidden_size, tc.vae_dim, list(tc.encoder_depth_list)
        self.C = [nf << i for i in range(ns)]
        # conv i: (Cin, k, stride, K = k Cin rounded up to 8); conv ns = head
        self.convs = [(1, 7, 1)] + [(self.C[i - 1], 2 * ratios[i - 1], ratios[i - 1]) for i in range(1, ns)] + [(self.C[-1], 7, 1)]
        self.K = [(k * ci + 7) & ~7 for ci, k, _ in self.convs]
        self.T, t = [], T
        for i in range(ns):
            if i:
                t = -(-t // ratios[i - 1])
            self.T.append(t)
        self.F = t
        self.maxTC = max(t * c for t, c in zip(self.T, self.C))
        self.max_bpr = max([8 * self.H] + [32 * c for c in self.C] + [4 * k for k in self.K])
        self.smin = 64 * self.max_bpr + 512

    def act(self, g):
        return 2 * _a256(g * self.maxTC * 4) + _a256(g * self.T[0] * 4) + _a256(g * self.F * self.D * 4)

    def workspace_min(self):
        return self.act(1) + self.smin

    def workspace_default(self, n):
        """Engine.voice_encode's default."""
        need = self.workspace_min()
        return min(need * n + (256 << 20), max(need, 2 << 30))


def chunk(S, bpr, M):
    R = min(((S - 512) // bpr) & ~63, VOICE_CHUNK_MAX)
    return min(max(R, 64), M)


def run_plan(cfg, n, T, ws):
    """What vv_voice_encode does with `ws` bytes: {g, groups, launches, chunks}; chunks[(name, group)] = (rows per chunk, chunk count)."""
    p = Plan(cfg, T)
    g = n
    while g > 1 and p.act(g) + p.smin > ws:
        g -= 1
    Sb = ws - p.act(g)
    out = dict(g=g, groups=[], launches=0, chunks={})

    def gemm(name, gi, bpr, M, per_chunk):
        R = chunk(Sb, bpr, M)
        out["chunks"][(name, gi)] = (R, -(-M // R))
        out["launches"] += per_chunk * -(-M // R)
        return R

    for gi, v0 in enumerate(range(0, n, g)):
        nv = min(g, n - v0)
        out["groups"].append(nv)
        for i in range(len(p.C)):
            gemm("conv%d" % i, gi, 4 * p.K[i], nv * p.T[i], 2)
            for j in range(p.depths[i]):
                out["launches"] += 2                                     # voice_rms + voice_dwconv
                gemm("ffn%d.%d" % (i, j), gi, 32 * p.C[i], nv * p.T[i], 4)
        gemm("head", gi, 4 * p.K[-1], nv * p.F, 2)
        gemm("connector", gi, 8 * p.H, nv * p.F, 4)
    return out


# ---- the cases ---------------------------------------------------------------------------------------------------------------------------
# name: (preset, n, T, workspace, options).  workspace: "default" (Engine.voice_encode's), "min" (g = 1, 64-row chunks of the widest
# GEMM), "g2" (two voices per group, minimum scratch).  options: eps (False: eps = NULL), zero_after (the last voice is zero from there),
# cpu_T (the length the CPU sensitivity test runs a full-width case at).
CASES = {
    "tiny_n1_T1": ("tiny", 1, 1, "default", {}),
    "tiny_n1_T6": ("tiny", 1, 6, "default", {}),
    "tiny_n1_T7": ("tiny", 1, 7, "default", {}),
    "tiny_n1_T3199": ("tiny", 1, 3199, "default", {}),
    "tiny_n1_T3200": ("tiny", 1, 3200, "default", {"eps": False}),
    "tiny_n1_T3201": ("tiny", 1, 3201, "default", {}),
    "tiny_n3_T16001": ("tiny", 3, 5 * HOP + 1, "default", {}),
    "tiny_n3_min": ("tiny", 3, 4 * HOP + 17, "min", {}),
    "tiny_n3_g2": ("tiny", 3, 4 * HOP + 17, "g2", {"eps": False}),
    "tiny_F64": ("tiny", 1, 64 * HOP, "default", {}),
    "tiny_F65": ("tiny", 1, 64 * HOP + 1, "default", {}),
    "small_n5_g2": ("small", 5, 2 * HOP + 1234, "g2", {"zero_after": 3000}),
    "1.5b_n2_T240000": ("1.5b-l2", 2, 240000, "default", {"zero_after": 171111, "cpu_T": 2 * HOP + 1111, "cpu_zero_after": 5000}),
    "1.5b_n3_min": ("1.5b-l2", 3, 3 * HOP + 100, "min", {}),
    "7b_n1": ("7b-l2", 1, 3 * HOP + 1, "default", {}),
    "tiny_chunk_max": ("tiny", 1, VOICE_CHUNK_MAX + 1000, "default", {}),
}


def case_workspace(cfg, name):
    preset, n, T, kind, _ = CASES[name]
    p = Plan(cfg, T)
    return {"default": p.workspace_default(n), "min": p.workspace_min(), "g2": p.act(2) + p.smin}[kind]


def case_inputs(cfg, name, cpu=False):
    """Seeded wavs [n, T], sigma [n], eps [n, F, D] or None (CPU tensors)."""
    preset, n, T, kind, o = CASES[name]
    za = o.get("zero_after")
    if cpu and "cpu_T" in o:
        T, za = o["cpu_T"], o.get("cpu_zero_after")
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    wavs = torch.randn(n, T, generator=g) * 0.05
    if za is not None:
        wavs[-1, za:] = 0
    sigma = torch.randn(n, generator=g) * (cfg.acoustic_tokenizer_config.fix_std / 0.8)
    eps = torch.randn(n, -(-T // HOP), cfg.acoustic_vae_dim, generator=g) if o.get("eps", True) else None
    return wavs, sigma, eps


# ---- float64 stage references (time-major [n, T, C], like the kernels' activations) ------------------------------------------------------
def _bf(t):
    return t.to(torch.bfloat16).double()


def _shift(a, d, cross=False):
    """a[t - d] per voice with zeros for t < d; cross: the previous voice's last rows instead (voice 0: zeros)."""
    n, T, Cc = a.shape
    if cross:
        return F.pad(a.reshape(n * T, Cc), (0, 0, d, 0))[:n * T].reshape(n, T, Cc)
    return F.pad(a, (0, 0, d, 0))[:, :T]


class VoiceRef:
    """The float64 stages of the voice encoder on one device.  `bug` selects a mutation of the stage (SENSITIVITY)."""

    def __init__(self, sd, cfg, device="cpu"):
        self.sd, self.cfg, self.dev = sd, cfg, device
        tc = cfg.acoustic_tokenizer_config
        self.eps, self.ns, self.depths = tc.layernorm_eps, len(tc.encoder_depth_list), list(tc.encoder_depth_list)
        self.ratios = list(reversed(tc.encoder_ratios))
        self.scale, self.bias = float(sd["model.speech_scaling_factor"]), float(sd["model.speech_bias_factor"])
        self._w = {}

    def w(self, name):
        if name not in self._w:
            self._w[name] = self.sd[name].to(self.dev).double()
        return self._w[name]

    def conv(self, i, x, bug=None):
        """The convolution in front of stage i (i = ns: the head conv): left pad k - s, stride-alignment zeros on the right."""
        name = "%s.head.conv.conv" % ENC if i == self.ns else "%s.downsample_layers.%d.0.conv.conv" % (ENC, i)
        W, b = self.w(name + ".weight"), self.w(name + ".bias")
        Co, Ci, k = W.shape
        s = 1 if i in (0, self.ns) else self.ratios[i - 1]
        n, T_in, _ = x.shape
        T_out = -(-T_in // s)
        if bug is None:
            xr = torch.cat([x, x.new_zeros(n, T_out * s - T_in, Ci)], 1)
            return conv_ref(xr, W, b, x.new_zeros(n, k - s, Ci), stride=s)[0]
        # the kernel's window operand [n, T_out, k, Ci] (rows outside the voice zero) against the tap-major weight [Co, k Ci]
        pad = k - s + (bug == "pad+1")
        right = (T_out - 1) * s + k - pad - T_in
        tail = x.new_zeros(n, max(right, 0), Ci)
        if bug == "align_next_voice" and n > 1 and right > 0:
            tail[:-1] = F.pad(x[1:, :right], (0, 0, 0, max(0, right - T_in)))
        xp = torch.cat([x.new_zeros(n, pad, Ci), x, tail], 1)
        win = xp.unfold(1, k, s)[:, :T_out]                                  # [n, T_out, Ci, k]
        win = win.reshape(n, T_out, Ci * k) if bug == "channel_major" else win.transpose(2, 3).reshape(n, T_out, k * Ci)
        if bug == "bf16":
            win = _bf(win)
        Wt = W.permute(0, 2, 1).reshape(Co, k * Ci).clone()
        if bug == "last_kblock":
            Wt[:, (-(-((k * Ci + 7) & ~7) // WG_BK) - 1) * WG_BK:] = 0
        return win @ Wt.T + b

    def _bw(self, i, j, n):
        return self.w("%s.stages.%d.%d.%s" % (ENC, i, j, n))

    def mix(self, i, j, x, bug=None):
        """x + gamma * dwconv7(RMSNorm(x)) (causal, per voice)."""
        nw, W, b = self._bw(i, j, "norm.weight"), self._bw(i, j, "mixer.conv.conv.conv.weight"), self._bw(i, j, "mixer.conv.conv.conv.bias")
        gamma = self._bw(i, j, "ffn_gamma" if bug == "gammas_swapped" else "gamma")
        if bug in (None, "gammas_swapped"):
            y = conv_ref(_rms(x, nw, self.eps), W, b, x.new_zeros(x.shape[0], 6, x.shape[-1]), groups=x.shape[-1])[0]
            return x + y * gamma
        inv = torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + self.eps)
        acc = b.expand_as(x).clone()
        for j7 in range(7):
            d = 6 - j7
            wj = W[:, 0, d if bug == "dw_reversed" else j7]
            xs = _shift(x, d, cross=bug == "dw_guard")
            iv = inv if bug == "dw_inv_row" else _shift(inv, d, cross=bug == "dw_guard")
            acc = acc + wj * xs * iv * nw
        return x + acc * gamma

    def ffn(self, i, j, x, bug=None):
        """x + ffn_gamma * linear2(GELU(linear1(RMSNorm(x))))."""
        u = _rms(x, self._bw(i, j, "ffn_norm.weight"), self.eps)
        u = (_bf(u) if bug == "ffn1_bf16" else u) @ self._bw(i, j, "ffn.linear1.weight").T + self._bw(i, j, "ffn.linear1.bias")
        u = F.gelu(u, approximate="tanh") if bug == "gelu_tanh" else F.gelu(u)
        W2 = self._bw(i, j, "ffn.linear2.weight")
        if bug == "ffn2_bf16":
            u = _bf(u)
        if bug == "last_kblock":
            W2 = W2.clone()
            W2[:, (-(-W2.shape[1] // WG_BK) - 1) * WG_BK:] = 0
        return x + (u @ W2.T + self._bw(i, j, "ffn.linear2.bias")) * self._bw(i, j, "ffn_gamma")

    def fc1(self, mean, sigma, eps, bug=None):
        """(mean + sigma[v] eps + bias) * scale, then the connector's fc1."""
        x = mean
        if eps is not None and bug != "no_eps":
            s = sigma.roll(-1) if bug == "neighbour_sigma" else sigma
            x = mean + s[:, None, None] * eps
        feat = x * self.scale + self.bias if bug == "scale_first" else (x + self.bias) * self.scale
        if bug == "bf16":
            feat = _bf(feat)
        return feat @ self.w(CON + ".fc1.weight").T + self.w(CON + ".fc1.bias")

    def fc2(self, y1, bug=None):
        u = _rms(y1, self.w(CON + ".norm.weight"), 1e-6)
        return (_bf(u) if bug == "bf16" else u) @ self.w(CON + ".fc2.weight").T + self.w(CON + ".fc2.bias")

    def stage(self, meta, prev, wavs, sigma, eps, bug=None):
        """The reference of the tap `meta` on its input `prev` (the previous tap; the stem reads wavs [n, T, 1], fc1 the mean)."""
        kind, i, j = meta[:3]
        if kind == VT_CONV:
            return self.conv(i, wavs if i == 0 else prev, bug)
        if kind == VT_MIX:
            return self.mix(i, j, prev, bug)
        if kind == VT_BLOCK:
            return self.ffn(i, j, prev, bug)
        if kind == VT_FC1:
            return self.fc1(prev, sigma, eps, bug)
        return self.fc2(prev, bug)


def tap_plan(cfg, T):
    """The (kind, stage, index, T, C) list vv_debug_voice_taps reports, in run order."""
    p, ns = Plan(cfg, T), len(Plan(cfg, T).C)
    out = []
    for i in range(ns):
        out.append((VT_CONV, i, 0, p.T[i], p.C[i]))
        for j in range(p.depths[i]):
            out += [(VT_MIX, i, j, p.T[i], p.C[i]), (VT_BLOCK, i, j, p.T[i], p.C[i])]
    return out + [(VT_CONV, ns, 0, p.F, p.D), (VT_FC1, ns, 0, p.F, p.H), (VT_EMBEDS, ns, 0, p.F, p.H)]


def chain(ref, cfg, wavs, sigma, eps):
    """The references chained without teacher forcing: (meta, tap) in tap order (float64, on ref's device)."""
    prev = None
    w = wavs.to(ref.dev).double()[:, :, None]
    s = sigma.to(ref.dev).double()
    e = None if eps is None else eps.to(ref.dev).double()
    for meta in tap_plan(cfg, wavs.shape[1]):
        prev = ref.stage(meta, prev, w, s, e)
        yield meta, prev


def tap_bound(meta, p):
    """The bound of a tap: BOUND, or K_SLOPE * K of the GEMM that wrote it (conv: its window; block: linear2, K = 4C; fc2: K = H)."""
    kind, i = meta[:2]
    K = {VT_CONV: lambda: p.K[i], VT_MIX: lambda: 0, VT_BLOCK: lambda: 4 * p.C[i], VT_FC1: lambda: p.D, VT_EMBEDS: lambda: p.H}[kind]()
    return max(BOUND, K_SLOPE * K)


def row_err(got, want):
    """Worst rel-L2 over (voice, time row) [n, T, C], each row's denominator floored at 1e-3 of the tap's RMS row norm."""
    got, want = got.double(), want.double()
    den = want.norm(dim=-1)
    floor = 1e-3 * float(den.pow(2).mean().sqrt()) + 1e-300
    return float(((got - want).norm(dim=-1) / den.clamp_min(floor)).max())


def _sd(preset):
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.synth import synth_state_dict
    cfg = preset_config(preset)
    return cfg, synth_state_dict(cfg, SEED, torch.bfloat16, parts=("acoustic_encoder", "connectors"))


# ---- CPU: the references against the oracle ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("preset", ["tiny", "small"])
def test_stage_references_match_the_oracle(preset):
    """The float64 stages chained without teacher forcing against `encoder_full` (the latent mean) and `voice_prompt_embeds(noise=...)`
    (the embeddings) at n = 3 and T = 1, 3199, 3 * 3200 + 100: <= 1e-5 rel-L2 per voice."""
    from oracle import vv_oracle as O
    cfg, sd = _sd(preset)
    ref = VoiceRef(sd, cfg)
    g = torch.Generator().manual_seed(11)
    worst = {"mean": 0.0, "embeds": 0.0}
    for T in (1, 3199, 3 * HOP + 100):
        wavs = torch.randn(3, T, generator=g) * 0.05
        std_n, eps = torch.randn(3, generator=g), torch.randn(3, -(-T // HOP), cfg.acoustic_vae_dim, generator=g)
        sigma = std_n * (cfg.acoustic_tokenizer_config.fix_std / 0.8)
        taps = list(chain(ref, cfg, wavs, sigma, eps))
        mean = [t for m, t in taps if m[:2] == (VT_CONV, ref.ns)][0]
        want_mean = O.encoder_full(sd, cfg.acoustic_tokenizer_config, wavs[:, None, :], ENC)
        F_ = mean.shape[1]
        want_emb = O.voice_prompt_embeds(sd, cfg, wavs, torch.ones(3, F_, dtype=torch.bool), noise=(std_n, eps)).view(3, F_, -1)
        for v in range(3):
            for key, got, want in (("mean", mean[v], want_mean[v]), ("embeds", taps[-1][1][v], want_emb[v])):
                e = float((got - want.double()).norm() / want.double().norm())
                worst[key] = max(worst[key], e)
                assert e <= 1e-5, (preset, T, v, key, e)
    report("voice_stage_reference_vs_oracle", preset=preset, worst=worst, bound=1e-5)
    assert min(worst.values()) > 0


# ---- CPU: the plan replica ------------------------------------------------------------------------------------------------------------
def test_plan_replica_reaches_each_case():
    """Each case reaches the grouping and chunking its name claims, by the replica of the host's plan (the GPU cases assert the launch
    count it predicts, and its workspace minimum against vv_voice_encode_workspace)."""
    from vibevoice_b200.configuration import preset_config
    for name, (preset, n, T, kind, o) in CASES.items():
        cfg = preset_config(preset)
        p, ws = Plan(cfg, T), case_workspace(cfg, name)
        r = run_plan(cfg, n, T, ws)
        assert p.F == -(-T // HOP)
        assert ws >= p.workspace_min()
        if kind == "min":                       # one voice per group, the widest GEMM in 64-row chunks, the others chunked in proportion
            assert r["g"] == 1 and r["groups"] == [1] * n, name
            assert chunk(ws - p.act(1), p.max_bpr, 10 ** 9) == 64
            assert any(cnt > 1 for _, cnt in r["chunks"].values()), name
        if kind == "g2":
            assert r["g"] == 2 and r["groups"] == [2] * (n // 2) + [1] * (n % 2), (name, r["groups"])
        if kind == "default":
            assert r["g"] == n, name
        report("voice_plan", case=name, g=r["g"], groups=r["groups"], launches=r["launches"], workspace=ws)
    cfg = preset_config("tiny")
    r = run_plan(cfg, 1, CASES["tiny_chunk_max"][2], case_workspace(cfg, "tiny_chunk_max"))
    assert r["chunks"][("conv0", 0)] == (VOICE_CHUNK_MAX, 2)                       # the stem conv splits at VOICE_CHUNK_MAX
    # small n = 5 at g = 2: some FFN chunk ends inside a voice
    cfg = preset_config("small")
    _, n, T, _, _ = CASES["small_n5_g2"]
    p, r = Plan(cfg, T), run_plan(cfg, n, T, case_workspace(cfg, "small_n5_g2"))
    mid = [(i, j) for i in range(len(p.C)) for j in range(p.depths[i])
           if r["chunks"][("ffn%d.%d" % (i, j), 0)][1] > 1 and r["chunks"][("ffn%d.%d" % (i, j), 0)][0] % p.T[i]]
    assert mid, r["chunks"]
    # F = 64 / 65: one / two 64-row tiles in the last stage and the connector
    for name, tiles in (("tiny_F64", 1), ("tiny_F65", 2)):
        assert -(-Plan(cfg, CASES[name][2]).F // 64) == tiles


# ---- CPU: sensitivity -------------------------------------------------------------------------------------------------------------------
# class: [(tap kind, which stages, bug)].  Conv stages: "stem" = 0, "strided" = 1 .. ns-1, "last_down" = ns-1, "head" = ns; block
# classes run on block 0 of every stage.
SENSITIVITY = {
    "stem left pad off by one": [(VT_CONV, "stem", "pad+1")],
    "strided left pad off by one": [(VT_CONV, "strided", "pad+1")],
    "stride-alignment row reads the next voice": [(VT_CONV, "strided", "align_next_voice")],
    "channel-major window": [(VT_CONV, "strided", "channel_major"), (VT_CONV, "head", "channel_major")],
    "dwconv t >= d guard dropped": [(VT_MIX, "blocks", "dw_guard")],
    "dwconv inv[row] for inv[row - d]": [(VT_MIX, "blocks", "dw_inv_row")],
    "dwconv taps reversed": [(VT_MIX, "blocks", "dw_reversed")],
    "bf16-only window conv operand": [(VT_CONV, "convs", "bf16")],
    "bf16-only FFN1 operand": [(VT_BLOCK, "blocks", "ffn1_bf16")],
    "bf16-only FFN2 operand": [(VT_BLOCK, "blocks", "ffn2_bf16")],
    "bf16-only fc1 operand": [(VT_FC1, "connector", "bf16")],
    "bf16-only fc2 operand": [(VT_EMBEDS, "connector", "bf16")],
    "GELU tanh for erf": [(VT_BLOCK, "blocks", "gelu_tanh")],
    "gamma and ffn_gamma swapped": [(VT_MIX, "blocks", "gammas_swapped")],
    "FFN2 last k-block dropped": [(VT_BLOCK, "blocks", "last_kblock")],
    "head conv last k-block dropped": [(VT_CONV, "head", "last_kblock")],
    "last downsample last k-block dropped": [(VT_CONV, "last_down", "last_kblock")],
    "sampling with the neighbouring voice's sigma": [(VT_FC1, "connector", "neighbour_sigma")],
    "sampling with the scale before the bias": [(VT_FC1, "connector", "scale_first")],
    "sampling with eps ignored": [(VT_FC1, "connector", "no_eps")],
}


def _site(meta, where, ns):
    kind, i, j = meta[:3]
    return {"stem": i == 0, "strided": 0 < i < ns, "last_down": i == ns - 1, "head": i == ns, "convs": True,
            "blocks": j == 0, "connector": True}[where]


def test_sensitivity_of_the_bound():
    """Every bug class moves its tap by >= 3x the tap's bound in at least one GPU case (at the case's own shapes and seeded inputs; the
    240 000 sample full-width case at cpu_T), applied to one stage's reference on that stage's input."""
    from vibevoice_b200.configuration import preset_config
    moved = {c: [] for c in SENSITIVITY}
    sds = {}
    for name, (preset, n, T, kind, o) in CASES.items():
        if preset not in sds:
            sds = {preset: _sd(preset)}
        cfg, sd = sds[preset]
        ref = VoiceRef(sd, cfg)
        wavs, sigma, eps = case_inputs(cfg, name, cpu=True)
        p = Plan(cfg, wavs.shape[1])
        w, s, e = wavs.double()[:, :, None], sigma.double(), None if eps is None else eps.double()
        prev, best = None, {c: 0.0 for c in SENSITIVITY}
        for meta, tap in chain(ref, cfg, wavs, sigma, eps):
            for c, sites in SENSITIVITY.items():
                for kind_, where, bug in sites:
                    if meta[0] == kind_ and _site(meta, where, ref.ns):
                        best[c] = max(best[c], row_err(ref.stage(meta, prev, w, s, e, bug), tap) / tap_bound(meta, p))
            prev = tap
        for c in SENSITIVITY:
            moved[c].append(best[c])
    caught = {c: sum(m >= 3 for m in v) for c, v in moved.items()}
    report("voice_stage_sensitivity", bound=BOUND, k_slope=K_SLOPE, cases=len(CASES), caught=caught,
           worst_case_ratio={c: max(v) for c, v in moved.items()})
    missed = [c for c, k in caught.items() if k == 0]
    assert not missed, missed


# ---- GPU ------------------------------------------------------------------------------------------------------------------------------
_MODELS = {}


def _model(preset):
    """One engine per preset, the most recent kept (7b-l2 and 1.5b-l2 do not need to share the GPU)."""
    from test_gpu_voice import make_model
    if preset not in _MODELS:
        for m in _MODELS.values():
            m[0].engine.close()
        _MODELS.clear()
        m, cfg, tok, sd = make_model(preset)
        _MODELS[preset] = (m, cfg, sd)
    return _MODELS[preset]


@pytest.fixture(scope="module", autouse=True)
def _close_models():
    yield
    for m in _MODELS.values():
        m[0].engine.close()
    _MODELS.clear()


def _encode(eng, wavs, sigma, eps, ws):
    """vv_voice_encode: (mean, embeds, kernels launched)."""
    n, T = wavs.shape
    mean = torch.full((n, eng.voice_frames(T), eng.config.acoustic_vae_dim), float("nan"), device=eng.device)
    before = eng.launch_count()
    emb = eng.voice_encode(wavs, sigma, eps, mean_out=mean, workspace_bytes=ws)
    torch.cuda.synchronize()
    return mean, emb, eng.launch_count() - before


def _taps(eng, wavs, sigma, eps, ws):
    before = eng.launch_count()
    taps, emb = eng.voice_taps(wavs, sigma, eps, workspace_bytes=ws)
    torch.cuda.synchronize()
    return taps, emb, eng.launch_count() - before


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_voice_taps_vs_float64(case):
    """Every tap against its float64 reference run on the GPU's own input to that stage; the launch count the plan replica predicts, for
    the tap call and vv_voice_encode; the tap call's mean and embeddings equal vv_voice_encode's bitwise."""
    preset, n, T, kind, o = CASES[case]
    m, cfg, sd = _model(preset)
    eng = m.engine
    p = Plan(cfg, T)
    assert eng.voice_workspace_bytes(n, T) == p.workspace_min()
    ws = case_workspace(cfg, case)
    plan = run_plan(cfg, n, T, ws)
    wavs, sigma, eps = case_inputs(cfg, case)
    mean, emb, n_enc = _encode(eng, wavs, sigma, eps, ws)
    taps, temb, n_tap = _taps(eng, wavs, sigma, eps, ws)
    assert [mt for mt, _ in taps] == tap_plan(cfg, T)
    assert n_enc == n_tap == plan["launches"], (case, n_enc, n_tap, plan["launches"])
    assert torch.equal(temb, emb) and torch.equal(taps[-1][1], emb)
    assert torch.equal([t for mt, t in taps if mt[:2] == (VT_CONV, len(p.C))][0], mean)
    ref = VoiceRef(sd, cfg, "cuda")
    w, s, e = wavs.cuda().double()[:, :, None], sigma.cuda().double(), None if eps is None else eps.cuda().double()
    worst, prev, bad = {}, None, []
    for meta, tap in taps:
        err, bound = row_err(tap, ref.stage(meta, prev, w, s, e)), tap_bound(meta, p)
        key = KINDS[meta[0]]
        worst[key] = max(worst.get(key, 0.0), err)
        if not err < bound:
            bad.append((meta, err, bound))
        prev = tap.double()
    del taps, prev
    report("voice_stage_taps", case=case, preset=preset, n=n, T=T, workspace=ws, g=plan["g"], launches=n_tap, worst=worst, bound=BOUND,
           k_slope=K_SLOPE)
    assert not bad, (case, bad[:8])


def _tiny_case(n=3, T=4 * HOP + 17, seed=21):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, T, generator=g) * 0.05, torch.randn(n, generator=g) * 0.6, torch.randn(n, -(-T // HOP), 64, generator=g)


@pytest.mark.gpu
def test_taps_do_not_depend_on_the_workspace():
    """At the minimum, a middle (g = 2) and the default workspace every tap, the mean and the embeddings are bit-identical."""
    m, cfg, sd = _model("tiny")
    eng = m.engine
    wavs, sigma, eps = _tiny_case()
    n, T = wavs.shape
    p = Plan(cfg, T)
    runs = []
    for ws in (p.workspace_min(), p.act(2) + p.smin + 65536, p.workspace_default(n)):
        taps, emb, k = _taps(eng, wavs, sigma, eps, ws)
        assert k == run_plan(cfg, n, T, ws)["launches"]
        runs.append((ws, run_plan(cfg, n, T, ws)["g"], taps, emb))
    assert [r[1] for r in runs] == [1, 2, 3]
    for ws, g, taps, emb in runs[1:]:
        assert torch.equal(emb, runs[0][3]), ws
        for (ma, a), (mb, b) in zip(taps, runs[0][2]):
            assert ma == mb and torch.equal(a, b), (ws, ma)
    report("voice_taps_workspace", workspaces=[r[0] for r in runs], groups=[r[1] for r in runs], bit_identical=True)


@pytest.mark.gpu
@pytest.mark.parametrize("fill", ["nan", "big"])
def test_a_voice_does_not_depend_on_its_neighbours(fill):
    """Each voice of a 5-voice group equals the same voice encoded alone, bitwise (mean and embeddings); with every neighbour's wav,
    sigma and eps NaN or +-1e4 the middle voice is still bit-identical and finite."""
    m, cfg, sd = _model("tiny")
    eng = m.engine
    wavs, sigma, eps = _tiny_case(n=5, T=2 * HOP + 555, seed=22)
    n, T = wavs.shape
    mean, emb, _ = _encode(eng, wavs, sigma, eps, None)
    assert run_plan(cfg, n, T, Plan(cfg, T).workspace_default(n))["g"] == 5
    alone = [_encode(eng, wavs[v:v + 1], sigma[v:v + 1], eps[v:v + 1], None) for v in range(n)]
    for v in range(n):
        assert torch.equal(mean[v], alone[v][0][0]) and torch.equal(emb[v], alone[v][1][0]), v
    bad_w, bad_s, bad_e = wavs.clone(), sigma.clone(), eps.clone()
    keep = 2
    others = [v for v in range(n) if v != keep]
    if fill == "nan":
        bad_w[others], bad_s[others], bad_e[others] = float("nan"), float("nan"), float("nan")
    else:
        sign = torch.where(torch.rand(len(others), T, generator=torch.Generator().manual_seed(3)) < 0.5, -1.0, 1.0)
        bad_w[others], bad_s[others], bad_e[others] = 1e4 * sign, 1e4, 1e4
    mean2, emb2, _ = _encode(eng, bad_w, bad_s, bad_e, None)
    assert torch.isfinite(emb2[keep]).all() and torch.isfinite(mean2[keep]).all()
    assert torch.equal(mean2[keep], alone[keep][0][0]) and torch.equal(emb2[keep], alone[keep][1][0])
    report("voice_isolation", fill=fill, n=n, T=T, bit_identical=True)


@pytest.mark.gpu
def test_voice_taps_errors():
    """The tap call's errors, each the code vv_voice_encode gives, with nothing launched: null argument, misaligned workspace or eps,
    workspace below the minimum, n or T out of range, eps without sigma, too little tap space; no encoder weights: VV_ERR_STATE."""
    from test_gpu_voice import make_model
    m, cfg, sd = _model("tiny")
    eng = m.engine
    n, T = 2, 3 * HOP + 5
    p = Plan(cfg, T)
    need_taps = sum(n * t * c for _, _, _, t, c in tap_plan(cfg, T))
    assert eng.lib.vv_debug_voice_taps(eng.h, None, n, T, None, None, None, None, 0, None, 0, None, None) == len(tap_plan(cfg, T))
    meta = np.zeros((len(tap_plan(cfg, T)), 5), dtype=np.int32)
    assert eng.lib.vv_debug_voice_taps(eng.h, None, n, T, None, None, None, None, 0, None, 0, NV.iptr(meta), None) == len(meta)
    assert [tuple(r) for r in meta.tolist()] == tap_plan(cfg, T)
    ws = p.workspace_min()
    wavs, sig = torch.randn(n, T, device="cuda"), torch.ones(n, device="cuda")
    eps = torch.zeros(n * p.F * 64 + 4, device="cuda")
    out = torch.zeros(n, p.F, p.H, device="cuda")
    work = torch.empty(ws + 256, dtype=torch.uint8, device="cuda")
    taps = torch.zeros(need_taps, device="cuda")
    P = lambda t, off=0: C.c_void_p(t.data_ptr() + off) if t is not None else None
    cases = {
        "null wavs": (None, n, T, P(sig), P(eps), P(out), P(work), ws, need_taps),
        "null embeds": (P(wavs), n, T, P(sig), P(eps), None, P(work), ws, need_taps),
        "null workspace": (P(wavs), n, T, P(sig), P(eps), P(out), None, ws, need_taps),
        "eps without sigma": (P(wavs), n, T, None, P(eps), P(out), P(work), ws, need_taps),
        "misaligned workspace": (P(wavs), n, T, P(sig), P(eps), P(out), P(work, 16), ws, need_taps),
        "misaligned eps": (P(wavs), n, T, P(sig), P(eps, 4), P(out), P(work), ws, need_taps),
        "workspace below the minimum": (P(wavs), n, T, P(sig), P(eps), P(out), P(work), ws - 1, need_taps),
        "n = 0": (P(wavs), 0, T, P(sig), P(eps), P(out), P(work), ws, need_taps),
        "T = 0": (P(wavs), n, 0, P(sig), P(eps), P(out), P(work), ws, need_taps),
        "T > 2^30": (P(wavs), n, (1 << 30) + 1, P(sig), P(eps), P(out), P(work), ws, need_taps),
        "tap space": (P(wavs), n, T, P(sig), P(eps), P(out), P(work), ws, need_taps - 1),
    }
    before = eng.launch_count()
    for what, (w, nn, TT, s, e, o, wk, wsb, nt) in cases.items():
        rc = eng.lib.vv_debug_voice_taps(eng.h, w, nn, TT, s, e, o, wk, wsb, P(taps), nt, None, eng.s)
        assert rc == -1, (what, rc)
        if what != "tap space":
            assert eng.lib.vv_voice_encode(eng.h, w, nn, TT, s, e, None, o, wk, wsb, eng.s) == -1, what
    assert eng.launch_count() == before
    torch.cuda.synchronize()
    assert not taps.any() and not out.any()
    assert eng.lib.vv_debug_voice_taps(eng.h, P(wavs), n, T, P(sig), P(eps), P(out), P(work), ws, P(taps), need_taps, None, eng.s) == len(meta)
    assert eng.launch_count() - before == run_plan(cfg, n, T, ws)["launches"]
    raw, _, _, _ = make_model("tiny", drop=(ENC + ".",))
    try:
        e2 = raw.engine
        assert e2.lib.vv_debug_voice_taps(e2.h, None, n, T, None, None, None, None, 0, None, 0, None, None) == -3
        assert e2.lib.vv_debug_voice_taps(e2.h, P(wavs), n, T, P(sig), P(eps), P(out), P(work), ws, P(taps), need_taps, None, e2.s) == -3
    finally:
        raw.engine.close()
