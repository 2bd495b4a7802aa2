"""The diffusion sampler solver step by solver step: every block of the `samp:` weight-stream program (AdaLN-FFN head layers, the final
layer, the CFG + DPM-Solver++ update with noisy_images_proj) and the preamble that feeds it (t-embedder, cond_proj, the all-steps AdaLN
modulation GEMM) against a float64 reference.

End to end the sampler is held to 2e-4 rel-L2 on the final latent (test_gpu_parity.py, test_gpu_presets.py).  The arithmetic is far
better than that: the float64 chain below and the fp32 oracle agree to ~2.5e-7.  A head FFN linear whose operand lost its bf16 lo half, a
bf16-only modulation operand or a dropped second-order step can move the final latent by less than 2e-4.  Here:

  * Taps: `vv_debug_sampler_taps` runs the production preamble, then the sampler program as one launch per block.  Each block is built by
    the production builder and checked stage by stage against the production program (same kernel variant, same K split).  After each
    block it copies out what the block wrote.
  * Teacher forcing: each tap is compared with its float64 reference, run on the GPU's own input to that block (the previous tap) and the
    GPU's own modulation rows.  Head-layer updates (out - in) relative to the reference update, v, noisy_images_proj and the preamble
    linears are held per row to BOUND; z_{i+1} and x0_i elementwise, relative to the size of the terms they sum, to DPM_BOUND.
  * Production tie: the chain's final latent against vv_diffusion_sample and vv_frame_tail on the same inputs, to TIE_BOUND.
  * Rows never mix: NaN / +-1e4 in the conditions of inactive rows leave every active row's taps finite and unchanged.
  * Sensitivity (no GPU): at the GPU cases' own widths, batch sizes, step counts and inputs, each bug class moves its checked tap by at
    least 3 x that tap's bound in at least one case.

Every figure is appended to reports/parity_report.jsonl.
"""
import ctypes
import ctypes.util

import numpy as np
import pytest
import torch

from vibevoice_b200.configuration import preset_config
from vibevoice_b200.schedule import DPMSolverMultistepScheduler
from vibevoice_b200.synth import SynthTokenizer, param_specs, synth_state_dict, synth_tensor

from test_gpu_parity import SEED, rel_l2, report
from test_gpu_scale import PARTS

# Measured on an NVIDIA H100 80GB HBM3 (700 W power limit), worst over every case below: preamble linears 8.9e-6 (t-embedder 2.6e-6 /
# 8.9e-6, cond_proj 8.6e-6, modulation 8.9e-6), head-layer updates 8.8e-6, v 4.2e-6, noisy_images_proj 4.2e-6; z 1.7e-7, x0 1.6e-7.
BOUND = 2e-5           # per row: head-layer update, v, noisy_images_proj output, preamble linears (the single-linear bound of
                       # test_gpu_stream.py)
DPM_BOUND = 1e-6       # z_{i+1}, x0_i: elementwise, relative to the sum of the magnitudes of the terms (fp32 rounding of a few terms)
TIE_BOUND = 2e-5       # chain vs production, and inactive-row sentinels vs finite.  The stream-K fp32 atomics are not reproducible: two
                       # vv_diffusion_sample calls on the same inputs differ by up to 3.3e-6 (final latent), the chain and production by
                       # up to 3.4e-6, and two tap runs by up to 6.3e-6 in one row of one tap (H100)
ORACLE_BOUND = 1e-6    # float64 chain vs the fp32 oracle
SENTINEL = 1e4
P = "model.prediction_head"

# tap kinds (include/vibevoice_b200.h, vv_debug_sampler_taps)
T_HID, TEMB, COND, MOD, LAYER, V, Z, X0, HX, LATENT = range(10)
# linear() kernels (vv_debug_gemv2's numbering) and stream-kernel variants the sampler can run on
LIN_GEMV, LIN_RING_NONE, LIN_RING_GENERIC, LIN_WGMMA = 0, 4, 7, 9
VAR_SAMP_NB16, VAR_SAMP, VAR_ALL = 0, 1, 7

# (preset, B, runs, environment switch): a run = (steps, cfg_scale, sde); the runs of a case share one engine, in this order.  Modulation
# rows N * 2B: 2, 4, 8 (GEMV), 10, 12, 40, 60 (tensor-core ring on tiny), 20 .. 1024 (wgmma at 0.5B / 1.5B / 7B widths; 7b-l2 B = 8 with
# 64 steps fills s_mod and the wgmma plane buffer).  cond_proj: GEMV at B <= 4, ring at B = 5, 8; t-embedder: GEMV at N <= 8, ring above.
# 7b-l2 at B = 5, 8 splits the head's gate/up and down along K.
CASES = [
    ("tiny", 1, [(1, 1.3, False), (5, 1.3, False), (30, 1.3, False)], None),
    ("tiny", 2, [(2, 1.0, False), (3, 1.3, False), (10, 3.0, True)], None),
    ("tiny", 2, [(10, 1.3, False)], "VV_STREAM_GENERIC"),
    ("streaming-0.5b-l4", 1, [(10, 1.3, False)], None),
    ("1.5b-l2", 1, [(1, 1.3, False), (10, 1.3, False)], None),
    ("1.5b-l2", 4, [(3, 1.3, False), (10, 1.3, False)], None),
    ("1.5b-l2", 4, [(10, 1.3, False)], "VV_STREAM_NO_NB16"),
    ("1.5b-l2", 5, [(10, 1.3, True), (2, 1.3, False)], None),
    ("1.5b-l2", 8, [(30, 1.3, False)], None),
    ("7b-l2", 5, [(10, 1.3, False)], None),
    ("7b-l2", 8, [(2, 1.3, False), (64, 1.3, False)], None),
]
CASE_IDS = ["%s-B%d%s" % (p, b, "-" + env if env else "") for p, b, _, env in CASES]


def case_seed(preset, B, run):
    return sum(map(ord, preset)) * 131 + B * 17 + run


def run_inputs(cfg, B, steps, sde, seed):
    """cond [2B, H] (LM hidden rows: positive b, negative B + b), noise [B, 64], step noise [steps, B, 64] (SDE) of one run."""
    g = torch.Generator().manual_seed(seed)
    cond = torch.randn(2 * B, cfg.decoder_config.hidden_size, generator=g)
    noise = torch.randn(B, 64, generator=g)
    sn = torch.randn(steps, B, 64, generator=g) if sde else None
    return cond, noise, sn


def make_scheduler(hc, sde):
    s = DPMSolverMultistepScheduler(num_train_timesteps=hc.ddpm_num_steps, beta_schedule=hc.ddpm_beta_schedule,
                                    prediction_type=hc.prediction_type)
    return s.from_config(s.config, algorithm_type="sde-dpmsolver++") if sde else s


def schedule(hc, steps, sde):
    """(timesteps as the engine receives them [N] fp32, coefficient rows [N] of (a0, s0, ks, kx, rinv, order, kn) as fp32 values)."""
    s = make_scheduler(hc, sde)
    s.set_timesteps(steps)
    coef = [tuple(float(x) for x in row) + ((0.0,) if not sde else ()) for row in s.coef]
    return torch.from_numpy(s.timesteps.numpy().astype(np.float32)), coef


# ---- weights ----------------------------------------------------------------------------------------------------------------------------
def head_state_dict(cfg):
    """The synthetic head tensors (synth_tensor is seeded per name: the same values the full checkpoint has)."""
    return {n: synth_tensor(n, s, k, SEED, dtype=torch.bfloat16) for n, s, k in param_specs(cfg, ("head",)) if n.startswith(P + ".")}


def head_weights(sd, hc, device):
    f = lambda n: sd["%s.%s" % (P, n)].to(device=device, dtype=torch.float64)
    L = hc.head_layers
    layers = [dict(norm=f("layers.%d.norm.weight" % l), wg=f("layers.%d.ffn.gate_proj.weight" % l), wu=f("layers.%d.ffn.up_proj.weight" % l),
                   wd=f("layers.%d.ffn.down_proj.weight" % l)) for l in range(L)]
    wmod = torch.cat([f("layers.%d.adaLN_modulation.1.weight" % l) for l in range(L)] + [f("final_layer.adaLN_modulation.1.weight")])
    return dict(wn=f("noisy_images_proj.weight"), wc=f("cond_proj.weight"), wt0=f("t_embedder.mlp.0.weight"), wt2=f("t_embedder.mlp.2.weight"),
                layers=layers, wf=f("final_layer.linear.weight"), wmod=wmod, L=L, eps=hc.rms_norm_eps)


_W = {}


def cpu_weights(preset):
    """float64 CPU head weights of a preset (the most recent one is kept)."""
    if preset not in _W:
        _W.clear()
        cfg = preset_config(preset)
        _W[preset] = head_weights(head_state_dict(cfg), cfg.diffusion_head_config, "cpu")
    return _W[preset]


# ---- float64 reference of each block ----------------------------------------------------------------------------------------------------
def _rb(t):
    return t.to(torch.bfloat16).to(t.dtype)


def _silu(x):
    return x * torch.sigmoid(x)


def _rms(x, eps):
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps)


def _t_freqs():
    """The engine's 128 frequencies: expf((-9.210340371976184f * j) / 128.0f) in fp32 on the host (vv_finalize_weights)."""
    lib = ctypes.util.find_library("m")
    expf = getattr(ctypes.CDLL(lib), "expf", None) if lib else None
    out = np.zeros(128, np.float32)
    for j in range(128):
        a = np.float32(np.float32(-9.210340371976184) * np.float32(j)) / np.float32(128.0)
        if expf is not None:
            expf.restype, expf.argtypes = ctypes.c_float, [ctypes.c_float]
            out[j] = expf(float(a))
        else:
            out[j] = np.exp(a, dtype=np.float32)
    return torch.from_numpy(out)


_FREQS = _t_freqs()


def t_features(ts):
    """TimestepEmbedder.timestep_embedding: [cos, sin] of the fp32 argument t * freq (timestep_feat_kernel), taken in float64."""
    a = (ts.float().cpu()[:, None] * _FREQS[None]).double()
    return torch.cat([a.cos(), a.sin()], -1)


def ref_thid(W, feat, bug=None):
    """silu(t_embedder.mlp.0(features)); bug "temb0_hi": bf16-only operand."""
    return _silu((_rb(feat) if bug == "temb0_hi" else feat) @ W["wt0"].T)


def ref_temb(W, thid, bug=None):
    return (_rb(thid) if bug == "temb2_hi" else thid) @ W["wt2"].T


def ref_cond(W, cond, bug=None):
    return (_rb(cond) if bug == "cond_hi" else cond) @ W["wc"].T


def ref_mod(W, condp, temb, bug=None):
    """AdaLN modulation of every step: Linear(silu(cond_proj + temb_i)) -> [N, 2B, (3L+2)H]."""
    c = _silu(condp[None] + temb[:, None])
    return (_rb(c) if bug == "mod_hi" else c) @ W["wmod"].T


def ref_layer(W, x, mod, li, bug=None, src=None):
    """Head layer li: x + gate * down(SwiGLU(gate/up(RMSNorm(x) * w * (1 + scale) + shift))).  mod [2B, (3L+2)H] of the step;
    src = the layer whose shift / scale / gate are read (a bug class); bug "gu_hi" / "down_hi": bf16-only operand."""
    H = x.shape[-1]
    s = 3 * H * (li if src is None else src)
    sh, sc, g = mod[:, s:s + H], mod[:, s + H:s + 2 * H], mod[:, s + 2 * H:s + 3 * H]
    w = W["layers"][li]
    h = _rms(x, W["eps"]) * w["norm"] * (1 + sc) + sh
    if bug == "gu_hi":
        h = _rb(h)
    a = _silu(h @ w["wg"].T) * (h @ w["wu"].T)
    if bug == "down_hi":
        a = _rb(a)
    return x + g * (a @ w["wd"].T)


def ref_final(W, x, mod, bug=None):
    H, s = x.shape[-1], 3 * W["L"] * x.shape[-1]
    h = _rms(x, W["eps"]) * (1 + mod[:, s + H:s + 2 * H]) + mod[:, s:s + H]
    return (_rb(h) if bug == "final_hi" else h) @ W["wf"].T


def ref_proj(W, z, bug=None):
    """noisy_images_proj of z' [B, 64] for both CFG halves -> [2B, H]."""
    z = _rb(z) if bug == "proj_hi" else z
    return torch.cat([z, z]) @ W["wn"].T


def ref_dpm(v, z, x0p, c, cfg, noise=None, swap=False):
    """CFG + DPM-Solver++ step with the engine's fp32 coefficients c = (a0, s0, ks, kx, rinv, order, kn).  Returns z', x0 and the
    elementwise scales the check divides by: the sums of the magnitudes of the terms that make up x0 and z'."""
    a0, s0, ks, kx, rinv, order, kn = c
    B = z.shape[0]
    vc, vu = (v[B:], v[:B]) if swap else (v[:B], v[B:])
    vv = vu + cfg * (vc - vu)
    x0 = a0 * z - s0 * vv
    zn = ks * z - kx * x0
    x0s = abs(a0) * z.abs() + abs(s0) * (vu.abs() + abs(cfg) * (vc.abs() + vu.abs()))
    zs = abs(ks) * z.abs() + abs(kx) * x0s
    if int(order) == 2:
        zn = zn - 0.5 * kx * (rinv * (x0 - x0p))
        zs = zs + 0.5 * abs(kx * rinv) * (x0s + x0p.abs())
    if noise is not None:
        zn = zn + kn * noise
        zs = zs + abs(kn) * noise.abs()
    return zn, x0, zs, x0s


def ref_sample(W, cond, noise, ts, coef, cfg, step_noise=None):
    """The whole sampler, chained: a dict with the preamble results and one record per step (inputs and outputs of every block)."""
    dev = W["wn"].device
    cond, z = cond.to(dev, torch.float64), noise.to(dev, torch.float64)
    feat = t_features(ts).to(dev)
    thid = ref_thid(W, feat)
    temb = ref_temb(W, thid)
    condp = ref_cond(W, cond)
    mod = ref_mod(W, condp, temb)
    x0p = torch.zeros_like(z)
    x = ref_proj(W, z)
    out = dict(feat=feat, thid=thid, temb=temb, cond=cond, condp=condp, mod=mod, x=x, steps=[])
    for i in range(len(coef)):
        rec = dict(x_in=x, z_in=z, x0p=x0p, layers=[])
        for li in range(W["L"]):
            x = ref_layer(W, x, mod[i], li)
            rec["layers"].append(x)
        v = ref_final(W, x, mod[i])
        sn = step_noise[i].to(dev, torch.float64) if step_noise is not None else None
        z, x0, _, _ = ref_dpm(v, z, x0p, coef[i], cfg, sn)
        x = ref_proj(W, z)
        rec.update(v=v, z=z, x0=x0, x=x, noise=sn)
        out["steps"].append(rec)
        x0p = x0
    out["latent"] = z
    return out


# ---- error measures ---------------------------------------------------------------------------------------------------------------------
def row_err(got, want):
    """Largest per-row rel-L2 (rows = the leading dimensions)."""
    g, w = got.reshape(-1, got.shape[-1]).double(), want.reshape(-1, want.shape[-1]).double()
    return float(((g - w).norm(dim=-1) / (w.norm(dim=-1) + 1e-30)).max())


def update_err(out, x, ref):
    """Largest per-row rel-L2 of the layer update out - x against ref - x."""
    return row_err(out - x, ref - x)


def dpm_err(got, want, scale):
    return float(((got.double() - want).abs() / (scale + 1e-30)).max())


# ---- CPU: the reference against the oracle, and what the bounds catch --------------------------------------------------------------------
@pytest.mark.parametrize("preset", ["tiny", "1.5b-l2"])
def test_reference_chain_vs_oracle(preset):
    """`ref_sample` against the oracle's `sample_speech_tokens` (fp32, bf16 weights), ODE at 10 and 30 steps and SDE at 10 steps."""
    from oracle import vv_oracle as O
    cfg = preset_config(preset)
    hc = cfg.diffusion_head_config
    sd = head_state_dict(cfg)
    W = cpu_weights(preset)
    g = torch.Generator().manual_seed(7)
    H = cfg.decoder_config.hidden_size
    worst = 0.0
    for steps, sde in ((10, False), (30, False), (10, True)):
        pos, neg = torch.randn(2, H, generator=g), torch.randn(2, H, generator=g)
        noise = torch.randn(4, 64, generator=g)
        sn = [torch.randn(4, 64, generator=g) for _ in range(steps)] if sde else None
        want = O.sample_speech_tokens(sd, pos, neg, 1.3, steps, noise, n_layers=hc.head_layers, eps=hc.rms_norm_eps,
                                      algorithm_type="sde-dpmsolver++" if sde else "dpmsolver++", step_noise=sn)
        ts, coef = schedule(hc, steps, sde)
        got = ref_sample(W, torch.cat([pos, neg]), noise[:2], ts, coef, float(np.float32(1.3)),
                         torch.stack(sn)[:, :2] if sde else None)["latent"]
        e = rel_l2(got, want)
        report("sampler_ref_vs_oracle", preset=preset, steps=steps, sde=sde, rel_l2=e)
        worst = max(worst, e)
    assert worst <= ORACLE_BOUND, worst


def expected_kernel(M, N, silu=False):
    """The kernel linear() picks for an M-row GEMM with N outputs, no prologue (vv_runtime.cu: linear)."""
    if M > 8 and -(-N // 128) * -(-M // 64) >= 96:
        return LIN_WGMMA
    if M >= 9:
        return LIN_RING_GENERIC if silu else LIN_RING_NONE
    return LIN_GEMV


def expected_variant(B, env):
    if env == "VV_STREAM_GENERIC":
        return VAR_ALL
    return VAR_SAMP_NB16 if 2 * B <= 8 and env != "VV_STREAM_NO_NB16" else VAR_SAMP


def test_cases_reach_every_kernel():
    """Between them the GPU cases run each preamble linear on every kernel linear() picks for it, and the sampler on every kernel variant."""
    mod, cond, temb, var = set(), set(), set(), set()
    for preset, B, runs, env in CASES:
        cfg = preset_config(preset)
        H, L = cfg.decoder_config.hidden_size, cfg.diffusion_head_config.head_layers
        cond.add(expected_kernel(2 * B, H))
        var.add(expected_variant(B, env))
        for steps, _, _ in runs:
            mod.add(expected_kernel(steps * 2 * B, (3 * L + 2) * H))
            temb.add(expected_kernel(steps, H))
    assert mod == {LIN_GEMV, LIN_RING_NONE, LIN_WGMMA}, mod
    assert cond == {LIN_GEMV, LIN_RING_NONE} and temb == {LIN_GEMV, LIN_RING_NONE}, (cond, temb)
    assert var == {VAR_SAMP_NB16, VAR_SAMP, VAR_ALL}, var
    assert any(p == "7b-l2" and s == 64 for p, _, runs, _ in CASES for s, _, _ in runs)


BUGS = ("temb0_hi", "temb2_hi", "cond_hi", "mod_hi", "gu_hi@first", "gu_hi@last", "down_hi@first", "down_hi@last", "final_hi", "proj_hi",
        "layer_mod_step-1", "layer_mod_step+1", "layer_mod_layer-1", "layer_mod_layer+1", "final_mod_step-1", "no_order2", "rinv_next",
        "x0_prev2", "cfg_swap", "noise_step-1", "noise_step+1", "noise_row")


def bug_moves(W, r, coef, cfg, steps):
    """{bug: (move / bound)} of one run at the checked steps, each on its checked tap with the same measure as the GPU check."""
    L = W["L"]
    mv = {}
    put = lambda b, m: mv.__setitem__(b, max(mv.get(b, 0.0), m))
    put("temb0_hi", row_err(ref_thid(W, r["feat"], "temb0_hi"), r["thid"]) / BOUND)
    put("temb2_hi", row_err(ref_temb(W, r["thid"], "temb2_hi"), r["temb"]) / BOUND)
    put("cond_hi", row_err(ref_cond(W, r["cond"], "cond_hi"), r["condp"]) / BOUND)
    put("mod_hi", row_err(ref_mod(W, r["condp"], r["temb"], "mod_hi"), r["mod"]) / BOUND)
    N = len(coef)
    for i in sorted({0, 1, N // 2, N - 1} & set(range(N))):
        s, mod = r["steps"][i], r["mod"][i]
        for li in sorted({0, L - 1}):
            x = s["x_in"] if li == 0 else s["layers"][li - 1]
            ref = s["layers"][li]
            tag = "first" if li == 0 else "last"
            put("gu_hi@" + tag, update_err(ref_layer(W, x, mod, li, "gu_hi"), x, ref) / BOUND)
            put("down_hi@" + tag, update_err(ref_layer(W, x, mod, li, "down_hi"), x, ref) / BOUND)
            for d in (-1, 1):
                if 0 <= i + d < N:
                    put("layer_mod_step%+d" % d, update_err(ref_layer(W, x, r["mod"][i + d], li), x, ref) / BOUND)
                if 0 <= li + d < L:
                    put("layer_mod_layer%+d" % d, update_err(ref_layer(W, x, mod, li, src=li + d), x, ref) / BOUND)
        xl = s["layers"][-1]
        put("final_hi", row_err(ref_final(W, xl, mod, "final_hi"), s["v"]) / BOUND)
        if i >= 1:
            put("final_mod_step-1", row_err(ref_final(W, xl, r["mod"][i - 1]), s["v"]) / BOUND)
        put("proj_hi", row_err(ref_proj(W, s["z"], "proj_hi"), s["x"]) / BOUND)
        z, x0, zs, x0s = ref_dpm(s["v"], s["z_in"], s["x0p"], coef[i], cfg, s["noise"])
        dz = lambda zb: dpm_err(zb, z, zs) / DPM_BOUND
        c = list(coef[i])
        if int(c[5]) == 2:
            put("no_order2", dz(ref_dpm(s["v"], s["z_in"], s["x0p"], tuple(c[:5]) + (1,) + tuple(c[6:]), cfg, s["noise"])[0]))
            if i + 1 < N:
                put("rinv_next", dz(ref_dpm(s["v"], s["z_in"], s["x0p"], tuple(c[:4]) + (coef[i + 1][4],) + tuple(c[5:]), cfg, s["noise"])[0]))
            if i >= 2:
                put("x0_prev2", dz(ref_dpm(s["v"], s["z_in"], r["steps"][i - 2]["x0"], coef[i], cfg, s["noise"])[0]))
        zb, x0b, _, _ = ref_dpm(s["v"], s["z_in"], s["x0p"], coef[i], cfg, s["noise"], swap=True)
        put("cfg_swap", max(dz(zb), dpm_err(x0b, x0, x0s) / DPM_BOUND))
        if s["noise"] is not None:
            for d in (-1, 1):
                if 0 <= i + d < N:
                    put("noise_step%+d" % d, dz(ref_dpm(s["v"], s["z_in"], s["x0p"], coef[i], cfg, r["steps"][i + d]["noise"])[0]))
            if s["noise"].shape[0] > 1:
                put("noise_row", dz(ref_dpm(s["v"], s["z_in"], s["x0p"], coef[i], cfg, s["noise"].roll(1, 0))[0]))
    return mv


def test_bounds_catch_bug_classes():
    """At every GPU run's widths, batch size, step count, cfg scale and inputs (steps 0, 1, N / 2 and N - 1), how far each bug class moves
    its checked tap, in units of that tap's bound.  Every class must reach >= 3 in at least one GPU case; the catching cases are reported."""
    caught = {b: [] for b in BUGS}
    worst = {b: 0.0 for b in BUGS}
    for preset, B, runs, env in CASES:
        cfg = preset_config(preset)
        hc = cfg.diffusion_head_config
        W = cpu_weights(preset)
        for k, (steps, cfg_scale, sde) in enumerate(runs):
            cond, noise, sn = run_inputs(cfg, B, steps, sde, case_seed(preset, B, k))
            ts, coef = schedule(hc, steps, sde)
            cf = float(np.float32(cfg_scale))
            r = ref_sample(W, cond, noise, ts, coef, cf, sn)
            tag = "%s-B%d-N%d-cfg%g%s" % (preset, B, steps, cfg_scale, "-sde" if sde else "")
            for b, m in bug_moves(W, r, coef, cf, steps).items():
                report("sampler_sensitivity", case=tag, bug=b, ratio=m)
                worst[b] = max(worst[b], m)
                if m >= 3:
                    caught[b].append(tag)
    report("sampler_sensitivity_summary", caught=caught, worst_ratio=worst)
    missed = [b for b in BUGS if not caught[b]]
    assert not missed, (missed, worst)


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------------
def build_model(preset, B):
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    cfg = preset_config(preset)
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, SEED, torch.bfloat16, parts=PARTS)
    m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=B)
    m.load_state_dict(sd, tok)
    return m, cfg, sd


def set_run(eng, hc, steps, sde, cond, noise, sn):
    """Solver tables, inputs and (SDE) step noise of one run on the engine."""
    eng.set_scheduler(make_scheduler(hc, sde))
    eng.set_diffusion_steps(steps)
    with torch.cuda.stream(eng.stream):
        eng.hidden.copy_(cond.cuda())
        eng.noise.copy_(noise.cuda())
        if sde:
            eng.step_noise[:steps].copy_(sn.cuda())
    eng.sync()


def tap_dict(taps):
    return {(m[0], m[1], m[2]): (m, t) for m, t in taps}


def check_taps(taps, W, B, ts, coef, cfg, cond, noise, sn):
    """Every tap against its float64 block reference run on the GPU's own block input.  Returns the worst error per tap kind."""
    T = tap_dict(taps)
    g = lambda k, s=-1, l=-1: T[(k, s, l)][1].to("cuda", torch.float64)
    N, L, M = len(coef), W["L"], 2 * B
    e = dict(t_hid=row_err(g(T_HID), ref_thid(W, t_features(ts).cuda())), temb=row_err(g(TEMB), ref_temb(W, g(T_HID))),
             cond=row_err(g(COND), ref_cond(W, cond.cuda().double())))
    mod = g(MOD).view(N, M, -1)
    e["mod"] = row_err(mod, ref_mod(W, g(COND), g(TEMB)))
    assert torch.equal(T[(Z, -1, -1)][1], noise) and not T[(X0, -1, -1)][1].any()
    e["hx"] = row_err(g(HX), ref_proj(W, g(Z)))
    e.update(layer=0.0, v=0.0, z=0.0, x0=0.0)
    for i in range(N):
        x = g(HX, i - 1)
        for li in range(L):
            y = g(LAYER, i, li)
            e["layer"] = max(e["layer"], update_err(y, x, ref_layer(W, x, mod[i], li)))
            x = y
        e["v"] = max(e["v"], row_err(g(V, i), ref_final(W, x, mod[i])))
        z, x0, zs, x0s = ref_dpm(g(V, i), g(Z, i - 1), g(X0, i - 1), coef[i], cfg, sn[i].cuda().double() if sn is not None else None)
        e["z"] = max(e["z"], dpm_err(g(Z, i), z, zs))
        e["x0"] = max(e["x0"], dpm_err(g(X0, i), x0, x0s))
        e["hx"] = max(e["hx"], row_err(g(HX, i), ref_proj(W, g(Z, i))))
    assert torch.equal(T[(LATENT, N - 1, -1)][1], T[(Z, N - 1, -1)][1])
    return e


BOUNDS = dict(t_hid=BOUND, temb=BOUND, cond=BOUND, mod=BOUND, layer=BOUND, v=BOUND, hx=BOUND, z=DPM_BOUND, x0=DPM_BOUND)


def check_meta(taps, preset, B, steps, env):
    cfg = preset_config(preset)
    H, L = cfg.decoder_config.hidden_size, cfg.diffusion_head_config.head_layers
    T = tap_dict(taps)
    assert tuple(T[(T_HID, -1, -1)][0][5:]) == (expected_kernel(steps, H, silu=True), 1)
    assert tuple(T[(TEMB, -1, -1)][0][5:]) == (expected_kernel(steps, H), 1)
    assert tuple(T[(COND, -1, -1)][0][5:]) == (expected_kernel(2 * B, H), 1)
    assert tuple(T[(MOD, -1, -1)][0][5:]) == (expected_kernel(steps * 2 * B, (3 * L + 2) * H), 1)
    assert [m[0] for m, _ in taps] == [T_HID, TEMB, COND, MOD, Z, X0, HX] + ([LAYER] * L + [V, Z, X0, HX]) * steps + [LATENT]
    blocks = [m for m, _ in taps if m[0] in (LAYER, V, HX)]
    assert all(m[5] == expected_variant(B, env) for m in blocks), blocks
    layer_stages = max(m[6] for m in blocks if m[0] == LAYER)
    if preset == "7b-l2" and B >= 5:
        assert layer_stages > 2, layer_stages          # gate/up and down split along K
    return layer_stages


def production_latents(eng, cfg_scale, B):
    """vv_diffusion_sample twice and vv_frame_tail once on the engine's current inputs (all rows active)."""
    eng.upload_frame_inputs(eng.noise.cpu(), list(range(B)))
    out = []
    for call in (eng.diffusion_sample, eng.diffusion_sample, eng.frame_tail):
        with torch.cuda.stream(eng.stream):
            eng.latent.fill_(float("nan"))
        call(cfg_scale)
        eng.sync()
        out.append(eng.latent.cpu())
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("preset,B,runs,env", CASES, ids=CASE_IDS)
def test_sampler_steps_vs_float64(preset, B, runs, env, monkeypatch):
    """Teacher-forced parity of every tap of every run; the tap meta (kernels, stream variant, K split); the chain's final latent tied to
    vv_diffusion_sample and vv_frame_tail."""
    if env:
        monkeypatch.setenv(env, "1")
    model, cfg, sd = build_model(preset, B)
    eng = model.engine
    hc = cfg.diffusion_head_config
    try:
        W = head_weights(sd, hc, "cuda")
        worst = {k: 0.0 for k in BOUNDS}
        tie = spread = 0.0
        for k, (steps, cfg_scale, sde) in enumerate(runs):
            cond, noise, sn = run_inputs(cfg, B, steps, sde, case_seed(preset, B, k))
            set_run(eng, hc, steps, sde, cond, noise, sn)
            ts, coef = schedule(hc, steps, sde)
            taps = eng.sampler_taps(cfg_scale)
            stages = check_meta(taps, preset, B, steps, env)
            with torch.cuda.stream(eng.stream):
                e = check_taps(taps, W, B, ts, coef, float(np.float32(cfg_scale)), cond, noise, sn)
            eng.sync()
            chain = tap_dict(taps)[(LATENT, steps - 1, -1)][1]
            p1, p2, tail = production_latents(eng, cfg_scale, B)
            t = max(rel_l2(chain, p1), rel_l2(chain, tail))
            report("sampler_steps", case=preset, B=B, env=env, steps=steps, cfg=cfg_scale, sde=sde, layer_stages=stages,
                   chain_vs_production=t, production_spread=rel_l2(p1, p2), **e)
            for n in worst:
                worst[n] = max(worst[n], e[n])
            tie, spread = max(tie, t), max(spread, rel_l2(p1, p2))
        report("sampler_steps_summary", case=preset, B=B, env=env, chain_vs_production=tie, production_spread=spread, **worst)
        bad = {n: v for n, v in worst.items() if not v <= BOUNDS[n]}
        assert not bad, bad
        assert tie <= TIE_BOUND, (tie, spread)
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("preset,B,active", [("tiny", 2, [0]), ("1.5b-l2", 5, [0, 2, 3])], ids=["tiny-B2", "1.5b-l2-B5"])
@pytest.mark.parametrize("fill", ["nan", "big"])
def test_inactive_rows_never_mix(preset, B, active, fill):
    """The conditions of inactive rows (both CFG halves) hold NaN or +-1e4: every active row's taps stay finite and match a run whose
    inactive rows are finite, within TIE_BOUND per row."""
    model, cfg, sd = build_model(preset, B)
    eng = model.engine
    hc = cfg.diffusion_head_config
    try:
        steps = 10
        cond, noise, _ = run_inputs(cfg, B, steps, False, case_seed(preset, B, 99))
        rows = active + [B + b for b in active]
        dead = [r for r in range(2 * B) if r not in rows]
        bad = cond.clone()
        sgn = (1 - 2 * (torch.arange(cfg.decoder_config.hidden_size) % 2)).float()
        bad[dead] = float("nan") if fill == "nan" else SENTINEL * sgn
        out = []
        for c in (cond, bad):
            set_run(eng, hc, steps, False, c, noise, None)
            out.append(eng.sampler_taps(1.3))
        worst = 0.0
        for (m, a), (_, b) in zip(*out):
            if m[0] == MOD:
                a, b = a.view(steps, 2 * B, -1)[:, rows], b.view(steps, 2 * B, -1)[:, rows]
            elif m[0] in (COND, LAYER, V, HX):
                a, b = a[rows], b[rows]
            elif m[0] in (Z, X0, LATENT):
                a, b = a[active], b[active]
            assert torch.isfinite(b).all(), m
            if m[0] == X0 and m[1] == -1:
                assert not b.any(), m                      # proj(-1) writes x0 = 0
                continue
            worst = max(worst, row_err(b, a))
        report("sampler_inactive_rows", case=preset, B=B, fill=fill, worst_rel_l2=worst)
        assert worst <= TIE_BOUND, worst
    finally:
        eng.close()


@pytest.mark.gpu
def test_tap_call_errors():
    """Before vv_set_diffusion_steps: VV_ERR_STATE; too little tap space: VV_ERR_INVALID with nothing launched or written."""
    import ctypes as C
    model, cfg, sd = build_model("tiny", 1)
    eng = model.engine
    try:
        lib, h = eng.lib, eng.h
        ptr = lambda t: C.c_void_p(t.data_ptr())
        call = lambda taps, n, meta: lib.vv_debug_sampler_taps(h, ptr(eng.hidden), ptr(eng.noise), 1.3, ptr(eng.latent), taps, n, meta, eng.s)
        assert call(None, 0, None) == -3                   # a loaded model has no solver tables until its first generate()
        eng.set_diffusion_steps(3)
        n = call(None, 0, None)
        meta = np.zeros((n, 7), np.int32)
        assert call(None, 0, meta.ctypes.data_as(C.c_void_p)) == n and (meta[:, 5] == -1).all()
        need = int((meta[:, 3].astype(np.int64) * meta[:, 4]).sum())
        buf = torch.full((need,), 7.0, device="cuda")
        before = eng.launch_count()
        assert call(ptr(buf), need - 1, None) == -1
        eng.sync()
        assert eng.launch_count() == before and bool((buf == 7.0).all())
        assert call(ptr(buf), need, None) == n
        eng.sync()
        assert not bool((buf == 7.0).any())
    finally:
        eng.close()
