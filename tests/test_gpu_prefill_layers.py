"""The native prompt prefill kernel by kernel: each decoder layer of `vv_lm_prefill` (csrc/vv_prefill.cuh) run alone through
`vv_debug_prefill_taps`, every kernel's output checked against a float64 reference of that stage on the GPU's own input to it.

End to end (test_gpu_prefill.py) the prefill is held to "no worse than TorchPrefill, below 1e-2" rel-L2 per tensor, which can hide a causal
mask one key off at a page edge, a skipped page tile, a missing cross-tile rescale, a wrong GQA head map or a partial N tile that drops
columns.  Every prefill kernel is deterministic (no split-K, no atomics), so here:

  * Teacher forcing: layer l runs on the GPU's own output of layer l - 1; each tap is compared with its stage's float64 reference run on
    the GPU's input to that stage (the previous tap; for attention the Q tap and the bf16 K / V the pool holds).
  * bf16 taps (norm1, Q, the K / V written to the pool, norm2, silu(gate) * up): within ULP_BOUND bf16 ulp per element of the unrounded
    float64 value (`_ulps`, with its near-zero floor).  The attention reference applies the kernel's two documented roundings
    ("kernel-rounded"): P = bf16(2^(s log2e / sqrt(hd) - m_t)) with m_t the row's running max after the 64-key page tile of the key, and
    the row sum from the unrounded terms; the attention tap is held to ATTN_BOUND ulp of its terms' scale (see there), and compared with
    exact float64 softmax attention within EXACT_BOUND.
  * fp32 residual updates (out - in) after the o- and down-projections: update_bound(K) per row; hidden_last: FINAL_BOUND.
  * Production tie: the chain of per-layer tap calls and one `vv_lm_prefill` give bit-identical K / V and hidden_last.
  * Sensitivity (no GPU): at the GPU cases' shapes, positions and inputs, each bug class moves its checked tap by at least 3x that tap's
    bound in at least one GPU case.

Every figure is appended to reports/parity_report.jsonl.
"""
import ctypes as C

import pytest
import torch

from vibevoice_b200.configuration import preset_config

from test_gpu_parity import rel_l2, report
from test_gpu_scale import _structured_kv
from test_gpu_lm_layers import (LM, PoolMirror, _rb, _rms, _rope, _ulps, build_model, config as lm_config, import_prefix, inv_freq,
                                layer_weights, lm_layer_state_dict)

ULP_BOUND = 1.0        # bf16 taps, per element
# Attention against the kernel-rounded reference, in bf16 ulps of max(|o_d|, sum_j P_j |v_jd| / l, the head's RMS / 16): the reference
# cannot know on which side of a bf16 rounding boundary the kernel's fp32 scores put each P, and a P rounded to the other neighbour moves
# o_d in proportion to |v_jd|, not to |o_d|.  H100: at most 0.51 ulp of that scale, while in ulps of |o_d| alone near-zero outputs of rows
# with heavy weights reach 4.1; up to 5.5 % of the elements (a 32 768-key row) are not bit-equal.
ATTN_BOUND = 1.0
UPDATE_BOUND = 2e-5    # residual updates, per row (the per-layer bound of test_gpu_lm_layers.py) ...


def update_bound(K):
    """... up to K = 8 000.  The error of one wgmma chain of K products grows about linearly with K: H100, worst per row 6.3e-6 at
    K = 4 864, 1.2e-5 at 8 960, 2.3e-5 at 18 944 (the 7b down-projection); a bound of 2.5e-9 K keeps a 2x margin there."""
    return max(UPDATE_BOUND, 2.5e-9 * K)

FINAL_BOUND = 1e-6     # hidden_last against the float64 final norm of the GPU's last output row
# Attention against EXACT float64 softmax: the kernel's bf16 P carries up to 2^-8 relative rounding per weight and its bf16 output another
# 2^-9; per row (all heads) that is ~1e-3 of the row's norm unless the heads cancel.  The bound is loose on purpose -- the
# kernel-rounded comparison is the tight check -- and only catches an attention that is wrong by more than its own rounding.
EXACT_BOUND = 1e-2
# exact-mode reference chain vs qwen2_forward(act_bf16=True) (fp32): they differ only where float64 and fp32 arithmetic round a bf16 operand
# or cache entry differently, but the synthetic weights' peaky attention amplifies those ties in layer 1; measured <= 2.2e-3 (1.5b-l2,
# L = 65, layer-1 K), while a wrong mask, RoPE or head map moves these tensors by O(1)
ORACLE_BOUND = 5e-3
PT_NORM1, PT_Q, PT_ATTN, PT_RESID1, PT_NORM2, PT_SWIGLU, PT_OUT = range(7)


def config(name):
    """A preset, a toy of test_gpu_lm_layers ("gqa8", "gqa1"), or "gqa3": tiny with 3 query heads on 1 kv head of 64 -- Nqkv = 320 is a
    partial 128-column N tile with the Q / K boundary (192) inside a tile, and the o-projection has K = 192."""
    if name != "gqa3":
        return lm_config(name)
    cfg = preset_config("tiny")
    dc = cfg.decoder_config
    dc.num_attention_heads, dc.num_key_value_heads, dc.head_dim = 3, 1, 64
    return cfg


# ---- the workspace rule of vv_lm_prefill (vv_runtime.cu: pf_bytes) ---------------------------------------------------------------------
def _a256(b):
    return (b + 255) // 256 * 256


def pf_bytes(dc, R):
    H, I, nq = dc.hidden_size, dc.intermediate_size, dc.num_attention_heads * dc.head_dim
    return _a256(R * 4 * H) + _a256(R * 2 * max(H, nq)) + _a256(R * 2 * max(I, nq))


def workspace(dc, n, kind):
    """"min": one 64-row chunk; "default": Engine.lm_prefill's default (the whole prompt, within 2 GB)."""
    need = pf_bytes(dc, 64)
    return need if kind == "min" else min(need * ((n + 63) // 64), max(need, 2 << 30))


def chunk_rows(dc, n, ws):
    R = min((n + 63) // 64 * 64, 65535 * 128)
    while R > 64 and pf_bytes(dc, R) > ws:
        R -= 64
    return R


# (config, n, pos0, workspace): page edges, unaligned pos0 (query tiles straddling pages), H = 128 (two k-blocks, fewer than the three-deep
# cp.async prefetch), head_dim 64, GQA 1 / 3 / 7 / 8, many chunks, and rows that end at the model's last position over a structured prefix
CASES = ([("tiny", n, p, w) for n in (1, 64, 65, 129) for p in (0, 77) for w in ("min", "default")] +
         [("tiny64", 200, 63, "default"), ("tiny64", 1000, 0, "min"),
          ("gqa1", 129, 1, "default"), ("gqa8", 129, 1, "default"), ("gqa3", 129, 0, "default"),
          ("streaming-0.5b-l4", 1000, 0, "default"), ("streaming-0.5b-l4", 65, 8127, "default")] +
         [("1.5b-l2", n, 0, "default") for n in (1, 63, 64, 65, 1000)] +
         [("1.5b-l2", 5000, 0, "min"), ("1.5b-l2", 129, 65407, "default"),
          ("7b-l2", 1000, 0, "default"), ("7b-l2", 777, 31991, "default")])
CASE_IDS = ["%s-n%d-p%d-%s" % c for c in CASES]
FRAGMENTED = ("1.5b-l2", 300, 70, "default")      # seq 1 on interleaved, descending pages (test_fragmented_pages)


def case_seed(name, n, pos0):
    return sum(map(ord, name)) * 131 + 7 * n + pos0


def case_inputs(dc, name, n, pos0):
    """The residual input of layer 0 [n, H] and the structured bf16 prefix [(k, v) [nkv, pos0, hd] per layer] (None when pos0 = 0)."""
    s = case_seed(name, n, pos0)
    x = torch.randn(n, dc.hidden_size, generator=torch.Generator().manual_seed(s)) * 0.5
    if not pos0:
        return x, None
    g = torch.Generator().manual_seed(s + 1)
    return x, [_structured_kv(dc.num_key_value_heads, pos0, dc.head_dim, g) for _ in range(dc.num_hidden_layers)]


# ---- float64 references -----------------------------------------------------------------------------------------------------------------
def _rot(x, ang):
    """RoPE of x [n, heads, hd] at fp32 angles ang [n, hd/2] (fp32(pos) * inv_freq in fp32, as HF and the kernel), cos / sin in float64."""
    a = ang.double()
    return _rope(x, a.cos()[:, None], a.sin()[:, None])


def angles(dc, pos, device="cpu"):
    return pos.float().to(device)[:, None] * inv_freq(dc).to(device)[None]


def qkv_ref(w, dc, h, pos, bug=None, R=None, pos0=0):
    """h [n, H] the bf16 norm1 operand (float64), pos [n] absolute positions -> rotated q [n, nh, hd], rotated k, v [n, nkv, hd]."""
    n, nh, nkv, hd = h.shape[0], dc.num_attention_heads, dc.num_key_value_heads, dc.head_dim
    q = (h @ w["wq"].T + w["bq"]).view(n, nh, hd)
    k = (h @ w["wk"].T + (0 if bug == "no_k_bias" else w["bk"])).view(n, nkv, hd)
    v = (h @ w["wv"].T + (0 if bug == "no_v_bias" else w["bv"])).view(n, nkv, hd)
    p = pos
    if bug == "rope_pos+1":
        p = pos + 1
    elif bug == "rope_pos-1":
        p = pos - 1
    elif bug == "rope_chunk_local":
        p = (pos - pos0) % R
    ang = angles(dc, p, h.device)
    if bug == "rope_interleaved":         # rotate (d, d+1) pairs instead of (d, d + hd/2)
        a = ang.double()
        cs, sn = a.cos()[:, None], a.sin()[:, None]
        rot = lambda t: torch.stack([t[..., 0::2] * cs - t[..., 1::2] * sn, t[..., 1::2] * cs + t[..., 0::2] * sn], -1).flatten(-2)
        return rot(q), rot(k), v
    return _rot(q, ang), _rot(k, ang), v


def scale_log2(hd):
    """The kernel's fp32 constant log2(e) / sqrt(hd)."""
    return float(torch.tensor(1.4426950408889634, dtype=torch.float32) / torch.tensor(float(hd), dtype=torch.float32).sqrt())


def attention(q, K, V, pos, mode, bug=None, scale_out=None):
    """Causal attention of rows q [r, nh, hd] at absolute positions pos [r] over keys K, V [Lk, nkv, hd] (positions 0 .. Lk-1), float64.
    mode "exact": float64 softmax.  mode "kernel": P = bf16(2^(s * log2e/sqrt(hd) - m_t)), m_t the row's running max after the 64-key
    tile holding the key; the row sum of the unrounded terms; tiles rescaled to the final max.  A row with no visible key gives 0.
    bug: one of the attention bug classes (the sensitivity test).  scale_out (kernel mode): filled with sum_j P_j |v_jd| / l."""
    r, nh, hd = q.shape
    Lk, nkv = K.shape[0], K.shape[1]
    dev = q.device
    G = nh // nkv
    j = torch.arange(Lk, device=dev)[None]
    p = pos.to(dev)[:, None]
    vis = j <= p + (1 if bug == "mask_p+1" else 0)
    if bug == "mask_no_diag":
        vis = j < p
    elif bug == "skip_tile":                       # rows with >= 3 tiles lose the tile halfway along
        vis = vis & ~((j // 64 == p // 128) & (p >= 128))
    elif bug == "drop_last_tile":                  # rows with >= 2 tiles lose the tile holding their own position
        vis = vis & ~((j // 64 == p // 64) & (p >= 64))
    hd_s = (64 if hd == 128 else 128) if bug == "scale_hd" else hd
    T = (Lk + 63) // 64
    out = torch.zeros(r, nh, hd, dtype=torch.float64, device=dev)
    for h in range(nh):
        g = h % nkv if bug == "gqa_mod" else h // G
        S = q[:, h] @ K[:, g].T                    # [r, Lk]
        if mode == "exact":
            s = (S * hd_s ** -0.5).masked_fill(~vis, float("-inf"))
            P = torch.softmax(s, -1).nan_to_num(0.0)
            out[:, h] = P @ V[:, g]
            continue
        s = (S * scale_log2(hd_s)).masked_fill(~vis, float("-inf"))
        s = torch.nn.functional.pad(s, (0, T * 64 - Lk), value=float("-inf")).view(r, T, 64)
        m = torch.cummax(s.amax(-1), 1).values     # running max after each tile [r, T]
        m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
        e = torch.exp2(s - m[..., None])
        scale = torch.ones_like(m) if bug == "no_rescale" else torch.exp2(m - m[:, -1:])
        l = (e.sum(-1) * scale).sum(-1, keepdim=True)
        Pw = (_rb(e) * scale[..., None]).view(r, T * 64)[:, :Lk]
        out[:, h] = ((Pw @ V[:, g]) / l).nan_to_num(0.0)
        if scale_out is not None:
            scale_out[:, h] = ((Pw @ V[:, g].abs()) / l).nan_to_num(0.0)
    return out


def _attn_ulps(got, want, scale):
    """|got - want| in bf16 ulps of max(|want|, scale, the head's RMS / 16) (ATTN_BOUND)."""
    floor = want.pow(2).mean(-1, keepdim=True).sqrt() / 16
    _, e = torch.frexp(torch.maximum(torch.maximum(want.abs(), scale), floor).clamp_min(1e-30))
    ulp = torch.ldexp(torch.ones_like(want), (e - 8).to(torch.int32))
    return float(((got.double() - want).abs() / ulp).max())


def _bf16_check(got, want):
    """(worst |got - want| in bf16 ulps of want, fraction of elements that differ from bf16(want))."""
    return _ulps(got, want), float((got.double() != _rb(want)).double().mean())


def _row_err(got, want):
    """worst per-row rel-L2 of got [n, D] against want."""
    return float(((got - want).norm(dim=-1) / want.norm(dim=-1).clamp_min(1e-30)).max())


def ref_chain(sd, dc, x):
    """The exact-mode reference of the whole stack from position 0 without teacher forcing: bf16 GEMM operands and K / V cache, Q unrounded
    (as the oracle has it), float64 everything else.  Returns (final-norm hidden [n, H], [(k, v) [n, nkv, hd] per layer])."""
    n = x.shape[0]
    pos = torch.arange(n)
    x = x.double()
    kv = []
    for l in range(dc.num_hidden_layers):
        w = layer_weights(sd, l, x.device)
        h = _rb(_rms(x, w["ln1"], dc.rms_norm_eps))
        q, k, v = qkv_ref(w, dc, h, pos)
        k, v = _rb(k), _rb(v)
        kv.append((k, v))
        o = attention(q, k, v, pos, "exact").reshape(n, -1)
        x = x + _rb(o) @ w["wo"].T
        h2 = _rb(_rms(x, w["ln2"], dc.rms_norm_eps))
        x = x + _rb(torch.nn.functional.silu(h2 @ w["wg"].T) * (h2 @ w["wu"].T)) @ w["wd"].T
    return _rms(x, sd["%s.norm.weight" % LM].to(x.device, torch.float64), dc.rms_norm_eps), kv


# ---- CPU: the reference against the oracle, and what the bounds catch ---------------------------------------------------------------------
@pytest.mark.parametrize("preset", ["tiny", "1.5b-l2"])
def test_reference_vs_oracle(preset):
    """The exact-mode reference chained over every layer (no teacher forcing, Q unrounded as in the oracle) against
    `oracle.qwen2_forward(act_bf16=True)` with a bf16 cache, at L = 1, 65 and 200: every row's hidden state and every layer's K / V."""
    from oracle import vv_oracle as O
    cfg = config(preset)
    dc = cfg.decoder_config
    sd = lm_layer_state_dict(cfg, range(dc.num_hidden_layers))
    sd["%s.norm.weight" % LM] = torch.ones(dc.hidden_size) + 0.1 * torch.randn(dc.hidden_size, generator=torch.Generator().manual_seed(3))
    sd32 = {k: v.float() for k, v in sd.items()}
    worst = 0.0
    for L in (1, 65, 200):
        x = torch.randn(L, dc.hidden_size, generator=torch.Generator().manual_seed(L)) * 0.5
        cache = O.KVCache(dc.num_hidden_layers, kv_bf16=True)
        want = O.qwen2_forward(sd32, dc, x, cache, 0, act_bf16=True)
        got, kv = ref_chain(sd, dc, x)
        errs = dict(hidden=rel_l2(got, want))
        for l, (k, v) in enumerate(kv):
            errs["k%d" % l] = rel_l2(k, cache.k[l].transpose(0, 1))
            errs["v%d" % l] = rel_l2(v, cache.v[l].transpose(0, 1))
        report("prefill_ref_vs_oracle", preset=preset, L=L, **errs)
        worst = max(worst, max(errs.values()))
    assert worst <= ORACLE_BOUND, worst


# bug class -> the tap that checks it
BUGS = {"mask_p+1": "attn", "mask_no_diag": "attn", "no_rescale": "attn", "skip_tile": "attn", "drop_last_tile": "attn", "gqa_mod": "attn",
        "scale_hd": "attn", "rope_chunk_local": "q", "rope_pos+1": "q", "rope_pos-1": "q", "rope_interleaved": "q", "no_k_bias": "k",
        "no_v_bias": "v", "gate_up_swapped": "swiglu", "resid_bf16": "o_update", "drop_kblock": "down_update"}


def _sample_rows(n, pos0):
    """local rows at and around page edges of their absolute position, chunk edges, the middle and the end"""
    rows = {0, 1, n // 2, n - 2, n - 1}
    for e in (64, 128, 1024, 4096):
        for p in (e - 1 - pos0, e - pos0):
            rows.add(p)
    return sorted(r for r in rows if 0 <= r < n)


def test_bound_catches_bug_classes():
    """Layer 0 of every GPU case (its shapes, positions, prefix and inputs; rows subsampled at page edges, the middle and the end): how
    far each bug class moves the tap that checks it, in units of that tap's bound.  Each class must reach 3x in at least one GPU case."""
    caught = {b: [] for b in BUGS}
    worst = {b: 0.0 for b in BUGS}
    by_cfg = {}
    for c in CASES + [FRAGMENTED]:
        by_cfg.setdefault(c[0], []).append(c)
    for name, cases in by_cfg.items():
        cfg = config(name)
        dc = cfg.decoder_config
        w = layer_weights(lm_layer_state_dict(cfg, [0]), 0, "cpu")
        eps, nh, hd = dc.rms_norm_eps, dc.num_attention_heads, dc.head_dim
        for _, n, pos0, wsk in cases:
            tag = "%s-n%d-p%d-%s" % (name, n, pos0, wsk)
            R = chunk_rows(dc, n, workspace(dc, n, wsk))
            x, pre = case_inputs(dc, name, n, pos0)
            x = x.double()
            pos = torch.arange(pos0, pos0 + n)
            rows = torch.tensor(_sample_rows(n, pos0))
            h = _rb(_rms(x, w["ln1"], eps))
            _, k, v = qkv_ref(w, dc, h, pos)
            K, V = _rb(k), _rb(v)
            if pre is not None:
                K = torch.cat([pre[0][0].transpose(0, 1).double(), K])
                V = torch.cat([pre[0][1].transpose(0, 1).double(), V])
            hs, ps = h[rows], pos[rows]
            q, k_r, v_r = qkv_ref(w, dc, hs, ps)
            qb = _rb(q)
            att_scale = torch.zeros(len(rows), nh, hd, dtype=torch.float64)
            att = attention(qb, K, V, ps, "kernel", scale_out=att_scale)
            x1 = x[rows] + _rb(att).reshape(len(rows), -1) @ w["wo"].T
            upd_o = x1 - x[rows]
            h2 = _rb(_rms(x1, w["ln2"], eps))
            g, u = h2 @ w["wg"].T, h2 @ w["wu"].T
            sw = torch.nn.functional.silu(g) * u
            upd_d = _rb(sw) @ w["wd"].T
            for bug, tap in BUGS.items():
                if tap == "attn":
                    move = _attn_ulps(_rb(attention(qb, K, V, ps, "kernel", bug=bug)), att, att_scale) / ATTN_BOUND
                elif tap in ("q", "k", "v"):
                    qq, kk, vv = qkv_ref(w, dc, hs, ps, bug=bug, R=R, pos0=pos0)
                    got, want = {"q": (qq, q), "k": (kk, k_r), "v": (vv, v_r)}[tap]
                    move = _ulps(_rb(got), want) / ULP_BOUND
                elif tap == "swiglu":
                    move = _ulps(_rb(torch.nn.functional.silu(u) * g), sw) / ULP_BOUND
                elif tap == "o_update":
                    move = _row_err(_rb(x1) - x[rows], upd_o) / update_bound(nh * hd)
                else:
                    move = _row_err(_rb(sw)[:, :-64] @ w["wd"][:, :-64].T, upd_d) / update_bound(dc.intermediate_size)
                report("prefill_layer_sensitivity", case=tag, bug=bug, tap=tap, ratio=move)
                worst[bug] = max(worst[bug], move)
                if move >= 3:
                    caught[bug].append(tag)
    report("prefill_layer_sensitivity_summary", caught=caught, worst_ratio=worst)
    missed = [b for b in BUGS if not caught[b]]
    assert not missed, (missed, worst)


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------------
def _pool_tokens(name):
    return max(p + n for c, n, p, _ in CASES + [FRAGMENTED] if c == name) + 2048


@pytest.fixture(scope="module")
def engines():
    """one model at a time (the cases are grouped by config): get(name) -> (model, state dict), KV pool initialised"""
    held = {}

    def get(name):
        if name not in held:
            for m, _ in held.values():
                m.engine.close()
            held.clear()
            torch.cuda.empty_cache()
            model, sd = build_model(config(name), 2)
            model.engine.kv_init(_pool_tokens(name))
            held[name] = (model, sd)
        return held[name]
    yield get
    for m, _ in held.values():
        m.engine.close()


def _reserve(eng, seq, n_tokens):
    assert eng.lib.vv_kv_reserve(eng.h, seq, n_tokens, eng.s) == 0


def run_layers(eng, sd, dc, seq, x, pos0, wsk, tag):
    """Every layer through vv_debug_prefill_taps on the GPU's own output of the layer below, each tap checked against its float64 stage.
    Returns {figure: worst over layers}.  Pages are reserved first, so each call's launch count is its kernels alone."""
    n, nh, nkv, hd, eps = x.shape[0], dc.num_attention_heads, dc.num_key_value_heads, dc.head_dim, dc.rms_norm_eps
    ws = workspace(dc, n, wsk)
    chunks = -(-n // chunk_rows(dc, n, ws))
    pos = torch.arange(pos0, pos0 + n, device="cuda")
    _reserve(eng, seq, pos0 + n)
    cur = x.cuda()
    worst = {}
    for l in range(dc.num_hidden_layers):
        w = layer_weights(sd, l, "cuda")
        before = eng.launch_count()
        taps, hl = eng.prefill_taps(seq, l, cur, pos0=pos0, workspace_bytes=ws)
        eng.sync()
        assert eng.launch_count() - before == 7 * chunks + 1, (tag, l, eng.launch_count() - before, chunks)
        t = [tap for _, tap in taps]
        K, V = (a.double() for a in eng.kv_read(seq, l, 0, pos0 + n))
        xd = cur.double()
        f = {}
        f["norm1_ulps"], f["norm1_neq"] = _bf16_check(t[PT_NORM1], _rms(xd, w["ln1"], eps))
        q, k, v = qkv_ref(w, dc, t[PT_NORM1].double(), pos)
        f["q_ulps"], f["q_neq"] = _bf16_check(t[PT_Q].view(n, nh, hd), q)
        f["k_ulps"], f["k_neq"] = _bf16_check(K[pos0:], k)
        f["v_ulps"], f["v_neq"] = _bf16_check(V[pos0:], v)
        qg = t[PT_Q].view(n, nh, hd).double()
        ga = t[PT_ATTN].view(n, nh, hd)
        att_scale = torch.zeros(n, nh, hd, dtype=torch.float64, device="cuda")
        att = attention(qg, K, V, pos, "kernel", scale_out=att_scale)
        f["attn_ulps_of_o"], f["attn_neq"] = _bf16_check(ga, att)                # reported: ulps of |o_d| alone
        f["attn_scale_ulps"] = _attn_ulps(ga, att, att_scale)
        del att, att_scale
        f["attn_exact_rel_l2"] = _row_err(ga.double().view(n, -1), attention(qg, K, V, pos, "exact").view(n, -1))
        x1 = t[PT_RESID1].double()
        f["o_update"] = _row_err(x1 - xd, t[PT_ATTN].double() @ w["wo"].T)
        f["norm2_ulps"], f["norm2_neq"] = _bf16_check(t[PT_NORM2], _rms(x1, w["ln2"], eps))
        h2 = t[PT_NORM2].double()
        f["swiglu_ulps"], f["swiglu_neq"] = _bf16_check(t[PT_SWIGLU], torch.nn.functional.silu(h2 @ w["wg"].T) * (h2 @ w["wu"].T))
        out = t[PT_OUT].double()
        f["down_update"] = _row_err(out - x1, t[PT_SWIGLU].double() @ w["wd"].T)
        report("prefill_layer", case=tag, layer=l, chunks=chunks, **f)
        for key, val in f.items():
            worst[key] = max(worst.get(key, 0.0), val)
        del w
        cur = t[PT_OUT]
    want = _rms(cur[-1].double(), sd["%s.norm.weight" % LM].to("cuda", torch.float64), eps)
    worst["hidden_last"] = rel_l2(hl, want)
    worst["chunks"] = chunks
    return worst


def _check(worst, dc, tag):
    report("prefill_layers_summary", case=tag, **worst)
    ulps = {k: v for k, v in worst.items() if k.endswith("_ulps")}
    assert max(ulps.values()) <= ULP_BOUND, (tag, ulps)
    assert worst["attn_scale_ulps"] <= ATTN_BOUND, (tag, worst["attn_scale_ulps"])
    assert worst["o_update"] <= update_bound(dc.num_attention_heads * dc.head_dim), (tag, worst["o_update"])
    assert worst["down_update"] <= update_bound(dc.intermediate_size), (tag, worst["down_update"])
    assert worst["attn_exact_rel_l2"] <= EXACT_BOUND, (tag, worst["attn_exact_rel_l2"])
    assert worst["hidden_last"] <= FINAL_BOUND, (tag, worst["hidden_last"])


def _load_prefix(eng, seq, pre):
    for l, (k, v) in enumerate(pre):
        import_prefix(eng, seq, l, k, v)
    eng.kv_set_len(seq, pre[0][0].shape[1])


@pytest.mark.gpu
@pytest.mark.parametrize("name,n,pos0,wsk", CASES, ids=CASE_IDS)
def test_prefill_layers_vs_float64(engines, name, n, pos0, wsk):
    """Teacher-forced per-kernel parity of every layer (see the module docstring); the call reaches the chunk count the workspace rule
    gives (16 for tiny64 n = 1000, 79 for 1.5b-l2 n = 5000 at the minimum workspace)."""
    model, sd = engines(name)
    eng = model.engine
    dc = eng.config.decoder_config
    tag = "%s-n%d-p%d-%s" % (name, n, pos0, wsk)
    with torch.cuda.stream(eng.stream):
        eng.kv_set_len(0, 0)
        x, pre = case_inputs(dc, name, n, pos0)
        if pre is not None:
            _load_prefix(eng, 0, pre)
        worst = run_layers(eng, sd, dc, 0, x, pos0, wsk, tag)
    eng.sync()
    assert worst["chunks"] == -(-n // chunk_rows(dc, n, workspace(dc, n, wsk)))
    if (name, n, wsk) in (("tiny64", 1000, "min"), ("1.5b-l2", 5000, "min")):
        assert worst["chunks"] == {1000: 16, 5000: 79}[n]
    _check(worst, dc, tag)


@pytest.mark.gpu
def test_fragmented_pages(engines):
    """1.5b-l2, 300 rows at pos0 = 70 on seq 1, whose pages are interleaved with the other sequences' and then taken from the free list in
    descending order (alternate reserves, then shrinks); the reference reads the context back through kv_read."""
    name, n, pos0, wsk = FRAGMENTED
    model, sd = build_model(config(name), 2)           # a fresh pool: its free list is n-1 .. 0, as PoolMirror starts
    eng = model.engine
    dc = eng.config.decoder_config
    try:
        _fragmented(eng, sd, dc, n, pos0, wsk)
    finally:
        eng.close()


def _fragmented(eng, sd, dc, n, pos0, wsk):
    eng.kv_init(_pool_tokens(FRAGMENTED[0]))
    mirror = PoolMirror(eng.kv_pages, 4)
    with torch.cuda.stream(eng.stream):
        for t in (64, 128):
            for s in (1, 0, 2, 3):
                _reserve(eng, s, t)
                mirror.reserve(s, t)
        for t in (64, 0):
            for s in (0, 2, 3):
                eng.kv_set_len(s, t)
                mirror.set_len(s, t)
        x, pre = case_inputs(dc, FRAGMENTED[0], n, pos0)
        _load_prefix(eng, 1, pre)
        mirror.reserve(1, pos0 + n)
        worst = run_layers(eng, sd, dc, 1, x, pos0, wsk, "fragmented")
    eng.sync()
    # seq 1: its own two pages (seqs 0, 2, 3 took the ones between), then the pages they gave back, newest first
    assert mirror.pages[1] == [0, 4, 3, 2, 1, 7], mirror.pages
    assert int(eng.lib.vv_kv_pages_free(eng.h)) == len(mirror.free)
    _check(worst, dc, "fragmented")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["7b-l2", "1.5b-l2", "tiny"])
def test_layer_chain_is_production(engines, name):
    """The chain of per-layer tap calls (final norm from the last) and one vv_lm_prefill on a fresh sequence, 1000 rows at the minimum and
    the default workspace: bit-identical K / V in every layer and hidden_last.  vv_lm_prefill launches 7 kernels per layer and chunk plus
    the final norm."""
    model, sd = engines(name)
    eng = model.engine
    dc = eng.config.decoder_config
    n = 1000
    x = case_inputs(dc, name, n, 0)[0].cuda()
    with torch.cuda.stream(eng.stream):
        for wsk in ("min", "default"):
            ws = workspace(dc, n, wsk)
            chunks = -(-n // chunk_rows(dc, n, ws))
            eng.kv_set_len(0, 0)
            eng.kv_set_len(1, 0)
            _reserve(eng, 0, n)
            _reserve(eng, 1, n)
            cur = x
            for l in range(dc.num_hidden_layers):
                taps, hl = eng.prefill_taps(0, l, cur, workspace_bytes=ws)
                cur = taps[PT_OUT][1]
            before = eng.launch_count()
            h = eng.lm_prefill(1, x, workspace_bytes=ws)
            eng.sync()
            launches = eng.launch_count() - before
            report("prefill_chain_vs_production", case=name, workspace=wsk, chunks=chunks, launches=launches,
                   hidden_equal=bool(torch.equal(hl, h)))
            assert launches == 7 * dc.num_hidden_layers * chunks + 1, (launches, chunks)
            assert torch.equal(hl, h), (name, wsk, rel_l2(hl, h))
            for l in range(dc.num_hidden_layers):
                k0, v0 = eng.kv_read(0, l, 0, n)
                k1, v1 = eng.kv_read(1, l, 0, n)
                assert torch.equal(k0, k1) and torch.equal(v0, v1), (name, wsk, l)


@pytest.mark.gpu
def test_tap_call_errors():
    """Each bad call returns the code vv_lm_prefill returns for it, with nothing launched: bad seq / n / pos0 (VV_ERR_INVALID), a workspace
    one byte short (VV_ERR_INVALID), no KV pool and before finalize (VV_ERR_STATE); and a bad layer or too little tap space
    (VV_ERR_INVALID)."""
    from vibevoice_b200.engine import Engine
    cfg = config("tiny")
    dc = cfg.decoder_config
    model, _ = build_model(cfg, 1)
    eng = model.engine
    P = lambda t: C.c_void_p(t.data_ptr())
    L, H = 100, dc.hidden_size
    e = torch.randn(L, H, device="cuda")
    out = torch.empty(H, device="cuda")
    need = pf_bytes(dc, 64)
    work = torch.empty(need, dtype=torch.uint8, device="cuda")
    tap_bytes = L * (2 * 2 * H + 2 * 4 * H + 2 * 2 * dc.num_attention_heads * dc.head_dim + 2 * dc.intermediate_size)
    taps = torch.empty(tap_bytes, dtype=torch.uint8, device="cuda")

    def both(e_, seq, pos0, n, ws=need, layer=0, tb=tap_bytes, x=None):
        x = eng if x is None else x
        a = x.lib.vv_lm_prefill(x.h, seq, pos0, n, P(e_), P(out), P(work), ws, x.s)
        b = x.lib.vv_debug_prefill_taps(x.h, seq, pos0, n, layer, P(e_), P(out), P(work), ws, P(taps), tb, None, x.s)
        return a, b

    try:
        n0 = eng.launch_count()
        assert both(e, 0, 0, L) == (-3, -3)                                   # no KV pool
        assert eng.launch_count() == n0
        eng.kv_init(4 * L)
        eng.sync()
        n0 = eng.launch_count()
        assert eng.lib.vv_debug_prefill_taps(eng.h, 0, 0, L, 0, None, None, None, 0, None, 0, None, None) == 7
        for seq, pos0, n in ((-1, 0, L), (2, 0, L), (0, 0, 0), (0, -1, L), (0, dc.max_position_embeddings - 10, 11)):
            assert both(e, seq, pos0, n) == (-1, -1), (seq, pos0, n)
        assert both(e, 0, 0, L, ws=need - 1) == (-1, -1)
        tap = lambda layer=0, tb=tap_bytes: eng.lib.vv_debug_prefill_taps(eng.h, 0, 0, L, layer, P(e), P(out), P(work), need, P(taps), tb,
                                                                           None, eng.s)
        assert tap(layer=-1) == -1 and tap(layer=dc.num_hidden_layers) == -1 and tap(tb=tap_bytes - 1) == -1
        eng.sync()
        assert eng.launch_count() == n0
        bare = Engine(cfg, eng.valid_ids, 1)
        try:
            assert both(e, 0, 0, L, x=bare) == (-3, -3)                      # before vv_finalize_weights
        finally:
            bare.close()
    finally:
        eng.close()


@pytest.mark.gpu
def test_embed_gather_grid_stride(engines):
    """vv_embed_gather over 70 000 ids (more than its 65 535-block grid: the grid-stride loop runs): every row bit-exact against the bf16
    table row widened to fp32; ids -1 and vocab_size give zero rows."""
    model, sd = engines("tiny")
    eng = model.engine
    dc = eng.config.decoder_config
    V, H, n = dc.vocab_size, dc.hidden_size, 70000
    ids = torch.randint(0, V, (n,), generator=torch.Generator().manual_seed(41))
    bad = torch.tensor([0, 1, 65534, 65535, 65536, n - 1])
    ids[bad] = torch.tensor([-1, V, -1, V, -1, V])
    d = ids.to(torch.int32).cuda()
    out = torch.full((n, H), float("nan"), device="cuda")
    before = eng.launch_count()
    assert eng.lib.vv_embed_gather(eng.h, C.c_void_p(d.data_ptr()), n, C.c_void_p(out.data_ptr()), eng.s) == 0
    eng.sync()
    assert eng.launch_count() == before + 1
    table = sd["%s.embed_tokens.weight" % LM].float()
    want = torch.zeros(n, H)
    ok = (ids >= 0) & (ids < V)
    want[ok] = table[ids[ok]]
    got = out.cpu()
    report("prefill_embed_gather", n=n, equal=bool(torch.equal(got, want)))
    assert torch.equal(got, want)
