"""The LM decode step layer by layer: every decoder layer of the `lmf:` weight-stream program (QKV + RMSNorm, paged attention with the K/V
append, o-projection with the split-partial merge, gate/up, down) against a float64 reference of one Qwen2 layer, and the KV pool's page
bookkeeping bit-exact.

End to end the decoder stack is held to 2e-3 (test_gpu_parity.py, test_gpu_presets.py, test_gpu_scale.py).  Each stage of the kernel is
accurate to about 1e-5 (activations, Q and P split into bf16 hi + lo, K / V bf16 on both sides), so that bound would let a Q or P that kept
only its hi half, one bf16-only linear operand, a lost split partial or a RoPE angle off by one position through.  Here:

  * Teacher forcing: layer l runs alone (`vv_lm_decode_range(l, l + 1)`, built by the same `lm_stream_prog_full` as the production
    `lmf:0:L` program) on the GPU's own output of layer l - 1, and its float64 reference runs on that same input over the K / V the pool
    holds, the newest entry being the bf16 K / V the GPU appended.  The error of the layer's UPDATE (out - in) relative to the reference
    update is held to BOUND per active row, so the residual stream cannot hide an attention error.
  * Attention isolated: the same case on a second engine whose mlp.down_proj weights are zero; its layer update is exactly Wo . attn.
  * Append: the K / V slot at kv_len of every row and layer is within one bf16 ulp of the float64 rotated k / v.
  * Production tie: the chain of single-layer calls (final norm on the last) and one `vv_lm_decode` on the same state agree to TIE_BOUND.
  * Sensitivity (no GPU): at the GPU cases' own shapes and contexts, each bug class moves the checked update by at least 3 x BOUND in at
    least one GPU case.

Every figure is appended to reports/parity_report.jsonl.
"""
import pytest
import torch

from vibevoice_b200.configuration import preset_config
from vibevoice_b200.synth import SynthTokenizer, param_specs, synth_state_dict, synth_tensor

from test_gpu_parity import SEED, rel_l2, report
from test_gpu_scale import PARTS, _structured_kv

BOUND = 2e-5           # per-layer update, per active row (the single-linear bound of test_gpu_stream.py); H100: <= 1.2e-5 (7b-l2, B = 4)
TIE_BOUND = 5e-4       # single-layer chain vs vv_lm_decode: the split-K fp32 atomics are not reproducible run to run; H100: up to 1.1e-4.
                       # A layer run at the wrong position or with a lost partial moves the output by far more (test_bound_catches_bug_classes)
ORACLE_BOUND = 1e-6    # float64 reference vs the fp32 oracle
STEPS = 3
LM = "model.language_model"
SENTINEL = 1e4


# ---- configurations -------------------------------------------------------------------------------------------------------------------
def config(name):
    """A preset, or one of two toy geometries: "gqa8" (8 query heads on 1 kv head, head_dim 128: all 16 MMA rows of the attention tile
    carry Q hi / lo) and "gqa1" (4 / 4 heads, head_dim 64: no grouping)."""
    if name not in ("gqa8", "gqa1"):
        return preset_config(name)
    cfg = preset_config("tiny")
    dc = cfg.decoder_config
    dc.num_attention_heads, dc.num_key_value_heads, dc.head_dim = (8, 1, 128) if name == "gqa8" else (4, 4, 64)
    return cfg


# (config, B, kv_len per row [2B] at the first step): the page edges and one long row; rows 0 .. B-1 commit every step, rows B .. 2B-1
# every other step, so the long rows of tiny, streaming, 1.5b-l2 and the toys reach the last position their model allows (max_position - 1)
CASES = [
    ("tiny", 2, [4093, 1, 62, 65]),
    ("tiny64", 2, [0, 63, 128, 4094]),
    ("streaming-0.5b-l4", 2, [8189, 64, 127, 1]),
    ("1.5b-l2", 1, [65533, 62]),
    ("1.5b-l2", 4, [61440, 0, 1, 62, 63, 64, 65, 127]),
    ("1.5b-l2", 8, [65533, 61440, 0, 1, 62, 63, 64, 65, 127, 128, 0, 1, 63, 64, 65, 128]),
    ("7b-l2", 4, [30777, 0, 1, 62, 63, 64, 65, 128]),
    ("7b-l2", 8, [30777, 127, 128, 0, 1, 62, 63, 64, 65, 127, 128, 0, 1, 62, 63, 64]),
    ("gqa8", 2, [4093, 0, 63, 64]),
    ("gqa1", 2, [4093, 1, 62, 128]),
]
CASE_IDS = ["%s-B%d" % (c, b) for c, b, _ in CASES]


def case_seed(name, B):
    return sum(map(ord, name)) * 131 + B


def case_data(cfg, B, lens, seed):
    """Structured bf16 prefixes ({(row, layer): (k, v) [nkv, L, hd]}) and the step inputs [STEPS, 2B, H] of one case."""
    dc = cfg.decoder_config
    g = torch.Generator().manual_seed(seed)
    pre = {}
    for r, L in enumerate(lens):
        for l in range(dc.num_hidden_layers):
            pre[(r, l)] = _structured_kv(dc.num_key_value_heads, L, dc.head_dim, g) if L else None
    xs = torch.randn(STEPS, 2 * B, dc.hidden_size, generator=g)
    return pre, xs


def inv_freq(dc):
    """Qwen2RotaryEmbedding.inv_freq in fp32, exactly as Engine.finalize uploads it."""
    return 1.0 / (dc.rope_theta ** (torch.arange(0, dc.head_dim, 2, dtype=torch.int64).float() / dc.head_dim))


def layer_weights(sd, l, device, zero_down=False):
    p = "%s.layers.%d." % (LM, l)
    f = lambda n: sd[p + n].to(device=device, dtype=torch.float64)
    w = dict(ln1=f("input_layernorm.weight"), wq=f("self_attn.q_proj.weight"), bq=f("self_attn.q_proj.bias"),
             wk=f("self_attn.k_proj.weight"), bk=f("self_attn.k_proj.bias"), wv=f("self_attn.v_proj.weight"),
             bv=f("self_attn.v_proj.bias"), wo=f("self_attn.o_proj.weight"), ln2=f("post_attention_layernorm.weight"),
             wg=f("mlp.gate_proj.weight"), wu=f("mlp.up_proj.weight"), wd=f("mlp.down_proj.weight"))
    if zero_down:
        w["wd"] = torch.zeros_like(w["wd"])
    return w


def lm_layer_state_dict(cfg, layers):
    """The synthetic LM tensors of the given layers only (synth_tensor is seeded per name: the same values the full checkpoint has)."""
    keep = tuple("%s.layers.%d." % (LM, l) for l in layers)
    return {n: synth_tensor(n, s, k, SEED, dtype=torch.bfloat16) for n, s, k in param_specs(cfg, ("lm",)) if n.startswith(keep)}


# ---- float64 reference of one Qwen2 decoder layer ---------------------------------------------------------------------------------------
def _rb(t):
    return t.to(torch.bfloat16).to(t.dtype)


def _rms(x, w, eps):
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * w


def _rope(x, cs, sn):
    h = x.shape[-1] // 2
    x1, x2 = x[..., :h], x[..., h:]
    return torch.cat([x1 * cs - x2 * sn, x2 * cs + x1 * sn], -1)


BUGS = ("q_hi", "p_hi", "x_qkv", "x_o", "x_gu", "x_down", "pos+1", "pos-1", "no_newest", "stale_slot", "drop_page")


def layer_ref(w, dc, x, kv, pos, inv, new=None, bug=None):
    """One Qwen2 decoder layer for R decode rows in float64.

    x [R, H] residual input; kv[r] = (K, V) [nkv, pos[r], hd] the row's cached entries; pos[r] its position (kv_len); inv the fp32
    inv_freq.  new[r] = (k, v) [nkv, hd]: the newest entry (what the GPU appended); None: this reference's own k / v rounded to bf16.
    RoPE angle = fp32(pos) * inv_freq in fp32 (HF), cos / sin of it in float64.  bug: one of BUGS (the sensitivity check).
    Returns (out [R, H], k_rot [R, nkv, hd], v [R, nkv, hd])."""
    R, dev = x.shape[0], x.device
    nh, nkv, hd, eps = dc.num_attention_heads, dc.num_key_value_heads, dc.head_dim, dc.rms_norm_eps
    G = nh // nkv
    op = lambda name, t: _rb(t) if bug == name else t
    h = op("x_qkv", _rms(x, w["ln1"], eps))
    q = (h @ w["wq"].T + w["bq"]).view(R, nh, hd)
    k = (h @ w["wk"].T + w["bk"]).view(R, nkv, hd)
    v = (h @ w["wv"].T + w["bv"]).view(R, nkv, hd)
    o = torch.empty(R, nh * hd, dtype=torch.float64, device=dev)
    k_rot = torch.empty_like(k)
    for r in range(R):
        p = pos[r] + (1 if bug == "pos+1" else -1 if bug == "pos-1" else 0)
        ang = (torch.tensor(float(p), dtype=torch.float32) * inv).to(dev, torch.float64)
        cs, sn = torch.cat([ang.cos(), ang.cos()]), torch.cat([ang.sin(), ang.sin()])
        qr, kr = _rope(q[r], cs[:hd // 2], sn[:hd // 2]), _rope(k[r], cs[:hd // 2], sn[:hd // 2])
        k_rot[r] = kr
        kn, vn = new[r] if new is not None else (_rb(kr), _rb(v[r]))
        K, V = kv[r]
        parts_k, parts_v = [K, kn[:, None]], [V, vn[:, None]]
        if bug == "no_newest":
            parts_k, parts_v = [K], [V]
        elif bug == "stale_slot":
            s = SENTINEL * (1 - 2 * (torch.arange(hd, device=dev) % 2)).double()
            parts_k.append(s.expand(nkv, 1, hd)); parts_v.append(s.expand(nkv, 1, hd))
        Kf, Vf = torch.cat(parts_k, 1), torch.cat(parts_v, 1)
        if bug == "drop_page" and pos[r] >= 640:
            pg = pos[r] // 64 // 2
            keep = torch.ones(Kf.shape[1], dtype=torch.bool, device=dev)
            keep[pg * 64:(pg + 1) * 64] = False
            Kf, Vf = Kf[:, keep], Vf[:, keep]
        if Kf.shape[1] == 0:                                      # "no_newest" on an empty context: nothing to attend to
            o[r] = 0
            continue
        qs = qr.view(nkv, G, hd) * hd ** -0.5
        if bug == "q_hi":
            qs = _rb(qs)
        s = qs @ Kf.transpose(1, 2)                               # [nkv, G, n]
        e = torch.exp(s - s.amax(-1, keepdim=True))
        den = e.sum(-1, keepdim=True)
        if bug == "p_hi":
            e = _rb(e)
        o[r] = ((e @ Vf) / den).reshape(nh * hd)
    x1 = x + op("x_o", o) @ w["wo"].T
    h2 = op("x_gu", _rms(x1, w["ln2"], eps))
    gu = torch.nn.functional.silu(h2 @ w["wg"].T) * (h2 @ w["wu"].T)
    return x1 + op("x_down", gu) @ w["wd"].T, k_rot, v


def _update_err(out, x, ref):
    return rel_l2(out - x, ref - x)


def _ulps(got_bf16, want):
    """|got - want| in units of the bf16 ulp of want [nkv, hd] (float64).  Elements below 1/16 of their head's RMS are measured in the ulp
    of that floor: k and v come out of a linear accurate to ~1e-6 of the vector's norm, which cannot place a near-zero element within
    its own ulp (2^-8 of itself) -- above the floor an ulp is >= 2.4e-4 of the RMS."""
    floor = want.pow(2).mean(-1, keepdim=True).sqrt() / 16
    _, e = torch.frexp(torch.maximum(want.abs(), floor).clamp_min(1e-30))
    ulp = torch.ldexp(torch.ones_like(want), (e - 8).to(torch.int32))
    return float(((got_bf16.double() - want).abs() / ulp).max())


# ---- CPU: the reference against the oracle, and what the bound catches ----------------------------------------------------------------
@pytest.mark.parametrize("preset", ["tiny", "1.5b-l2"])
def test_layer_reference_vs_oracle(preset):
    """`layer_ref` against `oracle.qwen2_forward` (fp32, bf16 cache) on one layer at a time: contexts 0, 63 and 200."""
    from oracle import vv_oracle as O
    cfg = config(preset)
    dc = cfg.decoder_config
    sd = lm_layer_state_dict(cfg, range(dc.num_hidden_layers))
    inv = inv_freq(dc)
    g = torch.Generator().manual_seed(5)
    worst = 0.0
    for l in range(dc.num_hidden_layers):
        w = layer_weights(sd, l, "cpu")
        for pos in (0, 63, 200):
            k, v = _structured_kv(dc.num_key_value_heads, pos, dc.head_dim, g)
            x = torch.randn(dc.hidden_size, generator=g)
            cache = O.KVCache(dc.num_hidden_layers, kv_bf16=True)
            if pos:
                cache.preload(l, k.float(), v.float())
            want = O.qwen2_forward(sd, dc, x[None], cache, pos, n_layers=1, final_norm=False, layer_begin=l)[0]
            new = [(cache.k[l][:, pos].double(), cache.v[l][:, pos].double())]
            got, _, _ = layer_ref(w, dc, x[None].double(), [(k.double(), v.double())], [pos], inv, new=new)
            e = rel_l2(got[0], want)
            report("lm_layer_ref_vs_oracle", preset=preset, layer=l, pos=pos, rel_l2=e, update_rel_l2=_update_err(got[0], x.double(), want.double()))
            worst = max(worst, e)
    assert worst <= ORACLE_BOUND, worst


def test_bound_catches_bug_classes():
    """At every GPU case's shapes, contexts and step-0 inputs (layer 0, full and zero-MLP weights), how far each bug class moves the
    per-row layer update.  Every class must move it by >= 3 x BOUND in at least one GPU case; the catching cases are reported."""
    caught = {b: [] for b in BUGS}
    worst = {b: 0.0 for b in BUGS}
    for name, B, lens in CASES:
        cfg = config(name)
        dc = cfg.decoder_config
        sd = lm_layer_state_dict(cfg, [0])
        inv = inv_freq(dc)
        pre, xs = case_data(cfg, B, lens, case_seed(name, B))
        kv = []
        for r, L in enumerate(lens):
            e = torch.zeros(dc.num_key_value_heads, 0, dc.head_dim, dtype=torch.float64)
            kv.append((pre[(r, 0)][0].double(), pre[(r, 0)][1].double()) if L else (e, e))
        x = xs[0].double()
        w_full = layer_weights(sd, 0, "cpu")
        for zero in (False, True):
            w = dict(w_full, wd=torch.zeros_like(w_full["wd"])) if zero else w_full
            base, _, _ = layer_ref(w, dc, x, kv, lens, inv)
            for bug in BUGS:
                out, _, _ = layer_ref(w, dc, x, kv, lens, inv, bug=bug)
                move = max(_update_err(out[r], x[r], base[r]) for r in range(len(lens)))
                tag = "%s-B%d%s" % (name, B, "-attn" if zero else "")
                report("lm_layer_sensitivity", case=tag, bug=bug, move=move, ratio=move / BOUND)
                worst[bug] = max(worst[bug], move)
                if move >= 3 * BOUND:
                    caught[bug].append(tag)
    report("lm_layer_sensitivity_summary", caught=caught, worst_ratio={b: worst[b] / BOUND for b in BUGS})
    missed = [b for b in BUGS if not caught[b]]
    assert not missed, (missed, worst)


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------------
def build_model(cfg, B, zero_down=False):
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, SEED, torch.bfloat16, parts=PARTS)
    if zero_down:
        for l in range(cfg.decoder_config.num_hidden_layers):
            sd["%s.layers.%d.mlp.down_proj.weight" % (LM, l)].zero_()
    m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=B)
    m.load_state_dict(sd, tok)
    return m, sd


def import_prefix(eng, seq, layer, k, v):
    """k, v [nkv, L, hd] bf16 -> positions [0, L) of (seq, layer) through vv_kv_write."""
    with torch.cuda.stream(eng.stream):
        eng.kv_write(seq, layer, 0, k.transpose(0, 1).contiguous().cuda(), v.transpose(0, 1).contiguous().cuda())
    eng.sync()


def load_case(eng, dc, pre, lens):
    for r, L in enumerate(lens):
        eng.kv_set_len(r, 0)
    for r, L in enumerate(lens):
        for l in range(dc.num_hidden_layers):
            if L:
                import_prefix(eng, r, l, *pre[(r, l)])
        eng.kv_set_len(r, L)
    assert [eng.kv_len(r) for r in range(len(lens))] == list(lens)


def run_layers(eng, W, dc, x, rows, **report_kw):
    """One decode step as a chain of single-layer calls on input x [2B, H] (device), each layer checked against `layer_ref` on its GPU
    input, for the rows in `rows`.  K / V are appended speculatively at kv_len; the caller commits.  Returns (output [2B, H], worst update
    error, worst append error in ulps)."""
    with torch.cuda.stream(eng.stream):     # one stream for the engine and the reference: no buffer is reused while another stream reads it
        return _run_layers(eng, W, dc, x, rows, **report_kw)


def _run_layers(eng, W, dc, x, rows, **report_kw):
    inv = inv_freq(dc)
    lens = [eng.kv_len(r) for r in range(2 * eng.B)]
    cur, worst, ulps = x.clone(), 0.0, 0.0
    for l in range(dc.num_hidden_layers):
        eng.embeds.copy_(cur)
        eng.lm_decode_range(l, l + 1, False)
        eng.sync()
        y = eng.hidden.clone()
        assert torch.isfinite(y[rows]).all(), l
        kv, new = [], []
        for r in rows:
            K, V = eng.kv_read(r, l, 0, lens[r] + 1)
            K, V = K.transpose(0, 1).double(), V.transpose(0, 1).double()
            kv.append((K[:, :lens[r]], V[:, :lens[r]]))
            new.append((K[:, lens[r]], V[:, lens[r]]))
        ref, k_rot, v = layer_ref(W[l], dc, cur[rows].double(), kv, [lens[r] for r in rows], inv, new=new)
        for i, r in enumerate(rows):
            e = _update_err(y[r].double(), cur[r].double(), ref[i])
            u = max(_ulps(new[i][0], k_rot[i]), _ulps(new[i][1], v[i]))
            report("lm_layer", layer=l, row=r, kv_len=lens[r], update_rel_l2=e, append_ulps=u, **report_kw)
            worst, ulps = max(worst, e), max(ulps, u)
        cur = y
    return cur, worst, ulps


def run_case(cfg, B, lens, zero_down, tag):
    dc = cfg.decoder_config
    model, sd = build_model(cfg, B, zero_down)
    eng = model.engine
    try:
        W = [layer_weights(sd, l, "cuda", zero_down) for l in range(dc.num_hidden_layers)]
        pre, xs = case_data(cfg, B, lens, case_seed(tag, B))
        eng.kv_init(sum(lens) + 64 * (2 * B + 8) + 256)
        load_case(eng, dc, pre, lens)
        rows = list(range(2 * B))
        worst, ulps, tie = 0.0, 0.0, 0.0
        for step in range(STEPS):
            x = xs[step].cuda()
            _, e, u = run_layers(eng, W, dc, x, rows, case=tag, B=B, zero_down=zero_down, step=step)
            worst, ulps = max(worst, e), max(ulps, u)
            if step == 0:
                # the production tie: chain with the final norm on the last call vs one vv_lm_decode, same kv_len
                with torch.cuda.stream(eng.stream):
                    cur = x.clone()
                    for l in range(dc.num_hidden_layers):
                        eng.embeds.copy_(cur)
                        eng.lm_decode_range(l, l + 1, l == dc.num_hidden_layers - 1)
                        cur = eng.hidden.clone()
                    eng.embeds.copy_(x)
                    eng.lm_decode()
                    prod = eng.hidden.clone()
                eng.sync()
                tie = max(rel_l2(cur[r], prod[r]) for r in rows)
            eng.kv_commit([1] * B + [step % 2] * B)
        assert [eng.kv_len(r) for r in rows] == [L + STEPS for L in lens[:B]] + [L + (STEPS // 2) for L in lens[B:]]
        return worst, ulps, tie
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,lens", CASES, ids=CASE_IDS)
def test_lm_layers_vs_float64(name, B, lens):
    """Teacher-forced per-layer parity, 3 steps (negative rows commit every other step), full and attention-isolated weights; the K / V
    append within one bf16 ulp; the single-layer chain tied to vv_lm_decode."""
    cfg = config(name)
    full, ulps, tie = run_case(cfg, B, lens, False, name)
    attn, ulps2, tie2 = run_case(cfg, B, lens, True, name)
    report("lm_layers_summary", case=name, B=B, update_rel_l2=full, attn_update_rel_l2=attn, append_ulps=max(ulps, ulps2),
           chain_vs_decode=max(tie, tie2))
    assert full <= BOUND and attn <= BOUND, (full, attn)
    assert max(ulps, ulps2) <= 1.0, (ulps, ulps2)
    assert max(tie, tie2) <= TIE_BOUND, (tie, tie2)


# ---- GPU: page bookkeeping ---------------------------------------------------------------------------------------------------------------
class PoolMirror:
    """The pool's free-list policy: initialised n-1 .. 0, pages popped from the back, released pages pushed back."""

    def __init__(self, n, seqs):
        self.free = list(range(n - 1, -1, -1))
        self.pages = [[] for _ in range(seqs)]

    def reserve(self, s, n_tokens):
        while len(self.pages[s]) < (n_tokens + 63) // 64:
            self.pages[s].append(self.free.pop())

    def set_len(self, s, n):
        while len(self.pages[s]) > (n + 63) // 64:
            self.free.append(self.pages[s].pop())


@pytest.fixture(scope="module")
def tiny_pool():
    cfg = config("tiny")
    model, sd = build_model(cfg, 2)
    W = [layer_weights(sd, l, "cuda") for l in range(cfg.decoder_config.num_hidden_layers)]
    yield model.engine, W, cfg.decoder_config
    model.engine.close()


def _pages_free(eng):
    return int(eng.lib.vv_kv_pages_free(eng.h))


def _step(eng, W, dc, x, rows, adv, **kw):
    out, e, u = run_layers(eng, W, dc, x, rows, **kw)
    eng.kv_commit(adv)
    assert e <= BOUND and u <= 1.0, (kw, e, u)
    return out


@pytest.mark.gpu
def test_fragmented_pages_and_delete_slot(tiny_pool):
    """Sequences grown alternately through vv_kv_reserve and shrunk with vv_kv_set_len get interleaved, descending and recycled pages;
    per-layer parity holds on them.  Then vv_kv_delete_slot on a middle slot and on a page-edge slot: the last entry moves into the
    deleted slot in every layer, every other slot is unchanged, pages past the next speculative entry return to the free list, and the
    next decode step matches the float64 layer over the post-delete pool."""
    eng, W, dc = tiny_pool
    eng.kv_init(64 * 40)
    n = eng.kv_pages
    mirror = PoolMirror(n, 4)
    reserve = lambda s, t: (eng.lib.vv_kv_reserve(eng.h, s, t, eng.s), mirror.reserve(s, t))
    set_len = lambda s, t: (eng.kv_set_len(s, t), mirror.set_len(s, t))
    for t in (64, 128, 192, 256, 320):
        for s in (0, 1, 2):
            reserve(s, t)
    set_len(1, 0)             # seq 1's five pages go back, newest on top
    set_len(2, 100)           # seq 2 keeps two
    for t in (64, 128, 192, 256, 320, 384, 448):
        reserve(0 if t % 128 else 3, t)
    eng.sync()
    assert _pages_free(eng) == len(mirror.free)
    g = torch.Generator().manual_seed(17)
    lens = {0: 420, 3: 330, 2: 65, 1: 0}
    for s, L in lens.items():
        for l in range(dc.num_hidden_layers):
            if L:
                import_prefix(eng, s, l, *_structured_kv(dc.num_key_value_heads, L, dc.head_dim, g))
        set_len(s, L)
    eng.sync()
    assert _pages_free(eng) == len(mirror.free)
    # seq 0: interleaved with seqs 1 / 2, then pages seq 1 gave back (descending); seq 3: only recycled pages, descending across a wrap
    assert mirror.pages[0] == [0, 3, 6, 9, 12, 10, 13] and mirror.pages[3] == [8, 11, 14, 1, 4, 7], mirror.pages
    for step in range(2):
        x = torch.randn(4, dc.hidden_size, generator=g).cuda()
        for s in range(4):
            mirror.reserve(s, eng.kv_len(s) + 1)
        _step(eng, W, dc, x, [0, 1, 2, 3], [1, 1, 1, 1], case="fragmented", step=step)
        assert _pages_free(eng) == len(mirror.free)
    for s, pos in ((0, 150), (3, 191)):
        L = eng.kv_len(s)
        reserve(s, L + 130)                  # two pages past the next speculative entry: the delete must give them back
        eng.sync()
        before = [eng.kv_read(s, l, 0, L) for l in range(dc.num_hidden_layers)]
        eng.kv_delete(s, pos)
        mirror.set_len(s, L)                 # keeps the page of the next speculative entry (position L - 1)
        eng.sync()
        assert eng.kv_len(s) == L - 1 and _pages_free(eng) == len(mirror.free), (s, _pages_free(eng), len(mirror.free))
        for l in range(dc.num_hidden_layers):
            k, v = eng.kv_read(s, l, 0, L - 1)
            k0, v0 = before[l]
            wk, wv = k0[:L - 1].clone(), v0[:L - 1].clone()
            wk[pos], wv[pos] = k0[L - 1], v0[L - 1]
            assert torch.equal(k, wk) and torch.equal(v, wv), (s, l)
    x = torch.randn(4, dc.hidden_size, generator=g).cuda()
    _step(eng, W, dc, x, [0, 1, 2, 3], [1, 1, 1, 1], case="after_delete")


@pytest.mark.gpu
def test_rejected_step_sees_only_its_own_entry(tiny_pool):
    """A step with advance = 0, then a different input at the same kv_len: the second step's attention sees its own appended entry only
    (the reference is built from the second step's append), and the slot holds the second step's K / V."""
    eng, W, dc = tiny_pool
    eng.kv_init(64 * 16)
    g = torch.Generator().manual_seed(23)
    lens = [70, 64, 1, 127]
    for s, L in enumerate(lens):
        for l in range(dc.num_hidden_layers):
            import_prefix(eng, s, l, *_structured_kv(dc.num_key_value_heads, L, dc.head_dim, g))
        eng.kv_set_len(s, L)
    x1, x2 = (torch.randn(4, dc.hidden_size, generator=g).cuda() for _ in range(2))
    _step(eng, W, dc, x1, [0, 1, 2, 3], [0, 0, 0, 0], case="rejected_first")
    first = [eng.kv_read(s, 0, lens[s], 1) for s in range(4)]
    assert [eng.kv_len(s) for s in range(4)] == lens
    _step(eng, W, dc, x2, [0, 1, 2, 3], [1, 1, 1, 1], case="rejected_second")
    for s in range(4):
        k, _ = eng.kv_read(s, 0, lens[s], 1)
        assert not torch.equal(k, first[s][0]), s


@pytest.mark.gpu
@pytest.mark.parametrize("nan", [False, True], ids=["finite", "nan"])
def test_stale_slots_past_the_length(tiny_pool, nan):
    """Slots (kv_len, page end) of the newest page hold a previous write: ±1e4 in K and V (finite), or NaN in V and K.  Rows whose
    newest page stays with the sequence (kv_len % 64 != 0) see the finite sentinels masked; for the NaN case the page is released with
    vv_kv_set_len and handed out again by the next step, as a recycled page is: it must arrive zeroed and the outputs stay finite."""
    eng, W, dc = tiny_pool
    eng.kv_init(64 * 16)
    g = torch.Generator().manual_seed(29)
    lens = [0, 64, 128, 192] if nan else [1, 62, 65, 100]
    nkv, hd = dc.num_key_value_heads, dc.head_dim
    for s, L in enumerate(lens):
        for l in range(dc.num_hidden_layers):
            if L:
                import_prefix(eng, s, l, *_structured_kv(nkv, L, hd, g))
        eng.kv_set_len(s, L)
    for s, L in enumerate(lens):
        end = (L // 64 + 1) * 64
        n = end - (L + 1)
        sgn = (1 - 2 * (torch.arange(hd) % 2)).float()
        fill = torch.full((n, nkv, hd), float("nan")) if nan else (SENTINEL * sgn).expand(n, nkv, hd)
        for l in range(dc.num_hidden_layers):
            with torch.cuda.stream(eng.stream):
                eng.kv_write(s, l, L + 1, fill.to(torch.bfloat16).contiguous().cuda(), fill.to(torch.bfloat16).contiguous().cuda())
        eng.sync()
        if not nan:
            k, _ = eng.kv_read(s, 0, L + 1, n)
            assert torch.equal(k.float().cpu(), fill.to(torch.bfloat16).float())
        eng.kv_set_len(s, L)              # nan: L % 64 == 0 -> the sentinel page goes back to the free list
    x = torch.randn(4, dc.hidden_size, generator=g).cuda()
    _step(eng, W, dc, x, [0, 1, 2, 3], [0, 0, 0, 0], case="stale_nan" if nan else "stale_finite")
    if nan:
        for s, L in enumerate(lens):
            k, v = eng.kv_read(s, 0, L + 1, 63)
            assert torch.count_nonzero(k) == 0 and torch.count_nonzero(v) == 0, s


@pytest.mark.gpu
def test_row_mode_off_rows_leave_the_pool_alone():
    """row_mode 0 on the streaming preset: a switched-off row writes no slot in any layer (the pool bytes at its kv_len are unchanged),
    and the other rows' results are the same as with every row on."""
    cfg = config("streaming-0.5b-l4")
    dc = cfg.decoder_config
    model, sd = build_model(cfg, 2)
    eng = model.engine
    try:
        W = [layer_weights(sd, l, "cuda") for l in range(dc.num_hidden_layers)]
        eng.kv_init(64 * 32)
        g = torch.Generator().manual_seed(31)
        lens = [100, 63, 64, 5]
        for s, L in enumerate(lens):
            for l in range(dc.num_hidden_layers):
                import_prefix(eng, s, l, *_structured_kv(dc.num_key_value_heads, L, dc.head_dim, g))
            eng.kv_set_len(s, L)
            for l in range(dc.num_hidden_layers):
                with torch.cuda.stream(eng.stream):
                    marker = torch.full((1, dc.num_key_value_heads, dc.head_dim), 3.0 + l, dtype=torch.bfloat16, device="cuda")
                    eng.kv_write(s, l, L, marker, marker)
        eng.sync()
        x = torch.randn(4, dc.hidden_size, generator=g).cuda()
        on = run_layers(eng, W, dc, x, [0, 1, 2, 3], case="row_mode_all")[0]
        for s, L in enumerate(lens):       # put the markers back
            for l in range(dc.num_hidden_layers):
                marker = torch.full((1, dc.num_key_value_heads, dc.head_dim), 3.0 + l, dtype=torch.bfloat16, device="cuda")
                with torch.cuda.stream(eng.stream):
                    eng.kv_write(s, l, L, marker, marker)
        eng.set_row_mode([1, 0, 1, 0])
        try:
            out, e, u = run_layers(eng, W, dc, x, [0, 2], case="row_mode_off")
        finally:
            eng.set_row_mode([1, 1, 1, 1])
        assert e <= BOUND and u <= 1.0, (e, u)
        for s in (1, 3):
            for l in range(dc.num_hidden_layers):
                k, v = eng.kv_read(s, l, lens[s], 1)
                assert (k.float() == 3.0 + l).all() and (v.float() == 3.0 + l).all(), (s, l)
        for r in (0, 2):
            d = rel_l2(out[r], on[r])
            report("lm_row_mode_other_rows", row=r, rel_l2=d)
            assert d <= TIE_BOUND, (r, d)
    finally:
        eng.close()
