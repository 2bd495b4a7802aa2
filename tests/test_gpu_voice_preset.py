"""`-m gpu` tests of voice presets: shared, reference-counted KV pages (`vv_kv_prefix_*`), the prefill that continues a sequence from
them, `generate(voice_preset=)` against the full prompt with the preset's voice noise, and `RequestQueue` with presets."""
import pytest
import torch

from vibevoice_b200 import _native as NV
from vibevoice_b200.configuration import preset_config
from vibevoice_b200.schedule import DPMSolverMultistepScheduler
from vibevoice_b200.synth import SynthTokenizer, synth_state_dict

pytestmark = pytest.mark.gpu

AUDIO_TOL = 1e-2          # closed loop, as test_gpu_queue.py
PARTS = ("lm", "head", "acoustic_decoder", "semantic", "connectors", "lm_head")     # all but the optional acoustic encoder


def rel_l2(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def make_model(preset, B, parts=None, **kw):
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    cfg = preset_config(preset)
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, 1234, torch.bfloat16) if parts is None else synth_state_dict(cfg, 1234, torch.bfloat16, parts=parts)
    m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=B, **kw)
    m.load_state_dict(sd, tok)
    return m, cfg, tok


def kv_all(eng, seq, pos0, n):
    return [eng.kv_read(seq, l, pos0, n) for l in range(eng.config.decoder_config.num_hidden_layers)]


def same_kv(a, b):
    return all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(a, b))


def embeds(cfg, L, seed):
    return (torch.randn(L, cfg.decoder_config.hidden_size, generator=torch.Generator().manual_seed(seed)) * 0.5).cuda()


def refused(fn):
    with pytest.raises(NV.VVError, match=r"failed \(-1\)"):
        fn()


def test_prefix_runtime():
    m, cfg, tok = make_model("tiny", 3, parts=PARTS, prefill_impl="native")
    eng = m.engine
    try:
        B, dc = eng.B, cfg.decoder_config
        eng.kv_init(4096)
        total = eng.kv_pages
        eng.lm_prefill(0, embeds(cfg, 200, 1))
        eng.kv_set_len(0, 200)
        refused(lambda: eng.kv_prefix_create(0, 100))                    # not a multiple of 64
        refused(lambda: eng.kv_prefix_create(0, 256))                    # beyond kv_len
        h = eng.kv_prefix_create(0, 192)
        assert eng.kv_prefix_tokens(h) == 192
        src = kv_all(eng, 0, 0, 192)
        free0 = eng.kv_pages_free()
        for s in (1, 2):
            eng.kv_prefix_attach(h, s)
            assert eng.kv_len(s) == 192
            assert same_kv(kv_all(eng, s, 0, 192), src)
        assert eng.kv_pages_free() == free0                              # nothing copied, no page taken
        refused(lambda: eng.kv_prefix_attach(h, 2))                      # not empty
        # every writer refuses the shared positions, of an attached sequence and of the source, and leaves the pool as it was
        kz = torch.zeros(4, dc.num_key_value_heads, dc.head_dim, dtype=torch.bfloat16, device=eng.device)
        for s in (0, 1):
            refused(lambda: eng.lm_prefill(s, embeds(cfg, 10, 2), pos0=100))
            refused(lambda: eng.prefill_taps(s, 0, embeds(cfg, 10, 2), pos0=150))
            refused(lambda: eng.kv_write(s, 0, 190, kz, kz))
            refused(lambda: eng.kv_delete(s, 5))
            refused(lambda: eng.kv_set_len(s, 100))
        eng.sync()
        assert eng.kv_pages_free() == free0 and eng.kv_len(0) == 200 and eng.kv_len(1) == 192
        for s in (0, 1, 2):
            assert same_kv(kv_all(eng, s, 0, 192), src), s
        # decode steps on sequence 1 write its own pages only
        eng.set_row_mode([0, 1, 0] + [0] * B)
        for i in range(70):                                              # crosses into a second private page
            with torch.cuda.stream(eng.stream):
                eng.embeds.copy_(torch.randn(2 * B, dc.hidden_size, generator=torch.Generator().manual_seed(i)).cuda())
            eng.lm_decode()
            eng.kv_commit([0, 1, 0] + [0] * B)
        eng.set_row_mode([1] * (2 * B))
        eng.sync()
        assert eng.kv_len(1) == 262 and eng.kv_seq_pages(1) == 5 and eng.kv_seq_pages(2) == 4     # 3 shared + own
        for s in (0, 1, 2):
            assert same_kv(kv_all(eng, s, 0, 192), src), s
        # the pool is whole again once every row is reset and the prefix released; the handle is gone
        for s in range(2 * B):
            eng.kv_set_len(s, 0)
        assert eng.kv_pages_free() == total - 3
        eng.kv_prefix_release(h)
        assert eng.kv_pages_free() == total and eng.kv_prefix_tokens(h) == -1
        refused(lambda: eng.kv_prefix_release(h))
        msg = eng.lib.vv_last_error()
        assert eng.kv_prefix_tokens(h) == -1 and eng.lib.vv_last_error() == msg     # a query leaves the last error alone
        # vv_kv_init drops every prefix
        eng.lm_prefill(0, embeds(cfg, 64, 3))
        eng.kv_set_len(0, 64)
        h2 = eng.kv_prefix_create(0, 64)
        eng.kv_init(4096)
        assert eng.kv_prefix_tokens(h2) == -1 and eng.kv_pages_free() == eng.kv_pages
    finally:
        eng.close()


@pytest.mark.parametrize("preset", ["tiny", "1.5b-l2", "7b-l2"])
def test_prefill_from_prefix_is_bit_equal(preset):
    """lm_prefill of the whole prompt against attach + prefill of the rest at pos0 = shared: last hidden state and every layer's K/V."""
    m, cfg, tok = make_model(preset, 2, parts=PARTS, prefill_impl="native")
    eng = m.engine
    try:
        eng.kv_init(8192)
        for Lp in (40, 64, 65, 200):
            L, shared = Lp + 37, Lp // 64 * 64
            e = embeds(cfg, L, Lp)
            h_one = eng.lm_prefill(0, e).cpu()
            if shared:
                eng.lm_prefill(1, e[:shared])
                eng.kv_set_len(1, shared)
                h = eng.kv_prefix_create(1, shared)
                eng.kv_set_len(1, 0)
                eng.kv_prefix_attach(h, 2)
            h_two = eng.lm_prefill(2, e[shared:], pos0=shared).cpu()
            assert torch.equal(h_one, h_two), (preset, Lp)
            assert same_kv(kv_all(eng, 0, 0, L), kv_all(eng, 2, 0, L)), (preset, Lp)
            for s in range(4):
                eng.kv_set_len(s, 0)
            if shared:
                eng.kv_prefix_release(h)
            assert eng.kv_pages_free() == eng.kv_pages
    finally:
        eng.close()


# ---- host API ---------------------------------------------------------------------------------------------------------------------------
def prefix_inputs(cfg, tok, seed, n_voices, Lp):
    """A voice prompt prefix as `VibeVoiceProcessor.voice_prefix` makes it: text ids with one run of diffusion slots per voice."""
    g = torch.Generator().manual_seed(seed)
    frames = [2 + (seed + i) % 3 for i in range(n_voices)]
    T = max(frames) * 3200
    wavs = torch.zeros(n_voices, T)
    masks = torch.zeros(n_voices, max(frames), dtype=torch.bool)
    ids = torch.randint(0, cfg.decoder_config.vocab_size - 20, (Lp,), generator=g)
    sim = torch.zeros(Lp, dtype=torch.bool)
    at = 30
    for i, f in enumerate(frames):
        wavs[i, :f * 3200] = torch.randn(f * 3200, generator=g) * 0.1
        masks[i, :f] = True
        ids[at - 1], ids[at + f] = tok.speech_start_id, tok.speech_end_id
        sim[at:at + f] = True
        at += f + 8
    ids[sim] = tok.speech_diffusion_id
    return dict(input_ids=ids[None], speech_input_mask=sim[None], speech_tensors=wavs, speech_masks=masks)


def full_request(pre, cfg, tok, n_script, seed):
    """The prefix followed by a script and <speech_start>, with the prefix's voices: what the processor gives for the whole prompt."""
    script = torch.randint(0, cfg.decoder_config.vocab_size - 20, (n_script,), generator=torch.Generator().manual_seed(seed))
    script[-1] = tok.speech_start_id
    ids = torch.cat([pre["input_ids"][0], script])[None]
    sim = torch.cat([pre["speech_input_mask"][0], torch.zeros(n_script, dtype=torch.bool)])[None]
    return dict(input_ids=ids, attention_mask=torch.ones_like(ids), speech_input_mask=sim, speech_tensors=pre["speech_tensors"],
                speech_masks=pre["speech_masks"])


def left_pad_batch(reqs, pad_id):
    L = max(r["input_ids"].shape[1] for r in reqs)
    out = {}
    for k, fill in (("input_ids", pad_id), ("attention_mask", 0), ("speech_input_mask", False)):
        out[k] = torch.cat([torch.cat([torch.full((1, L - r[k].shape[1]), fill, dtype=r[k].dtype), r[k]], dim=1) for r in reqs])
    out["speech_tensors"] = torch.cat([r["speech_tensors"] for r in reqs])
    out["speech_masks"] = torch.cat([r["speech_masks"] for r in reqs])
    return out


def use_solver(m, solver, steps):
    m.model.noise_scheduler = DPMSolverMultistepScheduler.from_config(m.engine.scheduler.config, algorithm_type=solver)
    m.set_ddpm_inference_steps(steps)


def assert_same(out, want, what):
    assert torch.equal(out.sequences, want.sequences), (what, out.sequences, want.sequences)
    assert torch.equal(out.reach_max_step_sample, want.reach_max_step_sample), what
    for a, b in zip(out.speech_outputs, want.speech_outputs):
        assert (a is None) == (b is None), what
        if a is not None:
            assert a.shape == b.shape and rel_l2(a, b) < AUDIO_TOL, (what, rel_l2(a, b))


@pytest.fixture(scope="module")
def tiny3():
    m, cfg, tok = make_model("tiny", 3, prefill_impl="native")
    yield m, cfg, tok
    m.engine.close()


@pytest.mark.parametrize("solver", ["dpmsolver++", "sde-dpmsolver++"])
@pytest.mark.parametrize("b", [1, 3])
def test_generate_with_preset_matches_full_prompt(tiny3, solver, b):
    m, cfg, tok = tiny3
    pre = prefix_inputs(cfg, tok, 3, 2, 70)
    P = m.voice_preset(pre, seed=9)
    assert P.shared == 64 and P.ids.numel() == 70
    reqs = [full_request(pre, cfg, tok, 9 + 6 * i, 50 + i) for i in range(b)]
    batch = left_pad_batch(reqs, tok.pad_id)
    n_rep = b
    noise = tuple(None if t is None else t.repeat(n_rep, *([1] * (t.dim() - 1))) for t in P.noise)
    use_solver(m, solver, 5)
    kw = dict(tokenizer=tok, cfg_scale=1.3, max_new_tokens=10, show_progress_bar=False)
    torch.manual_seed(7)
    want = m.generate(**batch, _voice_noise=noise, prefill_impl="native", **kw)
    for attempt in range(2):                           # the first call builds the shared pages, the second attaches them
        torch.manual_seed(7)
        got = m.generate(**batch, voice_preset=P, **kw)
        assert P.resident()
        assert_same(got, want, (solver, b, attempt))
    P.release()
    assert not P.resident()


def test_generate_refuses_bad_presets(tiny3):
    m, cfg, tok = tiny3
    pre = prefix_inputs(cfg, tok, 4, 1, 66)
    P = m.voice_preset(pre, seed=1)
    r = full_request(pre, cfg, tok, 8, 3)
    with pytest.raises(ValueError, match="is_prefill"):
        m.generate(**r, voice_preset=P, is_prefill=False, tokenizer=tok, max_new_tokens=2)
    with pytest.raises(ValueError, match="decode"):
        m.generate(**r, voice_preset=P, prefill_impl="decode", tokenizer=tok, max_new_tokens=2)
    bad = dict(r, input_ids=r["input_ids"].clone())
    bad["input_ids"][0, 5] += 1
    with pytest.raises(ValueError, match="prefix ids"):
        m.generate(**bad, voice_preset=P, tokenizer=tok, max_new_tokens=2)


# ---- queue ------------------------------------------------------------------------------------------------------------------------------
def queue_requests(cfg, tok, presets, pres):
    """presets / pre: two presets and their prefix inputs; requests with either preset or none (some of those with a voice of their own)."""
    from test_gpu_queue import requests as plain
    plain_reqs = plain(cfg, tok, 4, 2, seed=5)
    out = []
    for i in range(8):
        k = i % 3
        if k == 2:
            r = dict(plain_reqs[i // 3])
            r["preset"] = None
        else:
            r = dict(inputs=full_request(pres[k], cfg, tok, 6 + 5 * i, 70 + i), preset=presets[k])
        r.update(cfg_scale=[1.3, 1.0, 3.0][i % 3], steps=[5, 10, 3, 20][i % 4], solver=["dpmsolver++", "sde-dpmsolver++"][(i // 2) % 2],
                 max_new_tokens=4 + 2 * i, seed=2000 + i)
        out.append(r)
    return out


def solo_preset(m, tok, r):
    use_solver(m, r["solver"], r["steps"])
    torch.manual_seed(r["seed"])
    inp = r["inputs"] if r["preset"] is None else {k: v for k, v in r["inputs"].items() if k in ("input_ids", "attention_mask")}
    return m.generate(**inp, tokenizer=tok, cfg_scale=r["cfg_scale"], max_new_tokens=r["max_new_tokens"], show_progress_bar=False,
                      voice_preset=r["preset"])


def check_resident_pages(eng, q):
    """The pool holds exactly the shared prefixes' pages (each once) plus every sequence's private pages, and the queue's accounting
    covers both: each live row's private pages within its charge, the prefixes within preset_pages()."""
    B = eng.B
    prefixes = dict(eng.prefix_pages)
    shared = [0] * (2 * B)
    for r, row in enumerate(q._rows):
        if row is not None and row.prefix is not None:
            prefixes[row.prefix] = row.req.preset.pages          # a released prefix stays while the row holds it
            shared[r] = row.req.preset.pages
    private = [eng.kv_seq_pages(s) - shared[s] for s in range(2 * B)]
    held = eng.kv_pages - eng.kv_pages_free()
    assert held == sum(prefixes.values()) + sum(private), (held, prefixes, private)
    for r, row in enumerate(q._rows):
        if row is not None:
            assert private[r] + private[B + r] <= row.req.pages, (r, private[r], private[B + r], row.req.pages)
    assert sum(prefixes.values()) <= q.preset_pages()
    assert held <= q.preset_pages() + q._pages_used + 2 * B, (held, q.preset_pages(), q._pages_used)


@pytest.mark.parametrize("kind", ["native", "native_chunked", "torch_prefill"])
def test_queue_with_presets_matches_solo(kind):
    from vibevoice_b200.serving import RequestQueue
    kw = dict(torch_prefill=True) if kind == "torch_prefill" else dict(prefill_impl="native")
    m, cfg, tok = make_model("tiny", 2, **kw)
    eng = m.engine
    try:
        pres = [prefix_inputs(cfg, tok, 11, 2, 90), prefix_inputs(cfg, tok, 12, 3, 140)]
        presets = [m.voice_preset(p, seed=20 + i) for i, p in enumerate(pres)]
        reqs = queue_requests(cfg, tok, presets, pres)
        q = RequestQueue(m, max_total_tokens=16384, max_prefill_tokens_per_frame=64 if kind == "native_chunked" else None)
        assert not any(p.resident() for p in presets)                   # the queue's pool starts without them
        rids = [q.submit(r["inputs"], cfg_scale=r["cfg_scale"], steps=r["steps"], solver=r["solver"], max_new_tokens=r["max_new_tokens"],
                         seed=r["seed"], voice_preset=r["preset"]) for r in reqs]
        got = {}
        for rid, out in q.run():
            got[rid] = out
            check_resident_pages(eng, q)
        assert all(p.resident() for p in presets)
        assert eng.kv_pages - eng.kv_pages_free() == sum(p.pages for p in presets) == q.preset_pages()
        for i, (rid, r) in enumerate(zip(rids, reqs)):
            assert_same(got[rid], solo_preset(m, tok, r), (kind, i))
        for s in range(2 * eng.B):
            eng.kv_set_len(s, 0)
        for p in presets:
            p.release()
        assert eng.kv_pages_free() == eng.kv_pages
    finally:
        eng.close()
