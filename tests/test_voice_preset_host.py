"""CPU tests of voice presets: `VibeVoiceProcessor.voice_prefix` against the full processor output, the validation of
`generate(voice_preset=)` and `RequestQueue.submit(voice_preset=)`, and the queue's use of the shared pages (build once, attach after,
page accounting, rebuild after a pool re-initialisation, release) on an engine stand-in that emulates the prefix ABI."""
import numpy as np
import pytest
import torch

from test_processor import StubTokenizer
from test_queue_host import RowFakeEngine


def test_voice_prefix_is_the_head_of_the_full_prompt():
    from vibevoice_b200.processor import VibeVoiceProcessor
    p = VibeVoiceProcessor(tokenizer=StubTokenizer())
    g = np.random.default_rng(1)
    voices = [g.standard_normal(3200 * k + 17 * k).astype(np.float32) * 0.1 for k in (2, 5, 1, 3)]
    for n in range(1, 5):
        script = "\n".join("Speaker %d: line %d of speaker %d." % (s, s, s) for s in range(n))
        full = p(text=script, voice_samples=voices[:n], return_tensors="pt")
        pre = p.voice_prefix(voices[:n])
        Lp = pre["input_ids"].shape[1]
        assert Lp < full["input_ids"].shape[1]
        assert torch.equal(pre["input_ids"][0], full["input_ids"][0, :Lp])
        assert torch.equal(pre["speech_input_mask"][0], full["speech_input_mask"][0, :Lp])
        assert not full["speech_input_mask"][0, Lp:].any()
        assert torch.equal(pre["speech_tensors"], full["speech_tensors"]) and torch.equal(pre["speech_masks"], full["speech_masks"])
    with pytest.raises(ValueError):
        p.voice_prefix([])


class PrefixFakeEngine(RowFakeEngine):
    """The queue's stand-in plus the prefix ABI (`kv_prefix_*`, `kv_epoch`, `prefix_pages`): a prefix keeps a copy of its source's
    first n K/V entries and attaching one copies them into the empty sequence; every call is logged."""

    kv_epoch = 0

    def kv_init(self, total_tokens):
        super().kv_init(total_tokens)
        self.kv_epoch += 1
        self.prefixes, self.prefix_pages = {}, {}
        self.log.append(("kv_init",))

    def kv_prefix_create(self, seq, n):
        assert n % 64 == 0 and 64 <= n <= self.kv_len(seq)
        kv = self.kv[seq]
        h = 1 + max(list(self.prefixes) + [getattr(self, "_last_handle", 0)])
        self._last_handle = h
        self.prefixes[h] = (n, [k[:, :n].clone() for k in kv.k], [v[:, :n].clone() for v in kv.v])
        self.prefix_pages[h] = n // 64
        self.log.append(("create", seq, n))
        return h

    def kv_prefix_attach(self, h, seq):
        assert self.kv_len(seq) == 0
        n, ks, vs = self.prefixes[h]
        kv = self.kv[seq]
        kv.k, kv.v = [k.clone() for k in ks], [v.clone() for v in vs]
        self.spec[seq] = False
        self.log.append(("attach", seq, n))

    def kv_prefix_release(self, h):
        del self.prefixes[h], self.prefix_pages[h]
        self.log.append(("release", h))

    def kv_prefix_tokens(self, h):
        return self.prefixes[h][0] if h in self.prefixes else -1


@pytest.fixture(scope="module")
def setup():
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference, VoicePreset
    from vibevoice_b200.synth import SynthTokenizer, synth_state_dict
    cfg = preset_config("tiny")
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, 1234, torch.float32)

    def make(B, native=True):
        m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=B, prefill_impl="native" if native else None)
        m.engine = PrefixFakeEngine(cfg, m._valid_ids(tok), B, weights=sd)
        m.engine.log = []
        m._scale, m._bias = float(sd["model.speech_scaling_factor"]), float(sd["model.speech_bias_factor"])
        return m

    def preset(m, Lp, seed):
        """a preset without voice frames: the host logic is the same, and it needs no acoustic encoder"""
        ids = torch.randint(0, cfg.decoder_config.vocab_size - 20, (Lp,), generator=torch.Generator().manual_seed(seed))
        return VoicePreset(m, ids, m.engine.embed_gather(ids).clone(), (None, None))
    return cfg, tok, make, preset


def _request(tok, cfg, p, n, seed):
    tail = torch.randint(0, cfg.decoder_config.vocab_size - 20, (n,), generator=torch.Generator().manual_seed(seed))
    tail[-1] = tok.speech_start_id
    return torch.cat([p.ids, tail])[None]


def _solo(m, tok, ids, p, r):
    m.set_ddpm_inference_steps(r["steps"])
    torch.manual_seed(r["seed"])
    return m.generate(input_ids=ids, tokenizer=tok, cfg_scale=r["cfg"], max_new_tokens=r["max_new"], show_progress_bar=False, voice_preset=p)


@pytest.mark.parametrize("chunk", [None, 64])
def test_queue_with_presets_matches_solo_and_shares_pages(setup, chunk):
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make, preset = setup
    m = make(2)
    P = [preset(m, 70, 1), preset(m, 130, 2)]
    reqs = []
    for i in range(6):
        p = [P[0], P[1], None][i % 3]
        ids = _request(tok, cfg, p, 4 + i, 10 + i) if p is not None else torch.tensor([[5 + i, 7, 9, tok.speech_start_id]])
        reqs.append(dict(ids=ids, p=p, cfg=[1.0, 1.3][i % 2], steps=[1, 3, 2][i % 3], max_new=[3, 5, 4][i % 3], seed=100 + i))
    q = RequestQueue(m, max_total_tokens=4096, max_prefill_tokens_per_frame=chunk)
    rids = [q.submit(dict(input_ids=r["ids"]), cfg_scale=r["cfg"], steps=r["steps"], max_new_tokens=r["max_new"], seed=r["seed"],
                     voice_preset=r["p"]) for r in reqs]
    got = dict(q.run())
    log = m.engine.log
    assert [e for e in log if e[0] == "create"] == [("create", 0, 64), ("create", 1, 128)]     # each preset built once, by its first request
    assert sorted(e[2] for e in log if e[0] == "attach") == [64, 128]                          # ... and attached by its second
    pf = [e for e in log if e[0] == "prefill"]
    assert pf[:2] == [("prefill", 0, 0, 64), ("prefill", 0, 64, 70 + 4 - 64)] if chunk is None else pf[0] == ("prefill", 0, 0, 64)
    assert all(p.resident() for p in P) and q.preset_pages() == 1 + 2 and q._pages_used == 0
    solo = make(2)
    Ps = [preset(solo, 70, 1), preset(solo, 130, 2)]
    for rid, r in zip(rids, reqs):
        want = _solo(solo, tok, r["ids"], None if r["p"] is None else Ps[P.index(r["p"])], r)
        assert torch.equal(got[rid].sequences, want.sequences), rid
        a, b = got[rid].speech_outputs[0], want.speech_outputs[0]
        assert (a is None) == (b is None) and (a is None or torch.allclose(a, b, rtol=1e-4, atol=1e-5)), rid


def test_queue_page_budget_rebuild_and_release(setup):
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make, preset = setup
    m = make(2)
    P = preset(m, 130, 3)                                  # 2 shared pages
    q = RequestQueue(m, max_total_tokens=192)             # 3 + 8 pages: 4 for the sequences' next entries, 7 for requests
    ids = _request(tok, cfg, P, 6, 1)                      # 136 + 8 + 2 tokens: 3 pages, 2 of them shared; negative 1 page
    for i in range(2):
        q.submit(dict(input_ids=ids), steps=1, max_new_tokens=8, seed=i, voice_preset=P)
    with pytest.raises(ValueError, match="max_total_tokens"):
        q.submit(dict(input_ids=_request(tok, cfg, P, 300, 2)), max_new_tokens=8, voice_preset=P)     # 2 + 6 pages
    assert [rid for rid, _ in q.run()] == [0, 1]
    # the preset's pages are charged once: 2 + 2 + 2 private pages fit in 7, so both requests ran at once (4 + 4 would not have)
    assert [e[:2] for e in m.engine.log if e[0] in ("create", "attach")] == [("create", 0), ("attach", 1)]
    assert q.preset_pages() == 2 and q._pages_used == 0
    # a new queue re-initialises the pool: the preset is built again by its first request
    q2 = RequestQueue(m, max_total_tokens=192)
    assert not P.resident() and q2.preset_pages() == 0
    q2.submit(dict(input_ids=ids), steps=1, max_new_tokens=4, seed=5, voice_preset=P)
    list(q2.run())
    assert [e[0] for e in m.engine.log if e[0] in ("kv_init", "create")][-2:] == ["kv_init", "create"] and P.resident()
    P.release()
    assert not P.resident() and m.engine.log[-1][0] == "release" and q2.preset_pages() == 0
    q2.submit(dict(input_ids=ids), steps=1, max_new_tokens=4, seed=6, voice_preset=P)
    list(q2.run())
    assert m.engine.log.count(("create", 0, 128)) >= 3 and P.resident()


def test_preset_validation(setup):
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make, preset = setup
    m, other = make(1), make(1)
    P = preset(m, 66, 4)
    ids = _request(tok, cfg, P, 5, 1)
    kw = dict(tokenizer=tok, max_new_tokens=2, show_progress_bar=False)
    with pytest.raises(ValueError, match="is_prefill"):
        m.generate(input_ids=ids, voice_preset=P, is_prefill=False, **kw)
    with pytest.raises(ValueError, match="decode"):
        m.generate(input_ids=ids, voice_preset=P, prefill_impl="decode", **kw)
    with pytest.raises(ValueError, match="this model"):
        other.generate(input_ids=ids, voice_preset=P, **kw)
    with pytest.raises(ValueError, match="presets for"):
        m.generate(input_ids=ids, voice_preset=[P, P], **kw)
    bad = ids.clone()
    bad[0, 3] += 1
    with pytest.raises(ValueError, match="prefix ids"):
        m.generate(input_ids=bad, voice_preset=P, **kw)
    with pytest.raises(ValueError, match="prefix ids"):
        m.generate(input_ids=P.ids[None], voice_preset=P, **kw)                  # nothing after the prefix
    sim = torch.zeros_like(ids, dtype=torch.bool)
    sim[0, -2] = True
    with pytest.raises(ValueError, match="speech positions past"):
        m.generate(input_ids=ids, speech_input_mask=sim, speech_tensors=torch.zeros(1, 3200), speech_masks=torch.ones(1, 1, dtype=torch.bool),
                   voice_preset=P, **kw)
    q = RequestQueue(m, max_total_tokens=1024)
    with pytest.raises(ValueError, match="prefix ids"):
        q.submit(dict(input_ids=bad), voice_preset=P)
    with pytest.raises(ValueError, match="speech positions past"):
        q.submit(dict(input_ids=ids, speech_input_mask=sim, speech_tensors=torch.zeros(1, 3200), speech_masks=torch.ones(1, 1, dtype=torch.bool)),
                 voice_preset=P)
    with pytest.raises(ValueError, match="this model"):
        RequestQueue(other, max_total_tokens=1024).submit(dict(input_ids=ids), voice_preset=P)


def test_queue_releases_idle_presets_instead_of_waiting_for_ever(setup):
    """A pool filled by resident presets: the request at the head no longer fits beside them.  The queue releases the presets no live
    or waiting request uses, and, with no row live, every one but the head's own; their requests build them again."""
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make, preset = setup
    m = make(2)
    A, Bp = preset(m, 130, 5), preset(m, 260, 6)           # 2 and 4 shared pages
    q = RequestQueue(m, max_total_tokens=192)             # 7 pages for requests
    calls = [0]
    progress = q._prefill_progress

    def guarded():                                         # a queue that can admit nothing and has no live row would spin here
        calls[0] += 1
        assert calls[0] < 500, "the queue admits nothing and serves nothing"
        return progress()
    q._prefill_progress = guarded
    q.submit(dict(input_ids=_request(tok, cfg, A, 6, 1)), steps=1, max_new_tokens=8, seed=0, voice_preset=A)
    assert len(list(q.run())) == 1 and A.resident() and q.preset_pages() == 2
    # B's request: 2 private + 4 shared pages fit in 7, but not beside A's 2: A is used by nobody and goes
    q.submit(dict(input_ids=_request(tok, cfg, Bp, 6, 2)), steps=1, max_new_tokens=8, seed=1, voice_preset=Bp)
    assert len(list(q.run())) == 1 and Bp.resident() and not A.resident() and q.preset_pages() == 4
    # a waiting request uses A: with no row live, B still goes (only the head's own preset stays), and A is built again after
    q.submit(dict(input_ids=_request(tok, cfg, A, 6, 3)), steps=1, max_new_tokens=8, seed=2, voice_preset=A)
    q.submit(dict(input_ids=_request(tok, cfg, Bp, 6, 4)), steps=1, max_new_tokens=8, seed=3, voice_preset=Bp)
    q2 = [rid for rid, _ in q.run()]
    assert q2 == [2, 3] and Bp.resident() and not A.resident() and q.preset_pages() == 4
    log = m.engine.log
    assert [e[2] for e in log if e[0] == "create"] == [128, 256, 128, 256]
    assert sum(1 for e in log if e[0] == "release") == 3
