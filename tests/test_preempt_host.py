"""CPU tests of `RequestQueue` priorities on the engine stand-in, extended here with parking: which row a higher-priority request
preempts, that parked requests resume (on any row) with exactly the tokens and, within float tolerance, the audio of their solo runs,
that parked pages stay charged, `cancel` in every state a request can be in, and that all-zero priorities change nothing."""
import random

import pytest
import torch

from oracle import vv_oracle as O
from test_voice_preset_host import PrefixFakeEngine


class ParkFakeEngine(PrefixFakeEngine):
    """The preset stand-in plus the parking ABI: a parked record is the sequence's K/V cache object itself (moved, not copied), and
    a row's codec state is a copy of its rows of every streaming buffer; every call is logged."""

    def kv_init(self, total_tokens):
        super().kv_init(total_tokens)
        self.parked, self._next_park = {}, 1

    def kv_park(self, seq):
        assert self.kv_len(seq) > 0 and not self.spec[seq]
        h, self._next_park = self._next_park, self._next_park + 1
        self.parked[h] = self.kv[seq]
        self.kv[seq] = O.KVCache(self.config.decoder_config.num_hidden_layers)
        self.log.append(("park", seq))
        return h

    def kv_unpark(self, h, seq):
        assert self.kv_len(seq) == 0
        self.kv[seq] = self.parked.pop(h)
        self.spec[seq] = False
        self.log.append(("unpark", seq))

    def kv_park_release(self, h):
        del self.parked[h]
        self.log.append(("park_release", h))

    def codec_state_save(self, row):
        return [{k: b[row].clone() for k, b in st.buf.items()} for st in (self.a_state, self.s_state)]

    def codec_state_load(self, row, saved):
        for st, rows in zip((self.a_state, self.s_state), saved):
            for k, b in st.buf.items():
                b[row] = rows[k] if k in rows else 0


@pytest.fixture(scope="module")
def setup():
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference, VoicePreset
    from vibevoice_b200.synth import SynthTokenizer, synth_state_dict
    cfg = preset_config("tiny")
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, 1234, torch.float32)

    def make(B):
        m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=B, prefill_impl="native")
        m.engine = ParkFakeEngine(cfg, m._valid_ids(tok), B, weights=sd)
        m.engine.log = []
        m._scale, m._bias = float(sd["model.speech_scaling_factor"]), float(sd["model.speech_bias_factor"])
        return m

    def preset(m, Lp, seed):
        ids = torch.randint(0, cfg.decoder_config.vocab_size - 20, (Lp,), generator=torch.Generator().manual_seed(seed))
        return VoicePreset(m, ids, m.engine.embed_gather(ids).clone(), (None, None))
    return cfg, tok, make, preset


def request(cfg, tok, L, max_new, seed, priority=None, preset=None, steps=2, cfg_scale=1.3):
    ids = torch.randint(0, cfg.decoder_config.vocab_size - 20, (1, L), generator=torch.Generator().manual_seed(seed))
    ids[0, -1] = tok.speech_start_id
    if preset is not None:
        ids = torch.cat([preset.ids[None], ids], dim=1)
    r = dict(inputs=dict(input_ids=ids), cfg_scale=cfg_scale, steps=steps, max_new_tokens=max_new, seed=seed, voice_preset=preset)
    if priority is not None:
        r["priority"] = priority
    return r


def drive(q, first, arrivals=None, after_frame=None):
    """Submit `first`, then run the queue; arrivals {n: [requests]} are submitted after the n-th frame, and after_frame(n) may act
    there too (both between frames, where a caller of run() acts between yields).  Returns ({rid: output}, [rids in submit order])."""
    rids = [q.submit(**r) for r in first]
    frames, frame = [0], q._frame

    def counted():
        done = frame()
        frames[0] += 1
        for r in (arrivals or {}).get(frames[0], []):
            rids.append(q.submit(**r))
        if after_frame is not None:
            done += after_frame(frames[0], [rid for rid, _ in done])
        return done
    q._frame = counted
    got = dict(q.run())
    return got, rids


def solo(m, tok, r, presets=None):
    m.set_ddpm_inference_steps(r["steps"])
    torch.manual_seed(r["seed"])
    p = r["voice_preset"]
    p = None if p is None else presets[p]
    return m.generate(input_ids=r["inputs"]["input_ids"], tokenizer=tok, cfg_scale=r["cfg_scale"], max_new_tokens=r["max_new_tokens"],
                      show_progress_bar=False, voice_preset=p)


def assert_same(out, want, what):
    assert torch.equal(out.sequences, want.sequences), (what, out.sequences, want.sequences)
    assert torch.equal(out.reach_max_step_sample, want.reach_max_step_sample), what
    a, b = out.speech_outputs[0], want.speech_outputs[0]
    assert (a is None) == (b is None), what
    if a is not None:
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-5), (what, float((a - b).abs().max()))


def events(m, kind):
    return [e[1] for e in m.engine.log if e[0] == kind]


def rows_of(m, kind):
    """rows of the positive sequences parked / unparked, in order"""
    return [s for s in events(m, kind) if s < m.engine.B]


@pytest.mark.parametrize("case", ["newest_of_equal", "lowest_first", "equal_never", "newest_by_admission"])
def test_which_row_is_parked(setup, case):
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make, _ = setup
    m = make(2)
    q = RequestQueue(m, max_total_tokens=4096)
    long = lambda s, p: request(cfg, tok, 6, 40, s, priority=p)
    if case == "newest_of_equal":              # rows 0 and 1 at priority 0: the later admission (row 1) goes
        first, arrive, want = [long(1, 0), long(2, 0)], {3: [long(9, 1)]}, [1]
    elif case == "lowest_first":               # row 0 at 0, row 1 at 1: priority 2 takes row 0 though it was admitted first
        first, arrive, want = [long(1, 0)], {1: [long(2, 1)], 3: [long(9, 2)]}, [0]
    elif case == "equal_never":                # a request of the running rows' own priority waits
        first, arrive, want = [long(1, 1), long(2, 1)], {3: [long(9, 1)]}, []
    else:                                      # row 0 finishes first and takes a third request: the newest admission is now row 0
        first, arrive, want = [request(cfg, tok, 6, 2, 1, priority=0), long(2, 0), long(3, 0)], {6: [long(9, 1)]}, [0]
    got, rids = drive(q, first, arrive)
    assert rows_of(m, "park") == want, m.engine.log
    assert q.parks == len(want)
    assert sorted(got) == sorted(rids) and q._pages_used == 0 and not m.engine.parked
    if want:                                   # the parked request resumed after the preemptor finished
        assert len(rows_of(m, "unpark")) == 1


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_parked_requests_match_solo(setup, seed):
    """Random scripts, priorities and arrival frames over 2 rows, some requests on a voice preset: every request equals its solo run."""
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make, preset = setup
    rnd = random.Random(seed)
    m, solo_m = make(2), make(2)
    P = preset(m, 70, 5)
    solo_presets = {P: preset(solo_m, 70, 5)}
    q = RequestQueue(m, max_total_tokens=8192)
    mk = lambda i, pr: request(cfg, tok, rnd.randint(4, 14), rnd.randint(16, 40), 100 * seed + i, priority=pr,
                               preset=P if rnd.random() < 0.3 else None, steps=rnd.choice([1, 2, 3]), cfg_scale=rnd.choice([1.0, 1.3, 3.0]))
    first = [mk(i, 0) for i in range(3)]
    arrivals, i = {}, 3
    for f in sorted(rnd.sample(range(2, 16), 5)):
        arrivals[f] = [mk(i, rnd.choice([0, 1, 2, 2]))]
        i += 1
    reqs = first + [r for f in sorted(arrivals) for r in arrivals[f]]
    got, rids = drive(q, first, arrivals)
    assert sorted(got) == sorted(rids) and q._pages_used == 0 and not m.engine.parked
    assert q.parks >= 1 and len(rows_of(m, "unpark")) == q.parks
    for rid, r in zip(rids, reqs):
        assert_same(got[rid], solo(solo_m, tok, r, solo_presets), (seed, rid))


def test_a_parked_request_resumes_on_another_row(setup):
    """Row 1 is parked for a priority-1 request; row 0 finishes first, so the parked request resumes on row 0."""
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make, _ = setup
    m, solo_m = make(2), make(2)
    q = RequestQueue(m, max_total_tokens=4096)
    reqs = [request(cfg, tok, 6, 8, 1, priority=0), request(cfg, tok, 8, 30, 2, priority=0)]
    arrive = {2: [request(cfg, tok, 7, 30, 3, priority=1)]}
    got, rids = drive(q, reqs, arrive)
    assert rows_of(m, "park") == [1] and rows_of(m, "unpark") == [0], m.engine.log
    for rid, r in zip(rids, reqs + arrive[2]):
        assert_same(got[rid], solo(solo_m, tok, r), rid)


@pytest.mark.parametrize("total,parks", [(64, 0), (128, 1)])
def test_parked_pages_stay_charged(setup, total, parks):
    """Budget = pages - 2B: 5 pages at 64 tokens, 6 at 128.  Two running requests hold 2 pages each; the priority-1 head needs 2 more,
    which preemption cannot free, so it preempts only when 2 + 2 + 2 fit."""
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make, _ = setup
    m = make(2)
    q = RequestQueue(m, max_total_tokens=total)
    reqs = [request(cfg, tok, 10, 8, s, priority=0) for s in (1, 2)]
    hi = request(cfg, tok, 10, 8, 3, priority=1)
    seen = []
    got, rids = drive(q, reqs, {1: [hi]}, after_frame=lambda n, done: seen.append(q._pages_used) or [])
    assert q.parks == parks and max(seen) <= q._budget
    assert sorted(got) == sorted(rids) and q._pages_used == 0


def test_cancel_in_each_state(setup):
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make, _ = setup
    m, solo_m = make(2), make(2)
    q = RequestQueue(m, max_total_tokens=4096, max_prefill_tokens_per_frame=64)
    first = [request(cfg, tok, 8, 40, 10, priority=0), request(cfg, tok, 8, 40, 15, priority=0),
             request(cfg, tok, 6, 8, 3, priority=0)]             # rids 0 and 1 run (14 and 10 steps with audio), rid 2 waits
    hi = request(cfg, tok, 8, 40, 13, priority=1)                   # rid 3 (16 steps): parks rid 1
    adm = request(cfg, tok, 200, 8, 5, priority=5)                  # rid 4: parks rid 0; a 200-token prompt admits over frames
    out = {}

    def act(n, done):
        if n == 2:
            out["waiting"] = q.cancel(2)
            q.submit(**hi)
        elif n == 3:
            assert [w.rid for w in q._waiting if w.parked is not None] == [1]
            out["parked"] = q.cancel(1)
            q.submit(**adm)
        elif n == 4:
            assert q._rows[0].req.rid == 4 and q._rows[0].step < 0 and q._waiting[0].parked is not None
            out["admitting"] = q.cancel(4)                          # rid 0 resumes on row 0 at the next admission
        elif n == 6:
            assert q._rows[1].req.rid == 3 and q._rows[1].step >= 1
            out["running"] = q.cancel(3)
        return []
    got, rids = drive(q, first, after_frame=act)
    assert sorted(got) == [0]
    assert q._pages_used == 0 and not m.engine.parked and all(r is None for r in q._rows) and not q._waiting
    for key, r in (("waiting", first[2]), ("admitting", adm)):
        assert torch.equal(out[key].sequences, r["inputs"]["input_ids"]) and out[key].speech_outputs == [None], key
    assert len(events(m, "park_release")) >= 1                     # the cancelled parked request's pages went back
    assert_same(got[0], solo(solo_m, tok, first[0]), "resumed")
    for key, r in (("parked", first[1]), ("running", hi)):          # a cancelled request is the head of its solo run
        o, want = out[key], solo(solo_m, tok, r)
        n = o.sequences.shape[1]
        assert n > r["inputs"]["input_ids"].shape[1] and torch.equal(o.sequences, want.sequences[:, :n]), key
        a, b = o.speech_outputs[0], want.speech_outputs[0]
        if a is not None:
            assert torch.allclose(a, b[..., :a.shape[-1]], rtol=1e-4, atol=1e-5), key
    with pytest.raises(KeyError):
        q.cancel(0)


def test_zero_priorities_change_nothing(setup):
    """Every priority 0, given or not, mid-run arrivals included: the same admissions, rows, frames and results."""
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make, _ = setup
    runs = []
    for given in (False, True):
        m = make(2)
        q = RequestQueue(m, max_total_tokens=4096)
        mk = lambda i: request(cfg, tok, 5 + 3 * i, [2, 9, 4, 12, 6][i % 5], 50 + i, priority=0 if given else None)
        got, rids = drive(q, [mk(i) for i in range(3)], {2: [mk(3)], 4: [mk(4), mk(5)]})
        assert q.parks == 0
        runs.append(([got[r] for r in rids], [e for e in m.engine.log if e[0] in ("prefill", "frame")], list(got)))
    (a, la, oa), (b, lb, ob) = runs
    assert la == lb and oa == ob
    for x, y in zip(a, b):
        assert torch.equal(x.sequences, y.sequences) and torch.equal(x.reach_max_step_sample, y.reach_max_step_sample)
        assert (x.speech_outputs[0] is None) == (y.speech_outputs[0] is None)
        assert x.speech_outputs[0] is None or torch.equal(x.speech_outputs[0], y.speech_outputs[0])
