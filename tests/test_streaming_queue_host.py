"""`serving.StreamingRequestQueue` on the CPU: the queue's host logic through the engine stand-in, extended here with the native engine's
per-row sampler (`sampler_per_row` / `set_row_sampler`), `eos_probs` and `tts_type_embed_rows`, all with the oracle's fp32 arithmetic one
row at a time, so a request served by the queue must give exactly what a solo `generate()` of the same request gives.

Covered: queue vs solo runs at max_slots 2 and 4 (sequences, flags, audio, streamer chunks) over requests with mixed text lengths, steps,
CFG scales and length limits, from cached prompts and from input_ids; requests ending by EOS (with the solo loop's post-EOS tail of `1`
tokens) and by their limit; slot reuse and the KV pool's release; text pushed in random pieces at random ticks; the launches of a tick;
`cancel` and the refusals."""
import random

import pytest
import torch

from oracle import vv_oracle as O
from oracle import vv_streaming as VS
from test_streaming_processor import _heads_engine_class, _prefilled
from vibevoice_b200 import serving
from vibevoice_b200 import streaming as S
from vibevoice_b200.configuration import preset_config
from vibevoice_b200.streamer import AudioStreamer
from vibevoice_b200.synth import synth_state_dict

EOS_BIAS = -0.3         # with the fixtures' weights some requests end by the classifier (some with a post-EOS tail), some by their limit


def _queue_engine_class():
    Heads = _heads_engine_class()

    class QueueFakeEngine(Heads):
        """`Heads` + per-row sampler settings, n-row EOS classifier and row-indexed type embeddings; sampler, acoustic decoder and
        connector run one row at a time (a solo run has one active row), and every launch a tick makes is logged."""

        def _setup(self, *a, **k):
            super()._setup(*a, **k)
            self.row_nmax, self.row_steps, self.row_cfg, self.log = 0, {}, {}, []

        def lm_decode_range(self, layer_begin, layer_end, final_norm, out=None):
            self.log.append(("lower" if layer_begin == 0 else "upper", tuple(getattr(self, "row_mode", []))))
            super().lm_decode_range(layer_begin, layer_end, final_norm, out)

        def sampler_per_row(self, n_max):
            self.row_nmax, self.row_steps, self.row_cfg = int(n_max), {}, {}

        def set_row_sampler(self, row, n_steps, solver, cfg_scale):
            assert self.row_nmax >= n_steps and solver == "dpmsolver++"
            self.row_steps[row], self.row_cfg[row] = int(n_steps), float(cfg_scale)

        def _rows(self):
            return self.active.nonzero().flatten().tolist()

        def diffusion_sample(self, cfg_scale):
            self.log.append(("sample", tuple(self._rows())))
            hc = self.config.diffusion_head_config
            for r in self._rows():
                steps, cfg = (self.row_steps[r], self.row_cfg[r]) if self.row_nmax else (self.n_steps, cfg_scale)
                noise = torch.cat([self.noise[r:r + 1], torch.zeros(1, 64)])
                self.latent[r:r + 1] = O.sample_speech_tokens(self.w, self.hidden[r:r + 1], self.hidden[self.B + r:self.B + r + 1], cfg, steps,
                                                              noise, hc.head_layers, hc.rms_norm_eps)

        def codec_decode(self):
            scale, bias = float(self.w["model.speech_scaling_factor"]), float(self.w["model.speech_bias_factor"])
            for r in self._rows():
                self.audio[r] = O.decoder_frame(self.w, self.config.acoustic_tokenizer_config, (self.latent[r:r + 1] / scale - bias)[:, None, :],
                                                self.a_state, torch.tensor([r]))[0, 0]

        def connect(self):
            for r in self._rows():
                self.embeds[r] = O.connector(self.w, "model.acoustic_connector", self.latent[r:r + 1])[0] + \
                    O.connector(self.w, "model.semantic_connector", self.feat[r:r + 1])[0]
            self.embeds[self.B:] = self.embeds[:self.B]

        def eos_probs(self, rows, hidden=None):
            self.log.append(("eos", tuple(rows)))
            h = self.hidden if hidden is None else hidden
            return [self.eos_prob(h[r]) for r in rows]

        def tts_type_embed_rows(self, src, src_rows, type_ids, dst_rows, dst):
            self.log.append(("type", tuple(dst_rows)))
            types = self.w["model.tts_input_types.weight"].float()
            vals = [src[s].float() + types[t] for s, t in zip(src_rows, type_ids)]
            for d, v in zip(dst_rows, vals):
                dst[d] = v

    return QueueFakeEngine


@pytest.fixture(scope="module")
def env(golden_module):
    g = golden_module("streaming")
    cfg = preset_config(g["preset"])
    sd = VS.streaming_state_dict(synth_state_dict(cfg, 1234, torch.float32), cfg, g["tts_layers"], eos_bias=EOS_BIAS)
    return g, cfg, sd


@pytest.fixture(scope="module")
def golden_module():
    import os
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    return lambda name: torch.load(os.path.join(here, name + ".pt"), weights_only=False)


def _model(env, slots):
    g, cfg, sd = env
    E = _queue_engine_class()
    m = S.VibeVoiceStreamingForConditionalGenerationInference(cfg, tts_backbone_num_hidden_layers=g["tts_layers"], max_slots=slots)
    m._new_engine = lambda: E(cfg, [0, 1], 2 * slots)
    m.load_state_dict(sd)
    return m


def _requests(env, n, seed):
    """n requests: every third from one of the fixtures' cached prompts, the others from input_ids; text lengths 0, < 5 and several
    windows; steps, CFG scales and length limits mixed."""
    g = env[0]
    rnd = random.Random(seed)
    gen = torch.Generator().manual_seed(seed)
    reqs = []
    for i in range(n):
        n_text = [0, 3, 4, 12, 17, 23, 9, 1][i % 8]
        r = dict(text=torch.randint(0, 2000, (n_text,), generator=gen), cfg_scale=rnd.choice([1.0, 1.5, 3.0]), steps=rnd.choice([2, 3, 5]),
                 max_new_tokens=rnd.randint(4, 40), seed=rnd.randint(0, 10 ** 6), streamer=i % 2 == 0)
        if i % 3 == 0:
            c = g[("eos", "windows", "short")[(i // 3) % 3]]
            r.update(kw=dict(input_ids=c["prompt"][None], tts_lm_input_ids=c["prompt"][None], neg_text_input_id=g["neg_id"]),
                     prefilled=c)
        else:
            r.update(kw=dict(input_ids=torch.randint(0, 2000, (rnd.randint(1, 7),), generator=gen)[None], neg_text_input_id=g["neg_id"]),
                     prefilled=None)
        reqs.append(r)
    return reqs


def _kw(r):
    kw = dict(r["kw"])
    if r["prefilled"] is not None:
        kw["all_prefilled_outputs"] = _prefilled(r["prefilled"])
    return kw


def _chunks(st):
    return list(st.get_stream(0)) if st is not None else None


def _solo(m, r):
    st = AudioStreamer(1) if r["streamer"] else None
    torch.manual_seed(r["seed"])
    m.set_ddpm_inference_steps(r["steps"])
    out = m.generate(tts_text_ids=r["text"][None], cfg_scale=r["cfg_scale"], max_new_tokens=r["max_new_tokens"], audio_streamer=st, **_kw(r))
    return out, _chunks(st)


def _same(out, ref):
    assert torch.equal(out.sequences, ref.sequences), (out.sequences, ref.sequences)
    assert torch.equal(out.reach_max_step_sample, ref.reach_max_step_sample)
    a, b = out.speech_outputs[0], ref.speech_outputs[0]
    assert (a is None) == (b is None)
    if a is not None:
        assert a.shape == b.shape and float((a - b).abs().max()) <= 1e-5


def _check_chunks(got, want):
    assert (got is None) == (want is None)
    if want is not None:
        assert len(got) == len(want) and all(torch.equal(x, y) for x, y in zip(got, want))


@pytest.fixture(scope="module")
def solo_refs(env):
    m = _model(env, 1)
    reqs = _requests(env, 10, 7)
    return reqs, [_solo(m, r) for r in reqs]


def _serve(m, reqs, pieces=None, seed=0):
    """Serve `reqs` on a queue; with `pieces`, each request's text arrives in random pieces of 1..7 tokens at random ticks."""
    q = serving.StreamingRequestQueue(m, max_total_tokens=4096)
    rnd = random.Random(seed)
    rids, streams, rest = [], {}, {}
    for r in reqs:
        st = AudioStreamer(1) if r["streamer"] else None
        text = r["text"].tolist()
        first = text if not pieces else text[:rnd.randint(0, 3)]
        rid = q.submit(tts_text_ids=torch.tensor(first, dtype=torch.long), text_complete=not pieces, cfg_scale=r["cfg_scale"],
                       steps=r["steps"], max_new_tokens=r["max_new_tokens"], seed=r["seed"], audio_streamer=st, **_kw(r))
        rids.append(rid)
        streams[rid] = st
        if pieces:
            rest[rid] = text[len(first):]
    outs, ticks = {}, []
    while len(outs) < len(reqs):
        for rid in list(rest):
            if rest[rid] and rnd.random() < 0.3 or not rest[rid] and rnd.random() < 0.5:
                k = rnd.randint(1, 7)
                piece, rest[rid] = rest[rid][:k], rest[rid][k:]
                q.push_text(rid, piece, complete=not rest[rid])
                if not rest[rid]:
                    del rest[rid]
        m.engine.log = []
        for rid, out in q.step():
            outs[rid] = out
        ticks.append((q.last_tick, list(m.engine.log)))
    return q, [outs[rid] for rid in rids], [_chunks(streams[rid]) for rid in rids], ticks


@pytest.mark.parametrize("slots", [2, 4])
def test_queue_matches_solo_runs(env, solo_refs, slots):
    reqs, refs = solo_refs
    m = _model(env, slots)
    q, outs, chunks, ticks = _serve(m, reqs)
    ended_by_eos = tail = 0
    for r, out, ch, (ref, ref_ch) in zip(reqs, outs, chunks, refs):
        _same(out, ref)
        _check_chunks(ch, ref_ch)
        if not bool(ref.reach_max_step_sample[0]) and ref.speech_outputs[0] is not None:
            ended_by_eos += 1
            L0 = r["kw"].get("tts_lm_input_ids", r["kw"]["input_ids"]).shape[1]
            tail += int((ref.sequences[0, L0:] == 1).sum()) > ref.speech_outputs[0].shape[-1] // 3200
    assert 0 < ended_by_eos < len(reqs)                                 # some by the classifier, some by the length limit
    assert tail > 0                                                     # frames of the solo loop's window after the EOS decision
    assert max(n_text + n_speech for (n_text, n_speech), _ in ticks) == slots         # slots were shared ...
    assert len(reqs) > slots                                                          # ... and reused
    assert q._pages_used == 0 and all(s is None for s in q._slots) and not q._reqs
    assert all(m.engine.kv_len(s) == 0 for s in range(4 * slots))


def test_queue_tick_launches(env, solo_refs):
    """Whatever the number of slots on each kind of unit, a tick makes at most one lower-stack and one upper-stack launch, one sampler
    pass, one type-embedding launch and one EOS-classifier launch."""
    reqs, _ = solo_refs
    m = _model(env, 4)
    _, _, _, ticks = _serve(m, reqs)
    mixed = 0
    for (n_text, n_speech), log in ticks:
        kinds = [k for k, _ in log]
        for k in ("lower", "upper", "sample", "type", "eos"):
            assert kinds.count(k) <= 1, log
        assert ("lower" in kinds) == (n_text > 0) and ("sample" in kinds) == (n_speech > 0)
        mixed += n_text > 0 and n_speech > 0
    assert mixed > 0


@pytest.mark.parametrize("slots", [2, 4])
def test_text_pushed_in_pieces_gives_the_same_output(env, solo_refs, slots):
    reqs, refs = solo_refs
    for seed in (1, 2):
        m = _model(env, slots)
        _, outs, chunks, _ = _serve(m, reqs, pieces=True, seed=seed)
        for out, ch, (ref, ref_ch) in zip(outs, chunks, refs):
            _same(out, ref)
            _check_chunks(ch, ref_ch)


def test_run_yields_every_request_and_refuses_to_wait_forever(env, solo_refs):
    reqs, refs = solo_refs
    m = _model(env, 2)
    q = serving.StreamingRequestQueue(m, max_total_tokens=4096)
    rids = [q.submit(tts_text_ids=r["text"], cfg_scale=r["cfg_scale"], steps=r["steps"], max_new_tokens=r["max_new_tokens"], seed=r["seed"],
                     **_kw(r)) for r in reqs[:4]]
    got = dict(q.run())
    assert sorted(got) == sorted(rids)
    for rid, (ref, _) in zip(rids, refs[:4]):
        _same(got[rid], ref)
    r = reqs[2]
    rid = q.submit(tts_text_ids=r["text"][:2], text_complete=False, max_new_tokens=r["max_new_tokens"], **_kw(r))
    with pytest.raises(RuntimeError, match="waits for text"):
        list(q.run())
    q.push_text(rid, r["text"][2:], complete=True)
    assert [k for k, _ in q.run()] == [rid]


def test_cancel(env, solo_refs):
    reqs, refs = solo_refs
    m = _model(env, 2)
    q = serving.StreamingRequestQueue(m, max_total_tokens=4096)
    st = [AudioStreamer(1) for _ in range(3)]
    rids = [q.submit(tts_text_ids=r["text"], cfg_scale=r["cfg_scale"], steps=r["steps"], max_new_tokens=r["max_new_tokens"], seed=r["seed"],
                     audio_streamer=s, **_kw(r)) for r, s in zip(reqs[3:6], st)]
    for _ in range(4):
        assert q.step() == []
    out = q.cancel(rids[0])                                             # live: what it produced so far, a prefix of the solo run
    ref = refs[3][0]
    n = out.sequences.shape[1]
    assert torch.equal(out.sequences[0], ref.sequences[0, :n]) and not bool(out.reach_max_step_sample[0])
    ch = _chunks(st[0])                                                 # its streamer has ended
    if out.speech_outputs[0] is not None:
        assert len(ch) == out.speech_outputs[0].shape[-1] // 3200
    waiting = q.cancel(rids[2])                                         # still waiting: nothing produced
    assert waiting.speech_outputs == [None] and _chunks(st[2]) == []
    with pytest.raises(KeyError):
        q.cancel(rids[0])
    rest = dict(q.run())
    assert list(rest) == [rids[1]]
    _same(rest[rids[1]], refs[4][0])
    assert q._pages_used == 0


def test_refusals(env, solo_refs):
    reqs, _ = solo_refs
    m = _model(env, 2)
    q = serving.StreamingRequestQueue(m, max_total_tokens=512)
    kw = _kw(reqs[1])
    ok = dict(tts_text_ids=reqs[1]["text"], max_new_tokens=8)
    with pytest.raises(ValueError, match="sde-dpmsolver"):
        q.submit(solver="sde-dpmsolver++", **ok, **kw)
    with pytest.raises(ValueError, match="steps"):
        q.submit(steps=0, **ok, **kw)
    with pytest.raises(ValueError, match="steps"):
        q.submit(steps=m._max_steps + 1, **ok, **kw)
    with pytest.raises(ValueError, match="stop_check_fn"):
        q.submit(stop_check_fn=lambda: False, **ok, **kw)
    with pytest.raises(ValueError, match="one request"):
        q.submit(tts_text_ids=reqs[1]["text"], max_new_tokens=8, input_ids=torch.zeros(2, 3, dtype=torch.long), neg_text_input_id=1)
    with pytest.raises(ValueError, match="batch size 1"):
        q.submit(audio_streamer=AudioStreamer(2), **ok, **kw)
    with pytest.raises(ValueError, match="KV pages"):
        q.submit(tts_text_ids=reqs[1]["text"], max_new_tokens=4000, **kw)
    rid = q.submit(**ok, **kw)
    with pytest.raises(ValueError, match="already complete"):
        q.push_text(rid, [5])
    with pytest.raises(KeyError):
        q.push_text(rid + 1, [5])
    with pytest.raises(ValueError, match="max_slots"):
        S.VibeVoiceStreamingForConditionalGenerationInference(env[1], tts_backbone_num_hidden_layers=1, max_slots=5)


def test_one_slot_model_keeps_the_row_layout(env):
    m = _model(env, 1)
    assert m.slot_rows(0) == (S.ROW_POS, S.ROW_TEXT, S.ROW_NEG) and m.engine.B == 2
    m4 = _model(env, 4)
    assert [m4.slot_rows(s) for s in range(4)] == [(0, 4, 8), (1, 5, 9), (2, 6, 10), (3, 7, 11)] and m4.engine.B == 8
