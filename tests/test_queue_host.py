"""CPU tests of `vibevoice_b200.serving.RequestQueue`'s host logic on the engine stand-in (tests/fake_engine.py), extended here with the
per-row sampler and the whole-prompt prefill: admission order and row reuse, per-request results equal to solo `generate()` runs of the
stand-in, and the refusal of every option the queue does not serve."""
import pytest
import torch

from fake_engine import FakeEngine
from oracle import vv_oracle as O


class RowFakeEngine(FakeEngine):
    """The stand-in plus what the queue needs: per-row sampler settings (each active row sampled with its own steps / solver / CFG scale)
    and the whole-prompt prefill of one sequence (`lm_prefill`, `embed_gather`)."""

    row_nmax = 0

    def sampler_per_row(self, n_max: int):
        self.row_nmax = int(n_max)
        self.row_set = {r: (max(self.row_nmax, 1), "dpmsolver++", 1.0) for r in range(self.B)}
        self.row_noise = {}
        self.log.append(("per_row", self.row_nmax))

    def set_row_sampler(self, row, n_steps, solver, cfg_scale):
        assert self.row_nmax >= n_steps >= 1
        self.row_set[row] = (int(n_steps), solver, float(cfg_scale))

    def upload_row_step_noise(self, row, noise):
        self.row_noise[row] = noise.float().clone()

    def embed_gather(self, ids):
        return self.embed_w[torch.as_tensor(ids).long().reshape(-1)]

    def lm_prefill(self, seq, embeds, pos0=0, workspace_bytes=None):
        self.log.append(("prefill", seq, int(pos0), int(embeds.shape[0])))
        kv = self.kv[seq]
        kv.truncate(pos0)
        self.spec[seq] = False
        return O.qwen2_forward(self.w, self.config.decoder_config, embeds.float(), kv, pos0)[-1]

    def kv_pages_free(self):
        return self.kv_pages

    def frame_tail(self, cfg_scale):
        if not self.row_nmax:
            return super().frame_tail(cfg_scale)
        cfg, w, B = self.config, self.w, self.B
        hc = cfg.diffusion_head_config
        rows = self.active.nonzero().flatten()
        self.log.append(("frame", rows.tolist()))
        lat = []
        for r in rows.tolist():
            n, solver, cs = self.row_set[r]
            kw = dict(algorithm_type=solver, step_noise=[self.row_noise[r][i:i + 1] for i in range(n)]) if solver != "dpmsolver++" else {}
            noise = torch.cat([self.noise[r:r + 1], torch.zeros(1, 64)])
            lat.append(O.sample_speech_tokens(w, self.hidden[r:r + 1], self.hidden[B + r:B + r + 1], cs, n, noise, hc.head_layers,
                                              hc.rms_norm_eps, **kw))
        lat = torch.cat(lat)
        scale, bias = float(w["model.speech_scaling_factor"]), float(w["model.speech_bias_factor"])
        audio = O.decoder_frame(w, cfg.acoustic_tokenizer_config, (lat / scale - bias)[:, None, :], self.a_state, rows)
        sem = O.encoder_frame(w, cfg.semantic_tokenizer_config, audio, self.s_state, rows)
        emb = O.connector(w, "model.acoustic_connector", lat) + O.connector(w, "model.semantic_connector", sem[:, 0])
        self.latent[rows] = lat
        self.audio[rows] = audio[:, 0]
        self.embeds[rows] = emb
        self.embeds[B:] = self.embeds[:B]


@pytest.fixture(scope="module")
def setup():
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    from vibevoice_b200.synth import SynthTokenizer, synth_state_dict
    cfg = preset_config("tiny")
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, 1234, torch.float32)

    def make(B):
        m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=B, prefill_impl="native")
        m.engine = RowFakeEngine(cfg, m._valid_ids(tok), B, weights=sd)
        m.engine.log = []
        m._scale, m._bias = float(sd["model.speech_scaling_factor"]), float(sd["model.speech_bias_factor"])
        return m
    return cfg, tok, make


def _requests(tok, vocab, n, seed=7):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        ids = torch.randint(0, vocab - 20, (1, 5 + 3 * i), generator=g)
        ids[0, -1] = tok.speech_start_id
        out.append(dict(input_ids=ids, cfg=[1.0, 1.3, 3.0][i % 3], steps=[1, 3, 5, 2][i % 4], max_new=[2, 6, 3, 8, 4, 5][i % 6],
                        seed=100 + i))
    return out


def _solo(model, tok, r):
    model.set_ddpm_inference_steps(r["steps"])
    torch.manual_seed(r["seed"])
    return model.generate(input_ids=r["input_ids"], tokenizer=tok, cfg_scale=r["cfg"], max_new_tokens=r["max_new"], show_progress_bar=False)


def test_queue_matches_solo_runs_and_reuses_rows(setup):
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make = setup
    reqs = _requests(tok, cfg.decoder_config.vocab_size, 6)
    model = make(2)
    q = RequestQueue(model, max_total_tokens=4096)
    rids = [q.submit(dict(input_ids=r["input_ids"]), cfg_scale=r["cfg"], steps=r["steps"], max_new_tokens=r["max_new"], seed=r["seed"])
            for r in reqs]
    assert rids == list(range(6))
    got = dict(q.run())
    assert sorted(got) == rids
    # admission: oldest first, each into the lowest free row; with 2 rows and 6 requests every row serves several requests
    prefills = [e for e in model.engine.log if e[0] == "prefill"]
    assert [p[3] for p in prefills] == [r["input_ids"].shape[1] for r in reqs]
    rows = [p[1] for p in prefills]
    assert rows[:2] == [0, 1] and rows.count(0) >= 2 and rows.count(1) >= 2
    assert model.engine.log[0] == ("per_row", max(r["steps"] for r in reqs)) and model.engine.log[-1] == ("per_row", 0)
    assert all(model.engine.kv_len(s) == 0 for s in range(4))
    solo_model = make(2)
    for rid, r in zip(rids, reqs):
        want = _solo(solo_model, tok, r)
        out = got[rid]
        assert torch.equal(out.sequences, want.sequences), (rid, out.sequences, want.sequences)
        assert torch.equal(out.reach_max_step_sample, want.reach_max_step_sample)
        a, b = out.speech_outputs[0], want.speech_outputs[0]
        assert (a is None) == (b is None)
        if a is not None:
            assert torch.allclose(a, b, rtol=1e-4, atol=1e-5), (rid, float((a - b).abs().max()))


def test_queue_prefill_chunks_match_whole_prompts(setup):
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make = setup
    reqs = _requests(tok, cfg.decoder_config.vocab_size, 3, seed=11)
    reqs[1]["input_ids"] = torch.cat([torch.randint(0, 100, (1, 150), generator=torch.Generator().manual_seed(3)),
                                      reqs[1]["input_ids"]], dim=1)
    outs = []
    for chunk in (None, 64):
        model = make(2)
        q = RequestQueue(model, max_total_tokens=4096, max_prefill_tokens_per_frame=chunk)
        for r in reqs:
            q.submit(dict(input_ids=r["input_ids"]), cfg_scale=r["cfg"], steps=r["steps"], max_new_tokens=r["max_new"], seed=r["seed"])
        outs.append(dict(q.run()))
        pf = [e for e in model.engine.log if e[0] == "prefill"]
        if chunk:
            assert max(p[3] for p in pf) <= 64 and any(p[2] > 0 for p in pf)
    for rid in outs[0]:
        assert torch.equal(outs[0][rid].sequences, outs[1][rid].sequences)
        a, b = outs[0][rid].speech_outputs[0], outs[1][rid].speech_outputs[0]
        assert (a is None) == (b is None) and (a is None or torch.allclose(a, b, rtol=1e-5, atol=1e-6))


def test_queue_waits_for_kv_pages(setup):
    """A request is admitted only while the pool holds its worst case: with room for one at a time the second waits for the first."""
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make = setup
    g = torch.Generator().manual_seed(5)
    model = make(2)
    q = RequestQueue(model, max_total_tokens=64)          # 1 + 8 pages: 4 for the sequences' next entries, 5 for requests
    for i in range(2):                                     # 40 + 70 + 2 and 70 + 2 tokens: 4 pages each
        ids = torch.randint(0, 100, (1, 40), generator=g)
        ids[0, -1] = tok.speech_start_id
        q.submit(dict(input_ids=ids), steps=2, max_new_tokens=70, seed=i)
    order = [rid for rid, _ in q.run()]
    assert order == [0, 1]
    rows = [e[1] for e in model.engine.log if e[0] == "prefill"]
    assert rows == [0, 0]                                  # the second request waited and took the first's row
    with pytest.raises(ValueError, match="max_total_tokens"):
        q.submit(dict(input_ids=torch.zeros(1, 400, dtype=torch.long)), max_new_tokens=8)


@pytest.mark.parametrize("opt,val,match", [
    ("audio_streamer", object(), "audio_streamer"),
    ("stop_check_fn", lambda: False, "stop_check_fn"),
    ("logits_processor", [lambda ids, s: s], "logits_processor"),
    ("refresh_negative", False, "refresh_negative"),
    ("generation_config", {"do_sample": True}, "do_sample"),
    ("generation_config", {"repetition_penalty": 1.2}, "repetition_penalty"),
    ("solver", "euler", "solver"),
    ("steps", 0, "steps"),
])
def test_queue_refuses_unsupported_options(setup, opt, val, match):
    from vibevoice_b200.modeling import ForcedTokenScript
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make = setup
    q = RequestQueue(make(1), max_total_tokens=1024)
    ids = torch.tensor([[1, 2, tok.speech_start_id]])
    with pytest.raises(ValueError, match=match):
        q.submit(dict(input_ids=ids), **{opt: val})
    with pytest.raises(ValueError, match="forced token scripts"):
        q.submit(dict(input_ids=ids), logits_processor=[ForcedTokenScript([[tok.eos_token_id]])])
    with pytest.raises(ValueError, match="one script per request"):
        q.submit(dict(input_ids=torch.ones(2, 3, dtype=torch.long)))
    q.submit(dict(input_ids=ids), generation_config={"do_sample": False}, max_new_tokens=2)      # greedy is served
    assert len(list(q.run())) == 1


def test_queue_refuses_prefill_chunks_on_torch_prefill(setup):
    from vibevoice_b200.serving import RequestQueue
    cfg, tok, make = setup
    m = make(1)
    m._prefill_impl, m._prefill = None, object()          # a model that prefills with TorchPrefill
    with pytest.raises(ValueError, match="max_prefill_tokens_per_frame"):
        RequestQueue(m, max_total_tokens=1024, max_prefill_tokens_per_frame=128)
