"""`RequestQueue` on the GPU: requests of different lengths, some with voice prompts, with mixed CFG scales, step counts and solvers, served
over B rows that each take several requests.  Per request the tokens and `reach_max_step_sample` must equal a solo `generate()` run under
the queue's RNG contract (`torch.manual_seed(seed)`, that request alone, its steps and solver) and the audio must be within the
closed-loop tolerance of the parity tests; the pool is free again afterwards; spreading prompts over frames changes nothing."""
import pytest
import torch

from vibevoice_b200.configuration import preset_config
from vibevoice_b200.schedule import DPMSolverMultistepScheduler
from vibevoice_b200.synth import SynthTokenizer, synth_state_dict

pytestmark = pytest.mark.gpu

AUDIO_TOL = 1e-2          # closed loop, as test_gpu_parity.py::test_sde_sampler_vs_oracle


def rel_l2(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def make_model(preset, B, **kw):
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    cfg = preset_config(preset)
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, 1234, torch.bfloat16)
    m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=B, **kw)
    m.load_state_dict(sd, tok)
    return m, cfg, tok


def requests(cfg, tok, n, B, seed, voices=True):
    """n single-script requests: the first B short, the rest longer (so every row serves at least two), every third with a voice."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        L0 = 12 + 5 * i
        ids = torch.randint(0, cfg.decoder_config.vocab_size - 20, (1, L0), generator=g)
        ids[0, -1] = tok.speech_start_id
        inp = dict(input_ids=ids, attention_mask=torch.ones(1, L0, dtype=torch.long))
        if voices and i % 3 == 1:
            nf = 2 + i % 2
            wav = torch.randn(1, nf * 3200, generator=g) * 0.1
            sim = torch.zeros(1, L0, dtype=torch.bool)
            sim[0, 2:2 + nf] = True
            ids[sim] = tok.speech_diffusion_id
            inp.update(speech_tensors=wav, speech_masks=torch.ones(1, nf, dtype=torch.bool), speech_input_mask=sim)
        out.append(dict(inputs=inp, cfg_scale=[1.3, 1.0, 3.0][i % 3], steps=[5, 10, 3, 20][i % 4],
                        solver=["dpmsolver++", "sde-dpmsolver++"][(i // 2) % 2], max_new_tokens=(3 + 2 * i) if i < B else 12 + i,
                        seed=1000 + i))
    return out


def serve(m, reqs, **kw):
    from vibevoice_b200.serving import RequestQueue
    eng = m.engine
    rows = []
    prefill = eng.lm_prefill

    def logged(seq, embeds, pos0=0, workspace_bytes=None):
        rows.append((seq, pos0, int(embeds.shape[0])))
        return prefill(seq, embeds, pos0=pos0, workspace_bytes=workspace_bytes)
    eng.lm_prefill = logged
    try:
        q = RequestQueue(m, max_total_tokens=16384, **kw)
        rids = [q.submit(r["inputs"], cfg_scale=r["cfg_scale"], steps=r["steps"], solver=r["solver"], max_new_tokens=r["max_new_tokens"],
                         seed=r["seed"]) for r in reqs]
        got = dict(q.run())
        assert sorted(got) == rids
        assert eng.kv_pages_free() == eng.kv_pages        # every page back in the pool
    finally:
        del eng.lm_prefill
    return [got[i] for i in rids], rows


def solo(m, tok, r):
    base = m.engine.scheduler
    m.model.noise_scheduler = DPMSolverMultistepScheduler.from_config(base.config, algorithm_type=r["solver"])
    m.set_ddpm_inference_steps(r["steps"])
    torch.manual_seed(r["seed"])
    out = m.generate(**r["inputs"], tokenizer=tok, cfg_scale=r["cfg_scale"], max_new_tokens=r["max_new_tokens"], is_prefill=True,
                     show_progress_bar=False)
    return out


def check(m, tok, reqs, got):
    for i, (r, out) in enumerate(zip(reqs, got)):
        want = solo(m, tok, r)
        assert torch.equal(out.sequences, want.sequences), (i, out.sequences, want.sequences)
        assert torch.equal(out.reach_max_step_sample, want.reach_max_step_sample), i
        a, b = out.speech_outputs[0], want.speech_outputs[0]
        assert (a is None) == (b is None), i
        if a is not None:
            assert a.shape == b.shape and rel_l2(a, b) < AUDIO_TOL, (i, rel_l2(a, b))


@pytest.mark.parametrize("B,n", [(2, 6), (4, 8)])
def test_queue_matches_solo_generate(B, n):
    m, cfg, tok = make_model("tiny", B, prefill_impl="native")
    try:
        reqs = requests(cfg, tok, n, B, seed=B)
        got, rows = serve(m, reqs)
        assert [p[2] for p in rows] == [r["inputs"]["input_ids"].shape[1] for r in reqs]        # oldest first, whole prompts
        assert all(sum(1 for p in rows if p[0] == r) >= 2 for r in range(B)), rows
        check(m, tok, reqs, got)
    finally:
        m.engine.close()


def test_queue_prefill_chunks_match_whole_prompts():
    m, cfg, tok = make_model("tiny", 2, prefill_impl="native")
    try:
        reqs = requests(cfg, tok, 5, 2, seed=7)
        ids = reqs[2]["inputs"]["input_ids"]
        long = torch.cat([torch.randint(0, 1000, (1, 300), generator=torch.Generator().manual_seed(1)), ids], dim=1)
        reqs[2]["inputs"] = dict(input_ids=long, attention_mask=torch.ones_like(long))
        whole, _ = serve(m, reqs)
        chunked, rows = serve(m, reqs, max_prefill_tokens_per_frame=128)
        assert max(p[2] for p in rows) <= 128 and any(p[1] > 0 for p in rows)
        for a, b in zip(whole, chunked):
            assert torch.equal(a.sequences, b.sequences)
            assert (a.speech_outputs[0] is None) == (b.speech_outputs[0] is None)
            if a.speech_outputs[0] is not None:
                assert rel_l2(b.speech_outputs[0], a.speech_outputs[0]) < AUDIO_TOL
    finally:
        m.engine.close()


def test_queue_torch_prefill_model():
    """A model that keeps the PyTorch prefill admits through it (and generate() uses it too)."""
    m, cfg, tok = make_model("tiny", 2, torch_prefill=True)
    try:
        reqs = requests(cfg, tok, 4, 2, seed=3)
        got, rows = serve(m, reqs)
        assert rows == []                                   # no native prefill call
        check(m, tok, reqs, got)
    finally:
        m.engine.close()


def test_queue_real_15b_layer_shapes():
    """Two requests at the 1.5B layer shapes (two decoder layers, full widths)."""
    m, cfg, tok = make_model("1.5b-l2", 2, prefill_impl="native")
    try:
        reqs = requests(cfg, tok, 2, 2, seed=5, voices=False)
        got, _ = serve(m, reqs)
        check(m, tok, reqs, got)
    finally:
        m.engine.close()
