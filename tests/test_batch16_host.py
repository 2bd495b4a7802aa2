"""CPU tests of the host logic at 9..16 prompts per GPU, on the engine stand-in (tests/fake_engine.py): the product `generate()` against
`oracle.generate` at B = 12 and 16 on random forced-token scripts, and `RequestQueue` admission, row reuse and results at max_batch = 16
against solo runs.  The GPU side of the same batch sizes is tests/test_gpu_batch16.py."""
import random

import pytest
import torch

from test_queue_host import RowFakeEngine, _requests, _solo


def _scripts(rnd, tok, B):
    """Well-formed random scripts: speaker turns <speech_start> <diffusion>+ <speech_end>, each row ending with its own EOS."""
    s, e, d, x = tok.speech_start_id, tok.speech_end_id, tok.speech_diffusion_id, tok.eos_token_id
    out = []
    for _ in range(B):
        row, prev = [], s
        for _ in range(rnd.randint(2, 8)):
            nxt = rnd.choice([d, d, d, e]) if prev in (s, d) else s
            row.append(nxt)
            prev = nxt
        row.append(x)
        out.append(row)
    return out


@pytest.mark.parametrize("B,seed", [(12, 0), (16, 1)])
def test_product_generate_at_b12_b16_matches_oracle(B, seed):
    from fake_engine import make_model
    from oracle import vv_oracle as O
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.modeling import ForcedTokenScript
    from vibevoice_b200.synth import SynthTokenizer, synth_state_dict
    rnd = random.Random(4000 + seed)
    cfg = preset_config("tiny")
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, 1234, torch.float32)
    scripts = _scripts(rnd, tok, B)
    lens = [rnd.randint(3, 10) for _ in range(B)]
    L = max(lens)
    ids = torch.randint(0, 1000, (B, L), generator=torch.Generator().manual_seed(seed))
    mask = torch.zeros(B, L, dtype=torch.long)
    for r, n in enumerate(lens):                            # left-padded ragged prompts
        mask[r, L - n:] = 1
        ids[r, :L - n] = tok.pad_id
    ids[:, -1] = tok.speech_start_id
    n_new = max(len(r) for r in scripts) + 1
    model = make_model(cfg, tok, sd, max_batch=B)
    model.set_ddpm_inference_steps(3)
    torch.manual_seed(91)
    out = model.generate(input_ids=ids, attention_mask=mask, tokenizer=tok, cfg_scale=1.3, is_prefill=False, max_new_tokens=n_new,
                         max_length_times=1e9, show_progress_bar=False, logits_processor=[ForcedTokenScript(scripts)])
    torch.manual_seed(91)
    ref = O.generate(sd, cfg, ids, mask, tok, cfg_scale=1.3, num_steps=3, max_new_tokens=n_new, max_length_times=1e9,
                     forced_tokens=scripts)
    assert torch.equal(out.sequences, ref.sequences), (scripts, out.sequences, ref.sequences)
    assert torch.equal(out.reach_max_step_sample, ref.reach_max_step_sample)
    assert len(out.speech_outputs) == B
    for a, b in zip(out.speech_outputs, ref.speech_outputs):
        assert (a is None) == (b is None)
        if a is not None:
            assert a.shape == b.shape
            assert float((a.double() - b.double()).norm() / b.double().norm()) < 1e-5


def test_queue_at_max_batch_16_matches_solo_runs():
    """24 requests over 16 rows: the first 16 fill rows 0..15 in order, the other 8 take rows as they free up; every result equals the
    request's solo run; every sequence is empty afterwards."""
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    from vibevoice_b200.serving import RequestQueue
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

    reqs = _requests(tok, cfg.decoder_config.vocab_size, 24, seed=16)
    model = make(16)
    q = RequestQueue(model, max_total_tokens=16384)
    rids = [q.submit(dict(input_ids=r["input_ids"]), cfg_scale=r["cfg"], steps=r["steps"], max_new_tokens=r["max_new"], seed=r["seed"])
            for r in reqs]
    got = dict(q.run())
    assert sorted(got) == rids
    prefills = [e for e in model.engine.log if e[0] == "prefill"]
    assert [p[3] for p in prefills] == [r["input_ids"].shape[1] for r in reqs]        # oldest first, whole prompts
    rows = [p[1] for p in prefills]
    assert rows[:16] == list(range(16))
    assert all(0 <= r < 16 for r in rows[16:])                                      # later requests reuse freed rows
    assert all(model.engine.kv_len(s) == 0 for s in range(32))
    solo_model = make(1)
    for rid, r in zip(rids, reqs):
        want = _solo(solo_model, tok, r)
        out = got[rid]
        assert torch.equal(out.sequences, want.sequences), (rid, out.sequences, want.sequences)
        assert torch.equal(out.reach_max_step_sample, want.reach_max_step_sample)
        a, b = out.speech_outputs[0], want.speech_outputs[0]
        assert (a is None) == (b is None)
        if a is not None:
            assert torch.allclose(a, b, rtol=1e-4, atol=1e-5), (rid, float((a - b).abs().max()))
