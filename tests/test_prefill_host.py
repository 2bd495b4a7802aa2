"""CPU tests of the `prefill_impl="native"` branch of `generate()`: the product's host code (embedding gather, voice scatter, one
`lm_prefill` call per row, lengths, the negative-row decode and the first token decision) driven through the CPU stand-in of the engine
with oracle arithmetic for the two prefill entry points, held to the reference's own `generate()` fixtures (`tests/golden/loop.pt`)."""
import pytest
import torch

from oracle import vv_oracle as O


def _prefill_engine_cls():
    from fake_engine import FakeEngine

    class PrefillFakeEngine(FakeEngine):
        """FakeEngine + the native prefill entry points (`vv_embed_gather`, `vv_lm_prefill`) in oracle arithmetic."""

        def embed_gather(self, ids):
            self.calls["embed_gather"] = self.calls.get("embed_gather", 0) + 1
            return self.embed_w[torch.as_tensor(ids).long().reshape(-1)].clone()

        def lm_prefill(self, seq, embeds, pos0=0, workspace_bytes=None):
            self.calls["lm_prefill"] = self.calls.get("lm_prefill", 0) + 1
            assert pos0 == len(self.kv[seq]) and embeds.dim() == 2 and embeds.dtype == torch.float32
            return O.qwen2_forward(self.w, self.config.decoder_config, embeds, self.kv[seq], pos0)[-1]

    return PrefillFakeEngine


def _native_model(cfg, tok, sd, B):
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=B, prefill_impl="native")
    m.engine = _prefill_engine_cls()(cfg, m._valid_ids(tok), B, weights=sd)
    m._scale, m._bias = float(sd["model.speech_scaling_factor"]), float(sd["model.speech_bias_factor"])
    return m


@pytest.mark.parametrize("case", ["scripted", "free", "maxlen", "norefresh1", "norefresh", "sde", "voice"])
def test_native_prefill_branch_against_reference_generate_fixture(golden, case):
    """Sequences and reach-max flags exact, audio within 1e-5 of the reference's generate(); one prefill call per row, no token-by-token
    prompt decode (the first decode call is the negative rows' <speech_start> step)."""
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.modeling import ForcedTokenScript
    from vibevoice_b200.synth import SynthTokenizer, synth_state_dict
    g = {**golden("loop"), **golden("loop2")}
    c = g[case]
    cfg = preset_config(g["preset"])
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, 1234, torch.float32)
    B = c["ids"].shape[0]
    model = _native_model(cfg, tok, sd, B)
    model.set_ddpm_inference_steps(g["num_steps"])
    extra = {}
    if "wavs" in c:                      # the prefill draws its Gaussian voice sample first, from the same CPU stream as the frame noise
        model._voice = lambda wavs, masks, scale, bias, noise=None: O.voice_prompt_embeds(sd, cfg, wavs, masks)
        extra = dict(is_prefill=True, speech_tensors=c["wavs"], speech_masks=c["voice_masks"], speech_input_mask=c["speech_input_mask"])
    else:
        extra = dict(is_prefill=False)
    if c.get("algorithm_type") == "sde-dpmsolver++":
        from vibevoice_b200.schedule import DPMSolverMultistepScheduler
        base = DPMSolverMultistepScheduler()
        model.model.noise_scheduler = base.from_config(base.config, algorithm_type="sde-dpmsolver++", beta_schedule="squaredcos_cap_v2")
    torch.manual_seed(c["seed"])
    out = model.generate(input_ids=c["ids"], attention_mask=c["mask"], tokenizer=tok, cfg_scale=g["cfg_scale"],
                         max_new_tokens=c["max_new_tokens"], max_length_times=c["max_length_times"], show_progress_bar=False,
                         logits_processor=[ForcedTokenScript(c["scripts"])] if c["scripts"] else None,
                         refresh_negative=c["refresh_negative"], **extra)
    assert torch.equal(out.sequences, c["sequences"])
    assert torch.equal(out.reach_max_step_sample, c["reach_max"])
    for a, b in zip(out.speech_outputs, c["audio"]):
        assert (a is None) == (b is None)
        if a is not None:
            assert a.shape == b.shape
            rel = float((a.double() - b.double()).norm() / b.double().norm())
            assert rel < 1e-5, rel
    calls = model.engine.calls
    assert calls["lm_prefill"] == B and calls["embed_gather"] == B


def test_native_prefill_is_opt_in():
    """Without the argument nothing changes: no model-level prefill default and no bf16 LM copy; with it no copy either, other values are
    refused, and the drop-in import path takes the argument too."""
    import inspect
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference as M
    from vibevoice_b200.synth import SynthTokenizer
    cfg = preset_config("tiny")
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    assert M(cfg, tok)._prefill_impl is None and M(cfg, tok)._torch_prefill is False
    m = M(cfg, tok, prefill_impl="native")
    assert m._prefill_impl == "native" and m._torch_prefill is False
    with pytest.raises(ValueError):
        M(cfg, tok, prefill_impl="torch")
    from vibevoice.modular.modeling_vibevoice_inference import VibeVoiceForConditionalGenerationInference as Drop
    assert "prefill_impl" in inspect.signature(Drop.__init__).parameters
