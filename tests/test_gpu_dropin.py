"""`-m gpu`: the body of the reference's `demo/inference_from_file.py:280-431` against this package, through the reference's own import
paths (`vibevoice.modular.modeling_vibevoice_inference`, `vibevoice.processor.vibevoice_processor`), on a synthetic checkpoint directory:
sharded safetensors with the reference's key names + `config.json` in the shipped format + `preprocessor_config.json` + tokenizer files,
two voice wavs on disk (one at 16 kHz: the shipped `en-Alice_woman.wav` is), a script file.  The calls and keyword arguments are the
demo's, unmodified; only the model path differs.  (The tests do not depend on a reference checkout, so the flow is restated here.)"""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from vibevoice_b200.configuration import preset_config
from vibevoice_b200.synth import synth_state_dict


def _write_tokenizer(d, vocab_cap):
    """A byte-level tokenizer with the Qwen2.5 special-token NAMES the VibeVoice tokenizers resolve their ids from
    (`modular_vibevoice_text_tokenizer.py:163-181`), small enough for the tiny preset's vocabulary."""
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast
    alphabet = sorted(pre_tokenizers.ByteLevel.alphabet())
    vocab = {ch: i for i, ch in enumerate(alphabet)}
    tk = Tokenizer(models.BPE(vocab=vocab, merges=[]))
    tk.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    tk.decoder = decoders.ByteLevel()
    specials = ["<|endoftext|>", "<|vision_start|>", "<|vision_end|>", "<|vision_pad|>", "<|image_pad|>"]
    fast = PreTrainedTokenizerFast(tokenizer_object=tk, eos_token="<|endoftext|>", pad_token="<|image_pad|>",
                                   additional_special_tokens=specials[1:])
    assert len(fast) <= vocab_cap
    fast.save_pretrained(str(d))


def _make_checkpoint(tmp_path, preset="tiny"):
    from safetensors.torch import save_file
    cfg = preset_config(preset)
    sd = synth_state_dict(cfg, 1234, torch.bfloat16)          # includes the acoustic ENCODER (voice prompts) and fix_std-free heads
    ck = tmp_path / "VibeVoice-synth"
    ck.mkdir()
    d = cfg.to_dict()
    d["model_type"] = "vibepod"                               # as shipped (configs/qwen2.5_1.5b_64k.json:37)
    (ck / "config.json").write_text(json.dumps(d))
    (ck / "preprocessor_config.json").write_text(json.dumps({"speech_tok_compress_ratio": 3200, "db_normalize": True}))
    keys = sorted(sd)
    third = len(keys) // 3
    parts = (keys[:third], keys[third:2 * third], keys[2 * third:])
    for i, part in enumerate(parts):
        save_file({k: sd[k].contiguous() for k in part}, str(ck / ("model-%05d-of-%05d.safetensors" % (i + 1, len(parts)))))
    _write_tokenizer(ck, cfg.decoder_config.vocab_size)
    return ck, cfg, sd


def _write_voices(tmp_path):
    from scipy.io import wavfile
    g = np.random.default_rng(3)
    paths = []
    for name, sr, secs in (("en-Alice_woman.wav", 16000, 0.45), ("en-Carter_man.wav", 24000, 0.30)):
        t = np.arange(int(sr * secs)) / sr
        x = 0.2 * np.sin(2 * np.pi * 180.0 * t) + 0.05 * g.standard_normal(t.shape[0])
        p = str(tmp_path / name)
        wavfile.write(p, sr, (np.clip(x, -1, 1) * 32767).astype(np.int16))
        paths.append(p)
    return paths


def test_demo_inference_from_file_body(tmp_path):
    ck, cfg, sd = _make_checkpoint(tmp_path)
    voice_samples = _write_voices(tmp_path)
    txt_path = tmp_path / "2p_short.txt"
    txt_path.write_text("Speaker 1: Hello there.\nSpeaker 2: Hi, fine thanks.\nSpeaker 1: Good.\n")
    output_dir = tmp_path / "outputs"

    # ---- demo/inference_from_file.py:26-28 ----
    from vibevoice.modular.modeling_vibevoice_inference import VibeVoiceForConditionalGenerationInference
    from vibevoice.processor.vibevoice_processor import VibeVoiceProcessor
    from vibevoice.modular.lora_loading import load_lora_assets  # noqa: F401

    # ---- :236-262 (script parsing is the processor's; the demo re-joins "Speaker N: text" lines) ----
    full_script = txt_path.read_text().strip().replace("’", "'")
    # ---- :280 ----
    processor = VibeVoiceProcessor.from_pretrained(str(ck))
    # ---- :283-332, device == "cuda" ----
    load_dtype, attn_impl_primary = torch.bfloat16, "flash_attention_2"
    model = VibeVoiceForConditionalGenerationInference.from_pretrained(str(ck), torch_dtype=load_dtype, device_map="cuda",
                                                                     attn_implementation=attn_impl_primary)
    # ---- :362-368 ----
    model.eval()
    model.set_ddpm_inference_steps(num_steps=10)
    if hasattr(model.model, "language_model"):
        print(f"Language model attention: {model.model.language_model.config._attn_implementation}")
    # ---- :371-383 ----
    inputs = processor(text=[full_script], voice_samples=[voice_samples], padding=True, return_tensors="pt", return_attention_mask=True)
    target_device = "cuda"
    for k, v in inputs.items():
        if torch.is_tensor(v):
            inputs[k] = v.to(target_device)
    # ---- :388-397 ----
    torch.manual_seed(0)
    outputs = model.generate(**inputs, max_new_tokens=None, cfg_scale=1.3, tokenizer=processor.tokenizer,
                             generation_config={"do_sample": False}, verbose=True, is_prefill=True)
    # ---- :402-431 ----
    assert outputs.speech_outputs and outputs.speech_outputs[0] is not None
    audio_samples = outputs.speech_outputs[0].shape[-1]
    input_tokens = inputs["input_ids"].shape[1]
    output_tokens = outputs.sequences.shape[1]
    generated = outputs.sequences[0, input_tokens:].tolist()
    os.makedirs(output_dir, exist_ok=True)
    output_path = os.path.join(output_dir, "2p_short_generated.wav")
    processor.save_audio(outputs.speech_outputs[0], output_path=output_path)

    # ---- what must hold ----
    tok = processor.tokenizer
    assert torch.equal(outputs.sequences[0, :input_tokens].cpu(), inputs["input_ids"][0].cpu())
    valid = {tok.speech_start_id, tok.speech_end_id, tok.speech_diffusion_id, tok.eos_token_id}
    assert set(generated) <= valid and output_tokens > input_tokens
    n_diff = generated.count(tok.speech_diffusion_id)
    assert n_diff >= 1 and audio_samples == 3200 * n_diff             # one 3200-sample chunk per <speech_diffusion> (:646-650)
    assert int(inputs["speech_input_mask"].sum()) == 4 + 3             # ceil(0.45 s * 24 kHz / 3200) + ceil(0.30 s * 24 kHz / 3200)
    from scipy.io import wavfile
    sr, wav = wavfile.read(output_path)
    assert sr == 24000 and wav.shape[0] == audio_samples and np.isfinite(wav).all() and float(np.abs(wav).max()) > 0
    # a second call on the same object with a longer prompt re-sizes the KV pool instead of failing (long-lived server, ADVICE r01)
    long_script = "\n".join("Speaker %d: %s" % (1 + i % 2, "and then some more words to say " * 3) for i in range(6))
    inputs2 = processor(text=[long_script], voice_samples=[voice_samples], padding=True, return_tensors="pt", return_attention_mask=True)
    assert inputs2["input_ids"].shape[1] > 2 * input_tokens
    out2 = model.generate(**inputs2, max_new_tokens=6, cfg_scale=1.3, tokenizer=processor.tokenizer, generation_config={"do_sample": False},
                          is_prefill=True, show_progress_bar=False)
    assert out2.sequences.shape[1] > inputs2["input_ids"].shape[1]
    # a tokenizer whose special ids differ from the ones the weights were packed for is refused, not silently mis-constrained
    class Other:
        speech_start_id, speech_end_id, speech_diffusion_id, eos_token_id, bos_token_id = 5, 6, 7, 8, None
    with pytest.raises(ValueError):
        model.generate(**inputs, max_new_tokens=2, tokenizer=Other(), is_prefill=True, show_progress_bar=False)
    # connector / full-head state dicts go in through the reference's own calls (lora_loading.py:57-66, 104-112)
    new_fc1 = {"fc1.weight": torch.randn(cfg.decoder_config.hidden_size, 64) * 0.05, "fc1.bias": torch.zeros(cfg.decoder_config.hidden_size)}
    res = model.model.acoustic_connector.load_state_dict(new_fc1, strict=False)
    assert "fc2.weight" in res.missing_keys and not res.unexpected_keys
    model.model.acoustic_connector.to(next(model.parameters()).device)
    torch.manual_seed(0)
    out3 = model.generate(**inputs, max_new_tokens=4, cfg_scale=1.3, tokenizer=processor.tokenizer, is_prefill=True, show_progress_bar=False)
    assert out3.sequences.shape[1] > input_tokens
    model.engine.close()


def test_sampling_with_hf_warpers_and_custom_processor(tmp_path):
    """`do_sample=True` with HF's sampling defaults (top_k = 50 over the WHOLE vocabulary before the constraint, :310-319) and a
    caller-supplied LogitsProcessor: both run on full-vocabulary logits from vv_lm_logits_full.  Checked against the same arithmetic in
    PyTorch on the hidden state the engine reports."""
    from transformers import LogitsProcessor
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    from vibevoice_b200.synth import SynthTokenizer
    cfg = preset_config("tiny")
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    sd = synth_state_dict(cfg, 1234, torch.bfloat16)
    model = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=2)
    model.load_state_dict(sd, tok)
    eng = model.engine
    # full logits == hidden @ E^T
    with torch.cuda.stream(eng.stream):
        eng.hidden.normal_(0, 1)
    eng.sync()
    got = eng.lm_logits_full().cpu()
    want = eng.hidden[:2].cpu() @ sd["model.language_model.embed_tokens.weight"].float().T
    assert float((got - want).norm() / want.norm()) < 2e-5

    class Boost(LogitsProcessor):          # pushes <speech_diffusion> above everything for 3 steps, then EOS
        def __init__(self):
            self.n = 0

        def __call__(self, input_ids, scores):
            self.n += 1
            scores = scores.clone()
            scores[:, tok.speech_diffusion_id if self.n <= 3 else tok.eos_token_id] += 1e4
            return scores
    ids = torch.randint(0, 1000, (2, 9), generator=torch.Generator().manual_seed(0))
    ids[:, -1] = tok.speech_start_id
    model.set_ddpm_inference_steps(4)
    out = model.generate(input_ids=ids, tokenizer=tok, cfg_scale=1.3, is_prefill=False, max_new_tokens=8, logits_processor=[Boost()],
                         show_progress_bar=False)
    d, x = tok.speech_diffusion_id, tok.eos_token_id
    assert out.sequences[:, 9:].tolist() == [[d, d, d, x], [d, d, d, x]]
    assert out.speech_outputs[0].shape == (1, 9600)
    # HF default top_k=50 over the full vocabulary: a random-init model rarely ranks a special id in its top 50 -> the reference's softmax
    # is NaN there and torch.multinomial raises; top_k=0 samples from the constrained softmax
    out = model.generate(input_ids=ids, tokenizer=tok, cfg_scale=1.3, is_prefill=False, max_new_tokens=4, show_progress_bar=False,
                         generation_config={"do_sample": True, "top_k": 0, "top_p": 0.9, "temperature": 0.7})
    assert set(out.sequences[:, 9:].flatten().tolist()) <= set(eng.valid_ids) | {tok.pad_token_id}
    model.engine.close()
