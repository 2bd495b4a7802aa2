"""`-m gpu`: the streaming-0.5B demo (`demo/streaming_inference_from_file.py`) against this package, from a shipped voice preset.

  * the demo's body through the reference's own import paths on a synthetic checkpoint directory at the shipped geometry (24 layers split
    4 / 20, H = 896, 14 / 2 heads of 64; reduced vocabulary) with tokenizer files, `preprocessor_config.json` and
    `voices/streaming_model/en-Mike_man.pt` = `tests/golden/streaming_preset.pt` (the shipped preset cut to 24 / 48 / 1 / 1 positions);
  * the import of the preset's K/V into the paged pool, bit for bit;
  * `generate(all_prefilled_outputs=...)` against the streaming oracle started from the same preset (`tests/streaming_oracle.py`);
  * `vv_eos_prob` against float64 and `vv_tts_type_embed` against PyTorch's fp32 add.
(The tests do not depend on a reference checkout, so the demo's flow is restated here.)
"""
import copy
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from vibevoice_b200.configuration import VibeVoiceConfig, preset_config
from vibevoice_b200.synth import synth_state_dict

from test_gpu_dropin import _write_tokenizer
from test_gpu_parity import SEED, rel_l2, report

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PARTS = ("lm", "head", "acoustic_decoder", "connectors", "lm_head")
TTS_LAYERS = 20
MAX_NEW = 40                       # the checkpoint's max_position_embeddings = cached TTS-LM positions + MAX_NEW: the demo passes
                                   # max_new_tokens=None, so this is where its loop stops when the classifier does not fire


def _preset():
    return torch.load(os.path.join(GOLDEN, "streaming_preset.pt"), map_location="cpu", weights_only=False)


def _cut_lengths():
    return torch.load(os.path.join(GOLDEN, "streaming_processor.pt"), weights_only=False)["preset"]["lengths"]


def _cfg():
    d = preset_config("streaming-0.5b").to_dict()
    d["decoder_config"]["vocab_size"] = 4096
    d["decoder_config"]["max_position_embeddings"] = _cut_lengths()["tts_lm"] + MAX_NEW
    return VibeVoiceConfig.from_dict(d)


@pytest.fixture(scope="module")
def shipped():
    """config, the streaming state dict (EOS classifier biased off) and its multi-speaker base, at the shipped geometry."""
    from oracle import vv_streaming as VS
    cfg = _cfg()
    assert cfg.decoder_config.num_hidden_layers == 24 and cfg.decoder_config.hidden_size == 896 and cfg.decoder_config.head_dim == 64
    base = synth_state_dict(cfg, SEED, torch.bfloat16, parts=PARTS)
    return cfg, base, VS.streaming_state_dict(base, cfg, TTS_LAYERS, eos_bias=-20.0)


def _model(cfg, sd):
    from vibevoice_b200 import streaming as S
    m = S.VibeVoiceStreamingForConditionalGenerationInference(cfg, tts_backbone_num_hidden_layers=TTS_LAYERS)
    m.load_state_dict(sd)
    return m


def _expected_sequence(prompt_len, text, max_length):
    """The reference loop's `sequences` when the classifier never fires: windows of 5 text ids, then 6 speech frames (a 1 each), until the
    length limit; also the number of frames whose audio is kept."""
    seq, frames, win = [None] * prompt_len, 0, 0
    while True:
        cur = text[win * 5:(win + 1) * 5]
        win += 1
        if cur:
            seq += cur
            if len(seq) > max_length:
                return seq, frames
        for _ in range(6):
            frames += 1
            seq.append(1)
            if len(seq) > max_length:
                break
        if len(seq) > max_length:
            return seq, frames


def test_demo_streaming_inference_from_file_body(tmp_path, shipped):
    from safetensors.torch import save_file
    cfg, _, sd = shipped
    ck = tmp_path / "VibeVoice-Realtime-synth"
    ck.mkdir()
    d = cfg.to_dict()
    d["model_type"] = "vibevoice_streaming"
    d["tts_backbone_num_hidden_layers"] = TTS_LAYERS
    d.pop("semantic_tokenizer_config", None)
    (ck / "config.json").write_text(json.dumps(d))
    (ck / "preprocessor_config.json").write_text(json.dumps({"processor_class": "VibeVoiceStreamingProcessor", "speech_tok_compress_ratio": 3200,
                                                             "db_normalize": True, "language_model_pretrained_name": "Qwen/Qwen2.5-0.5B"}))
    keys = sorted(sd)
    half = len(keys) // 2
    for i, part in enumerate((keys[:half], keys[half:])):
        save_file({k: sd[k].contiguous() for k in part}, str(ck / ("model-%05d-of-00002.safetensors" % (i + 1))))
    _write_tokenizer(ck, cfg.decoder_config.vocab_size)
    voices = tmp_path / "voices" / "streaming_model"
    voices.mkdir(parents=True)
    (voices / "en-Mike_man.pt").write_bytes(open(os.path.join(GOLDEN, "streaming_preset.pt"), "rb").read())
    txt_path = tmp_path / "1p_short.txt"
    txt_path.write_text("Hello there, this is a streaming test.\n")
    output_dir = tmp_path / "outputs"

    # ---- demo/streaming_inference_from_file.py:31-32 ----
    from vibevoice.modular.modeling_vibevoice_streaming_inference import VibeVoiceStreamingForConditionalGenerationInference
    from vibevoice.processor.vibevoice_streaming_processor import VibeVoiceStreamingProcessor
    # ---- :220-228 (the script file is read, stripped and its quotes normalised) ----
    full_script = txt_path.read_text(encoding="utf-8").strip().replace("’", "'").replace("“", '"').replace("”", '"')
    processor = VibeVoiceStreamingProcessor.from_pretrained(str(ck))
    # ---- :230-262, device == "cuda" ----
    load_dtype, attn_impl_primary = torch.bfloat16, "flash_attention_2"
    model = VibeVoiceStreamingForConditionalGenerationInference.from_pretrained(str(ck), torch_dtype=load_dtype, device_map="cuda",
                                                                              attn_implementation=attn_impl_primary)
    try:
        # ---- :279-284 ----
        model.eval()
        model.set_ddpm_inference_steps(num_steps=5)
        if hasattr(model.model, "language_model"):
            print(f"Language model attention: {model.model.language_model.config._attn_implementation}")
        # ---- :286-311 ----
        target_device = "cuda"
        voice_sample = str(voices / "en-Mike_man.pt")
        all_prefilled_outputs = torch.load(voice_sample, map_location=target_device, weights_only=False)
        inputs = processor.process_input_with_cached_prompt(text=full_script, cached_prompt=all_prefilled_outputs, padding=True,
                                                            return_tensors="pt", return_attention_mask=True)
        for k, v in inputs.items():
            if torch.is_tensor(v):
                inputs[k] = v.to(target_device)
        # ---- :316-326 ----
        torch.manual_seed(0)
        outputs = model.generate(**inputs, max_new_tokens=None, cfg_scale=1.5, tokenizer=processor.tokenizer,
                                 generation_config={"do_sample": False}, verbose=True,
                                 all_prefilled_outputs=copy.deepcopy(all_prefilled_outputs) if all_prefilled_outputs is not None else None)
        # ---- :330-360 ----
        assert outputs.speech_outputs and outputs.speech_outputs[0] is not None
        audio_samples = outputs.speech_outputs[0].shape[-1]
        output_path = os.path.join(output_dir, "1p_short_generated.wav")
        os.makedirs(output_dir, exist_ok=True)
        processor.save_audio(outputs.speech_outputs[0], output_path=output_path)
    finally:
        model.engine.close()

    # ---- what must hold ----
    lengths = _cut_lengths()
    tts_ids = inputs["tts_lm_input_ids"][0].cpu()
    assert tts_ids.numel() == lengths["tts_lm"] and inputs["input_ids"].shape[1] == lengths["lm"]
    seq = outputs.sequences[0].cpu()
    assert torch.equal(seq[:tts_ids.numel()], tts_ids)
    text = inputs["tts_text_ids"][0].cpu().tolist()
    assert len(text) > 5                                                # at least two text windows
    want, frames = _expected_sequence(tts_ids.numel(), text, cfg.decoder_config.max_position_embeddings)
    assert seq[tts_ids.numel():].tolist() == want[tts_ids.numel():]     # text windows of 5 and speech windows of 6 interleave
    assert bool(outputs.reach_max_step_sample[0])
    assert audio_samples == 3200 * frames
    from scipy.io import wavfile
    sr, wav = wavfile.read(output_path)
    assert sr == 24000 and wav.shape[0] == audio_samples and np.isfinite(wav).all() and float(np.abs(wav).max()) > 0


def test_preset_import_is_bit_exact(shipped):
    """After generate() has imported the preset (stopped before its first window), every layer of the three imported streams holds the
    preset's K/V bit for bit, the streams have the preset's lengths, and the two TTS-LM rows hold its last hidden states."""
    from streaming_oracle import cache_layers
    from vibevoice_b200.streaming import ROW_NEG, ROW_POS, ROW_TEXT
    cfg, _, sd = shipped
    preset, lengths = _preset(), _cut_lengths()
    m = _model(cfg, sd)
    try:
        out = m.generate(input_ids=torch.zeros(1, lengths["lm"], dtype=torch.long), tts_lm_input_ids=torch.zeros(1, lengths["tts_lm"], dtype=torch.long),
                         tts_text_ids=torch.tensor([[5, 6, 7]]), neg_text_input_id=0, all_prefilled_outputs=copy.deepcopy(preset),
                         stop_check_fn=lambda: True)
        assert out.speech_outputs == [None]
        eng = m.engine
        for row, name, layer0 in ((ROW_TEXT, "lm", 0), (ROW_POS, "tts_lm", m.low), (ROW_NEG, "neg_tts_lm", m.low)):
            kvs = cache_layers(preset[name].past_key_values)
            assert eng.kv_len(row) == lengths[name]
            for j, (k, v) in enumerate(kvs):
                kd, vd = eng.kv_read(row, layer0 + j, 0, lengths[name])
                assert torch.equal(kd.cpu(), k[0].transpose(0, 1)) and torch.equal(vd.cpu(), v[0].transpose(0, 1)), (name, j)
        eng.sync()
        assert torch.equal(eng.hidden[ROW_POS].cpu(), preset["tts_lm"].last_hidden_state[0, -1].float())
        assert torch.equal(eng.hidden[ROW_NEG].cpu(), preset["neg_tts_lm"].last_hidden_state[0, -1].float())
    finally:
        m.engine.close()


@pytest.mark.parametrize("case,eos_bias,n_text,max_new,cfg_scale", [("eos", 20.0, 12, 40, 1.5), ("windows", -20.0, 12, 30, 1.5),
                                                                    ("short", -20.0, 3, 7, 1.3)])
def test_generate_from_preset_vs_oracle(shipped, case, eos_bias, n_text, max_new, cfg_scale):
    """eos: the classifier fires inside the first speech window; windows: text-less windows up to the length limit; short: text shorter
    than one window, the limit hit inside a speech window."""
    from oracle import vv_streaming as VS
    from streaming_oracle import generate_from_prefilled
    cfg, base, _ = shipped
    sd = VS.streaming_state_dict(base, cfg, TTS_LAYERS, eos_bias=eos_bias)
    preset, lengths = _preset(), _cut_lengths()
    g = torch.Generator().manual_seed(11)
    text = torch.randint(0, 2000, (n_text,), generator=g)
    tts_ids = torch.full((lengths["tts_lm"],), 3, dtype=torch.long)
    m = _model(cfg, sd)
    try:
        m.set_ddpm_inference_steps(5)
        torch.manual_seed(0)
        out = m.generate(input_ids=torch.full((1, lengths["lm"]), 3), tts_lm_input_ids=tts_ids[None], tts_text_ids=text[None], neg_text_input_id=3,
                         cfg_scale=cfg_scale, max_new_tokens=max_new, all_prefilled_outputs=copy.deepcopy(preset))
    finally:
        m.engine.close()
    torch.manual_seed(0)
    ref = generate_from_prefilled(sd, cfg, TTS_LAYERS, preset, tts_ids, text, cfg_scale=cfg_scale, num_steps=5, max_new_tokens=max_new,
                                  kv_bf16=True)
    assert torch.equal(out.sequences, ref.sequences), (out.sequences, ref.sequences)
    assert torch.equal(out.reach_max_step_sample, ref.reach_max_step_sample)
    n_frames = int((ref.sequences[0, lengths["tts_lm"]:] == 1).sum())
    if case == "eos":
        assert not bool(ref.reach_max_step_sample[0]) and ref.sequences.shape[1] == lengths["tts_lm"] + 5 + 6
        assert ref.speech_outputs[0].shape[-1] < 3200 * n_frames          # frames after the classifier fired are not kept
    else:
        assert bool(ref.reach_max_step_sample[0])
    e = rel_l2(out.speech_outputs[0].cpu(), ref.speech_outputs[0])
    report("streaming_generate_from_preset", case=case, audio_rel_l2=e)
    assert e < 1e-2, e


def _heads_engine(preset):
    from oracle import vv_streaming as VS
    cfg = preset_config(preset)
    tts = 1 if preset == "tiny" else 3
    base = synth_state_dict(cfg, SEED, torch.float32, parts=PARTS)
    sd = VS.streaming_state_dict(base, cfg, tts)
    return _model_n(cfg, sd, tts), sd, cfg


def _model_n(cfg, sd, tts):
    from vibevoice_b200 import streaming as S
    m = S.VibeVoiceStreamingForConditionalGenerationInference(cfg, tts_backbone_num_hidden_layers=tts)
    m.load_state_dict(sd)
    return m


@pytest.mark.parametrize("preset", ["tiny", "streaming-0.5b-l4"])
def test_eos_prob_kernel_vs_float64(preset):
    m, sd, cfg = _heads_engine(preset)
    eng = m.engine
    try:
        H = cfg.decoder_config.hidden_size
        w1, b1 = sd["tts_eos_classifier.fc1.weight"].double(), sd["tts_eos_classifier.fc1.bias"].double()
        w2, b2 = sd["tts_eos_classifier.fc2.weight"].double()[0], sd["tts_eos_classifier.fc2.bias"].double()[0]
        g = torch.Generator().manual_seed(5)
        for scale in (1.0, 1e3):
            for _ in range(4):
                h = torch.randn(H, generator=g) * scale
                pre = w1 @ h.double() + b1
                ref = float(w2 @ torch.relu(pre) + b2)
                mag = float(w2.abs() @ ((w1 * h.double()).abs().sum(1) + b1.abs()) + b2.abs())   # sum of |every product and bias|
                hd = h.to(eng.device)
                torch.cuda.synchronize()                                     # the engine reads its inputs on its own stream
                p = eng.eos_prob(hd)
                lg = eng.eos_logit
                assert abs(lg - ref) <= 1e-6 * mag, (scale, lg, ref, mag)
                assert abs(p - float(torch.sigmoid(torch.tensor(lg, dtype=torch.float64)))) <= 1e-6
                assert (p > 0.5) == (lg > 0) or abs(lg) < 1e-6
                assert eng.eos_prob(hd) == p and eng.eos_logit == lg         # bit-identical from call to call
                report("eos_prob_kernel", preset=preset, scale=scale, logit_err_over_mag=abs(lg - ref) / mag)
    finally:
        eng.close()


def test_tts_type_embed_kernel_is_the_fp32_add():
    m, sd, cfg = _heads_engine("streaming-0.5b-l4")
    eng = m.engine
    try:
        H = cfg.decoder_config.hidden_size
        types = sd["model.tts_input_types.weight"].float()
        g = torch.Generator().manual_seed(9)
        for t in (0, 1):
            src = (torch.randn(H, generator=g) * 3).to(eng.device)
            dst = torch.full((4, H), float("nan"), device=eng.device)
            torch.cuda.synchronize()                                         # the engine reads its inputs on its own stream
            eng.tts_type_embed(src, t, [0, 2], dst)
            eng.sync()
            want = src.cpu() + types[t]
            assert torch.equal(dst[0].cpu(), want) and torch.equal(dst[2].cpu(), want)
            assert torch.isnan(dst[1]).all() and torch.isnan(dst[3]).all()
            dst[0].copy_(src)
            torch.cuda.synchronize()
            eng.tts_type_embed(dst[0], t, [0, 2], dst)                       # src aliasing a destination row
            eng.sync()
            assert torch.equal(dst[0].cpu(), want) and torch.equal(dst[2].cpu(), want)
        with pytest.raises(ValueError):
            eng.tts_type_embed(src, 0, [4], dst)
    finally:
        eng.close()


def test_multi_speaker_engine_has_no_streaming_heads():
    from vibevoice_b200 import _native as N
    from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
    from vibevoice_b200.synth import SynthTokenizer
    cfg = preset_config("tiny")
    tok = SynthTokenizer(cfg.decoder_config.vocab_size)
    m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=1)
    m.load_state_dict(synth_state_dict(cfg, SEED, torch.bfloat16), tok)
    try:
        assert not m.engine.has_tts_heads
        with pytest.raises(N.VVError):
            m.engine.eos_prob()
    finally:
        m.engine.close()
