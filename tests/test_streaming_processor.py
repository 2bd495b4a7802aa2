"""CPU tests of the streaming-0.5B demo surface (`demo/streaming_inference_from_file.py`):

  * `VibeVoiceStreamingProcessor` against the reference's own processor (`tests/golden/streaming_processor.pt`, written by
    `tools/make_streaming_golden.py`), its error surface and its offline tokenizer resolution;
  * the shipped voice-preset format (`tests/golden/streaming_preset.pt`: a cut `en-Mike_man.pt`) as the demo loads it;
  * the streaming oracle started from `all_prefilled_outputs` against the reference's own generate() (`tests/golden/streaming.pt`);
  * the product's streaming host loop (engine stand-in) from the same prefilled outputs, with and without the engine's type-embedding /
    EOS methods.
"""
import copy
import json
import os
from types import SimpleNamespace

import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class StubTokenizer:
    """What the streaming processor needs of the tokenizer: `pad_id` and `encode` (one id per UTF-8 byte, offset past the specials)."""
    pad_id = 3

    def encode(self, text, add_special_tokens=False):
        assert add_special_tokens is False
        return [10 + b for b in text.encode("utf-8")]

    def decode(self, ids, **kw):
        return bytes(i - 10 for i in ids).decode("utf-8")

    def batch_decode(self, seqs, **kw):
        return [self.decode(s) for s in seqs]


# (text, return_tensors, return_attention_mask): one text shorter than one 5-token window, one with surrounding whitespace, one non-ASCII
CASES = [
    ("Hi", "pt", True),
    ("  \tHello there, this is the streaming demo.  \n\n", "pt", True),
    ("Café naïve — déjà vu", "pt", True),
    ("Café naïve — déjà vu", None, True),
    ("  short  ", "pt", False),
]


def _preset():
    return torch.load(os.path.join(GOLDEN, "streaming_preset.pt"), weights_only=False)


def _processor():
    from vibevoice.processor.vibevoice_streaming_processor import VibeVoiceStreamingProcessor
    return VibeVoiceStreamingProcessor(tokenizer=StubTokenizer())


def _same(a, b):
    if torch.is_tensor(b):
        return torch.is_tensor(a) and a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)
    return type(a) is type(b) and a == b


def test_streaming_processor_matches_the_reference(golden):
    g = golden("streaming_processor")
    assert [(c["text"], c["return_tensors"], c["return_attention_mask"]) for c in g["cases"]] == CASES
    proc, preset = _processor(), _preset()
    for c in g["cases"]:
        out = proc.process_input_with_cached_prompt(text=c["text"], cached_prompt=preset, padding=True, return_tensors=c["return_tensors"],
                                                    return_attention_mask=c["return_attention_mask"])
        ref = c["out"]
        assert set(out) == set(ref), (c["text"], sorted(out), sorted(ref))
        for k in ref:
            assert _same(out[k], ref[k]), (c["text"], k, out[k], ref[k])
        assert out.input_ids is out["input_ids"]                  # attribute access, as the demo's `inputs.items()` / `**inputs` use it


def test_streaming_processor_surface(tmp_path):
    proc = _processor()
    with pytest.raises(NotImplementedError):
        proc()
    with pytest.raises(NotImplementedError):
        proc(text="Hi")
    assert proc.decode(StubTokenizer().encode("abc")) == "abc"
    assert proc.batch_decode([StubTokenizer().encode("ab")]) == ["ab"]
    proc.save_pretrained(str(tmp_path / "p"))
    cfg = json.loads((tmp_path / "p" / "preprocessor_config.json").read_text())
    assert cfg["processor_class"] == "VibeVoiceStreamingProcessor" and cfg["speech_tok_compress_ratio"] == 3200 and cfg["db_normalize"] is True
    from scipy.io import wavfile
    wav = proc.save_audio(torch.linspace(-0.5, 0.5, 3200)[None], output_path=str(tmp_path / "out" / "a.wav"))
    sr, x = wavfile.read(wav)
    assert sr == 24000 and x.shape == (3200,)


def _write_tokenizer(d):
    """A byte-level tokenizer with the Qwen2.5 special-token names the VibeVoice tokenizers resolve their ids from."""
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast
    vocab = {ch: i for i, ch in enumerate(sorted(pre_tokenizers.ByteLevel.alphabet()))}
    tk = Tokenizer(models.BPE(vocab=vocab, merges=[]))
    tk.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    tk.decoder = decoders.ByteLevel()
    specials = ["<|endoftext|>", "<|vision_start|>", "<|vision_end|>", "<|vision_pad|>", "<|image_pad|>"]
    PreTrainedTokenizerFast(tokenizer_object=tk, eos_token="<|endoftext|>", pad_token="<|image_pad|>",
                            additional_special_tokens=specials[1:]).save_pretrained(str(d))


def test_streaming_processor_from_pretrained_stays_offline(tmp_path, monkeypatch):
    from vibevoice.processor.vibevoice_streaming_processor import VibeVoiceStreamingProcessor as P
    monkeypatch.setenv("HF_HUB_OFFLINE", "1")
    monkeypatch.setenv("HF_HOME", str(tmp_path / "hf"))                 # an empty cache: nothing resolves from it
    ck = tmp_path / "ckpt"
    ck.mkdir()
    (ck / "preprocessor_config.json").write_text(json.dumps({"speech_tok_compress_ratio": 3200, "db_normalize": False,
                                                             "language_model_pretrained_name": "Qwen/Qwen2.5-0.5B"}))
    _write_tokenizer(ck)
    p = P.from_pretrained(str(ck))
    tok = p.tokenizer
    assert tok.pad_id == tok.convert_tokens_to_ids("<|image_pad|>") and tok.speech_start_id == tok.convert_tokens_to_ids("<|vision_start|>")
    assert p.db_normalize is False and p.audio_normalizer is None
    out = p.process_input_with_cached_prompt(text=" Hello ", cached_prompt=_preset(), return_tensors="pt")
    assert out["tts_text_ids"].tolist() == [tok.encode("Hello\n", add_special_tokens=False)]
    assert P.from_pretrained(str(tmp_path / "nowhere"), tokenizer=StubTokenizer()).tokenizer.pad_id == 3   # explicit tokenizer first
    bare = tmp_path / "bare"
    bare.mkdir()
    (bare / "preprocessor_config.json").write_text(json.dumps({"language_model_pretrained_name": "Qwen/Qwen2.5-0.5B"}))
    with pytest.raises(FileNotFoundError, match="tokenizer="):
        P.from_pretrained(str(bare))
    with pytest.raises(FileNotFoundError, match="tokenizer="):
        P.from_pretrained(str(tmp_path / "not-a-dir"))


def test_streaming_preset_fixture_loads_as_the_demo_loads_it(golden):
    meta = golden("streaming_processor")["preset"]
    p = torch.load(os.path.join(GOLDEN, "streaming_preset.pt"), map_location="cpu", weights_only=False)
    q = copy.deepcopy(p)
    from streaming_oracle import cache_layers
    assert meta["name"] == "en-Mike_man" and sorted(p) == ["lm", "neg_lm", "neg_tts_lm", "tts_lm"]
    for name, n_layers in (("lm", 4), ("tts_lm", 20), ("neg_lm", 4), ("neg_tts_lm", 20)):
        o = q[name]
        assert type(o).__name__ == "BaseModelOutputWithPast" and type(o.past_key_values).__name__ == "DynamicCache"
        assert hasattr(o.past_key_values, "key_cache")           # the transformers-4.x cache layout the shipped files carry
        kvs = cache_layers(o.past_key_values)
        n = meta["lengths"][name]
        assert len(kvs) == n_layers and o.last_hidden_state.shape == (1, n, 896) and o["last_hidden_state"] is o.last_hidden_state
        for (k, v), (k0, v0) in zip(kvs, cache_layers(p[name].past_key_values)):
            assert k.shape == v.shape == (1, 2, n, 64) and k.dtype == torch.bfloat16
            assert torch.equal(k, k0) and torch.equal(v, v0) and k.data_ptr() != k0.data_ptr()
    assert meta["lengths"]["lm"] != meta["lengths"]["tts_lm"]


def _prefilled(c):
    return {k: SimpleNamespace(past_key_values=tuple(v["kv"]), last_hidden_state=v["hidden"]) for k, v in c["prefilled"].items()}


@pytest.mark.parametrize("case", ["eos", "windows", "short"])
def test_oracle_from_prefilled_outputs_matches_the_reference(golden, case):
    """The fixtures carry the four prefilled outputs the reference's own streaming generate() started from."""
    from oracle import vv_streaming as VS
    from streaming_oracle import generate_from_prefilled
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.synth import synth_state_dict
    g = golden("streaming")
    c = g[case]
    cfg = preset_config(g["preset"])
    sd = VS.streaming_state_dict(synth_state_dict(cfg, 1234, torch.float32), cfg, g["tts_layers"], eos_bias=c["eos_bias"])
    torch.manual_seed(c["seed"])
    r = generate_from_prefilled(sd, cfg, g["tts_layers"], _prefilled(c), c["prompt"], c["text"], cfg_scale=c["cfg_scale"],
                                num_steps=g["num_steps"], max_new_tokens=c["max_new_tokens"])
    assert torch.equal(r.sequences, c["sequences"])
    assert torch.equal(r.reach_max_step_sample, c["reach_max"])
    a, b = r.speech_outputs[0], c["audio"]
    assert (a is None) == (b is None)
    if a is not None:
        assert a.shape == b.shape and float((a.double() - b.double()).norm() / b.double().norm()) < 5e-3


def _heads_engine_class():
    """The engine stand-in plus the native engine's streaming-head methods (`has_tts_heads`, `tts_type_embed`, `eos_prob`), with the oracle's
    arithmetic (`vv_streaming.eos_logit`, the fp32 add): the loop then takes the branch the native engine takes."""
    import fake_engine
    from oracle import vv_streaming as VS

    class HeadsFakeEngine(fake_engine.FakeEngine):
        calls_heads = 0

        @property
        def has_tts_heads(self) -> bool:
            return "model.tts_input_types.weight" in self.w and "tts_eos_classifier.fc1.weight" in self.w

        def tts_type_embed(self, src, type_id, rows, dst):
            HeadsFakeEngine.calls_heads += 1
            v = src.float() + self.w["model.tts_input_types.weight"].float()[type_id]
            for r in rows:
                dst[r] = v

        def eos_prob(self, hidden=None):
            HeadsFakeEngine.calls_heads += 1
            h = self.hidden[0] if hidden is None else hidden
            return torch.sigmoid(VS.eos_logit(self.w, h[None]))[0, 0].item()

    return HeadsFakeEngine


@pytest.mark.parametrize("engine", ["heads", "plain"])
@pytest.mark.parametrize("case", ["eos", "windows", "short"])
def test_streaming_host_loop_from_prefilled_matches_the_oracle(golden, monkeypatch, case, engine):
    """The product loop through an engine stand-in from the fixtures' prefilled outputs, once with the native engine's head methods
    ("heads": the loop's type embeddings and EOS classifier are engine calls) and once without them (the loop's own fp32 ops): the same
    sequences and flags as the oracle started from them, the same audio up to the fp32 rounding of running a text window token by token
    rather than as one block (1.4e-4 measured)."""
    import fake_engine
    from oracle import vv_streaming as VS
    from streaming_oracle import generate_from_prefilled
    from vibevoice_b200 import streaming as S
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.synth import synth_state_dict
    g = golden("streaming")
    c = g[case]
    cfg = preset_config(g["preset"])
    sd = VS.streaming_state_dict(synth_state_dict(cfg, 1234, torch.float32), cfg, g["tts_layers"], eos_bias=c["eos_bias"])
    m = S.VibeVoiceStreamingForConditionalGenerationInference(cfg, tts_backbone_num_hidden_layers=g["tts_layers"])
    E = _heads_engine_class() if engine == "heads" else fake_engine.FakeEngine
    monkeypatch.setattr(m, "_new_engine", lambda: E(cfg, [0, 1], 2))
    m.load_state_dict(sd)
    assert (m._host_heads is None) == (engine == "heads")
    m.set_ddpm_inference_steps(g["num_steps"])
    torch.manual_seed(c["seed"])
    out = m.generate(input_ids=c["prompt"][None], tts_lm_input_ids=c["prompt"][None], tts_text_ids=c["text"][None], neg_text_input_id=g["neg_id"],
                     cfg_scale=c["cfg_scale"], max_new_tokens=c["max_new_tokens"], all_prefilled_outputs=_prefilled(c))
    if engine == "heads":
        assert E.calls_heads > 0
    torch.manual_seed(c["seed"])
    ref = generate_from_prefilled(sd, cfg, g["tts_layers"], _prefilled(c), c["prompt"], c["text"], cfg_scale=c["cfg_scale"],
                                  num_steps=g["num_steps"], max_new_tokens=c["max_new_tokens"])
    assert torch.equal(out.sequences, ref.sequences) and torch.equal(out.sequences, c["sequences"])
    assert torch.equal(out.reach_max_step_sample, ref.reach_max_step_sample)
    a, b = out.speech_outputs[0], ref.speech_outputs[0]
    assert (a is None) == (b is None)
    if a is not None:
        assert a.shape == b.shape and float((a.double() - b.double()).norm() / b.double().norm()) < 1e-3


@pytest.mark.parametrize("engine", ["heads", "plain"])
def test_streaming_checkpoint_without_heads_is_refused(monkeypatch, engine):
    """The streaming loop needs the type embeddings and the EOS classifier: an engine with the head methods reports whether the checkpoint
    had them, and without those methods the loop checks the checkpoint itself."""
    import fake_engine
    from oracle import vv_streaming as VS
    from vibevoice_b200 import _native as N
    from vibevoice_b200 import streaming as S
    from vibevoice_b200.configuration import preset_config
    from vibevoice_b200.synth import synth_state_dict
    cfg = preset_config("tiny")
    sd = VS.streaming_state_dict(synth_state_dict(cfg, 1234, torch.float32), cfg, 1)
    sd = {k: v for k, v in sd.items() if not k.startswith("tts_eos_classifier.")}
    m = S.VibeVoiceStreamingForConditionalGenerationInference(cfg, tts_backbone_num_hidden_layers=1)
    E = _heads_engine_class() if engine == "heads" else fake_engine.FakeEngine
    monkeypatch.setattr(m, "_new_engine", lambda: E(cfg, [0, 1], 2))
    with pytest.raises(N.VVError, match="lacks"):
        m.load_state_dict(sd)
