"""Writes the streaming-0.5B demo fixtures from a reference checkout (VV_REFERENCE_ROOT, as for `oracle/make_golden.py`):

    VV_REFERENCE_ROOT=<reference checkout> python tools/make_streaming_golden.py

  tests/golden/streaming_preset.pt     the shipped voice preset `demo/voices/streaming_model/en-Mike_man.pt` (the smallest) with every
                                       stream cut to its first positions (CUT) and the pickled classes unchanged (BaseModelOutputWithPast
                                       holding a transformers-4.x DynamicCache): what `torch.load` returns in the streaming demo
  tests/golden/streaming_processor.pt  the reference's own VibeVoiceStreamingProcessor on the texts of tests/test_streaming_processor.py
                                       with the cut preset as `cached_prompt`; also records the preset's name and cut lengths

The tests only read the committed files; this script is the recipe that made them.
"""
from __future__ import annotations

import copy
import importlib.util
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from oracle.make_golden import GOLDEN_DIR  # noqa: E402

PRESET = "en-Mike_man"
CUT = {"lm": 24, "tts_lm": 48, "neg_lm": 1, "neg_tts_lm": 1}   # the text and TTS streams keep different lengths, as shipped


def cut_preset(preset):
    """Every K / V / hidden tensor cut to its first CUT[name] positions (cloned: a saved view would keep the whole storage)."""
    out = copy.deepcopy(preset)
    for name, n in CUT.items():
        o = out[name]
        o.last_hidden_state = o.last_hidden_state[:, :n].clone()
        c = o.past_key_values
        c.key_cache = [k[:, :, :n].clone() for k in c.key_cache]
        c.value_cache = [v[:, :, :n].clone() for v in c.value_cache]
        if hasattr(c, "_seen_tokens"):
            c._seen_tokens = n
    return out


def reference_processor_module():
    """The reference's vibevoice_streaming_processor.py, loaded from its file: this repository's drop-in `vibevoice` package shadows
    the reference's on sys.path."""
    base = os.path.join(ref_shim.REFERENCE_ROOT, "vibevoice", "processor")
    sys.modules.setdefault("refproc", types.ModuleType("refproc"))
    spec0 = importlib.util.spec_from_file_location("refproc.vibevoice_tokenizer_processor", os.path.join(base, "vibevoice_tokenizer_processor.py"))
    m0 = importlib.util.module_from_spec(spec0); sys.modules[spec0.name] = m0; spec0.loader.exec_module(m0)
    path = os.path.join(base, "vibevoice_streaming_processor.py")
    src = open(path).read().replace("from .vibevoice_tokenizer_processor", "from refproc.vibevoice_tokenizer_processor")
    mod = types.ModuleType("refproc.vibevoice_streaming_processor"); mod.__file__ = path
    exec(compile(src, path, "exec"), mod.__dict__)
    return mod


def main():
    if not ref_shim.reference_available():
        raise SystemExit("set VV_REFERENCE_ROOT to a reference checkout")
    ref_shim.load_reference()
    shipped = torch.load(os.path.join(ref_shim.REFERENCE_ROOT, "demo", "voices", "streaming_model", PRESET + ".pt"), map_location="cpu",
                         weights_only=False)
    preset = cut_preset(shipped)
    path = os.path.join(GOLDEN_DIR, "streaming_preset.pt")
    torch.save(preset, path)
    print("wrote", path, os.path.getsize(path), "bytes")

    spec = importlib.util.spec_from_file_location("vv_streaming_processor_inputs", os.path.join(ROOT, "tests", "test_streaming_processor.py"))
    tp = importlib.util.module_from_spec(spec); spec.loader.exec_module(tp)
    ref = reference_processor_module().VibeVoiceStreamingProcessor(tokenizer=tp.StubTokenizer(), audio_processor=None)
    cases = []
    for text, return_tensors, return_attention_mask in tp.CASES:
        enc = ref.process_input_with_cached_prompt(text=text, cached_prompt=preset, padding=True, return_tensors=return_tensors,
                                                   return_attention_mask=return_attention_mask)
        cases.append(dict(text=text, return_tensors=return_tensors, return_attention_mask=return_attention_mask, out=dict(enc)))
    data = dict(preset=dict(name=PRESET, lengths=dict(CUT)), cases=cases)
    path = os.path.join(GOLDEN_DIR, "streaming_processor.pt")
    torch.save(data, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
