"""TEST INFRASTRUCTURE ONLY -- compatibility shim that lets the *unmodified* reference
arithmetic modules of a reference checkout (VV_REFERENCE_ROOT) import here (transformers 5.5.0, no
`diffusers`).  It is used by `oracle/make_golden.py` (golden-vector generation) only; nothing in the
product path, `bench.py` or the tests may import it (they run without a reference checkout).

What it patches (all outside the reference tree, nothing is copied from it):
  * fake `diffusers` package providing the five names `vibevoice/schedule/dpm_solver.py:23-26`
    imports (ConfigMixin, register_to_config, SchedulerMixin, SchedulerOutput,
    KarrasDiffusionSchedulers, deprecate, randn_tensor);
  * `AutoModel.register` forced to `exist_ok=True` (transformers 5.5.0 ships its own
    `vibevoice_acoustic_tokenizer` model type, `modular_vibevoice_tokenizer.py:1188` collides);
  * alias for the removed `transformers.models.qwen2.tokenization_qwen2_fast`
    (`modular_vibevoice_text_tokenizer.py:7`).
"""
from __future__ import annotations

import functools
import inspect
import os
import sys
import types
from dataclasses import dataclass

REFERENCE_ROOT = os.environ.get("VV_REFERENCE_ROOT", "")      # a checkout of vibevoice-community/VibeVoice


def reference_available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "vibevoice", "modular"))


def _install_fake_diffusers():
    if "diffusers" in sys.modules:
        return
    import torch

    class _Cfg(dict):
        def __getattr__(self, k):
            try:
                return self[k]
            except KeyError as e:  # pragma: no cover
                raise AttributeError(k) from e

    class ConfigMixin:
        config_name = None

        def register_to_config(self, **kw):
            if not hasattr(self, "_internal_dict"):
                self._internal_dict = _Cfg()
            self._internal_dict.update(kw)

        @property
        def config(self):
            return self._internal_dict

        @classmethod
        def from_config(cls, config, **kw):
            d = dict(config)
            d.update(kw)
            sig = inspect.signature(cls.__init__)
            return cls(**{k: v for k, v in d.items() if k in sig.parameters})

    def register_to_config(init):
        @functools.wraps(init)
        def wrapper(self, *args, **kwargs):
            sig = inspect.signature(init)
            bound = sig.bind(self, *args, **kwargs)
            bound.apply_defaults()
            cfg = {k: v for k, v in bound.arguments.items() if k != "self"}
            ConfigMixin.register_to_config(self, **cfg)
            init(self, *args, **kwargs)

        return wrapper

    class SchedulerMixin:
        pass

    @dataclass
    class SchedulerOutput:
        prev_sample: "torch.Tensor"

    import enum

    class KarrasDiffusionSchedulers(enum.Enum):
        DPMSolverMultistepScheduler = 1

    def deprecate(*a, **k):
        return None

    def randn_tensor(shape, generator=None, device=None, dtype=None, layout=None):
        return torch.randn(shape, generator=generator, dtype=dtype).to(device)

    pkg = types.ModuleType("diffusers")
    cu = types.ModuleType("diffusers.configuration_utils")
    cu.ConfigMixin, cu.register_to_config = ConfigMixin, register_to_config
    ut = types.ModuleType("diffusers.utils")
    ut.deprecate = deprecate
    tu = types.ModuleType("diffusers.utils.torch_utils")
    tu.randn_tensor = randn_tensor
    sch = types.ModuleType("diffusers.schedulers")
    su = types.ModuleType("diffusers.schedulers.scheduling_utils")
    su.KarrasDiffusionSchedulers = KarrasDiffusionSchedulers
    su.SchedulerMixin, su.SchedulerOutput = SchedulerMixin, SchedulerOutput
    pkg.configuration_utils, pkg.utils, pkg.schedulers = cu, ut, sch
    ut.torch_utils, sch.scheduling_utils = tu, su
    for m in (pkg, cu, ut, tu, sch, su):
        sys.modules[m.__name__] = m


def _patch_transformers():
    from transformers.models.auto import auto_factory

    orig = auto_factory._LazyAutoMapping.register
    if not getattr(orig, "_vv_patched", False):

        def register(self, key, value, exist_ok=False):
            return orig(self, key, value, exist_ok=True)

        register._vv_patched = True
        auto_factory._LazyAutoMapping.register = register

    name = "transformers.models.qwen2.tokenization_qwen2_fast"
    if name not in sys.modules:
        try:
            from transformers.models.qwen2 import tokenization_qwen2 as tq

            mod = types.ModuleType(name)
            fast = getattr(tq, "Qwen2TokenizerFast", None) or getattr(tq, "Qwen2Tokenizer")
            mod.Qwen2TokenizerFast = fast
            sys.modules[name] = mod
        except Exception:  # pragma: no cover
            pass


_LOADED = {}


def load_reference():
    """Import the reference arithmetic modules; returns a namespace of the symbols the oracle
    is pinned against.  Raises RuntimeError when the reference checkout is absent."""
    if _LOADED:
        return _LOADED["ns"]
    if not reference_available():
        raise RuntimeError("reference tree not present at %s" % REFERENCE_ROOT)
    _install_fake_diffusers()
    _patch_transformers()
    # this repo ships a drop-in `vibevoice/` alias package; make sure the names below resolve to the REFERENCE tree
    for name in [n for n in sys.modules if n == "vibevoice" or n.startswith("vibevoice.")]:
        f = getattr(sys.modules[name], "__file__", "") or ""
        if not f.startswith(REFERENCE_ROOT):
            del sys.modules[name]
    if REFERENCE_ROOT in sys.path:
        sys.path.remove(REFERENCE_ROOT)
    sys.path.insert(0, REFERENCE_ROOT)
    import importlib

    cfg = importlib.import_module("vibevoice.modular.configuration_vibevoice")
    head = importlib.import_module("vibevoice.modular.modular_vibevoice_diffusion_head")
    tok = importlib.import_module("vibevoice.modular.modular_vibevoice_tokenizer")
    dpm = importlib.import_module("vibevoice.schedule.dpm_solver")
    ns = types.SimpleNamespace(cfg=cfg, head=head, tok=tok, dpm=dpm)
    try:
        ns.modeling = importlib.import_module("vibevoice.modular.modeling_vibevoice")
    except Exception as e:  # pragma: no cover - only the connector lives here
        ns.modeling = None
        ns.modeling_error = repr(e)
    _LOADED["ns"] = ns
    return ns


# ---------------------------------------------------------------------------------------------------------------------
# Running the reference's OWN generate() loop (modeling_vibevoice_inference.py:326-695) in this container.
#
# The loop body is the reference's, unmodified.  What does not survive the installed transformers 5.5.0 is the glue it borrows
# from `transformers.generation.GenerationMixin` -- private API of transformers 4.51.3, the version the reference pins
# (`pyproject.toml:20`).  That third-party glue is absent here, so its published 4.51.3 behaviour is restated below, and the few
# private-signature changes are adapted.  Nothing of the reference is copied or edited; the patches are applied to the imported
# class object at run time, and only `oracle/make_golden.py` uses them.
#
#   * `_prepare_generation_config(gc, use_model_defaults, **kw)`      -> 5.5.0 dropped the positional flag (inference.py:269-276)
#   * `_prepare_cache_for_generation(gc, kw, assistant, B, maxlen, device)` -> a DynamicCache that still exposes the
#     `.key_cache` / `.value_cache` lists the loop edits in place (inference.py:556-561, 609-616)
#   * `_update_model_kwargs_for_generation` (4.51.3): past <- outputs.past_key_values; attention_mask gets one column of
#     ones; cache_position <- cache_position[-1:] + 1                                                    (inference.py:483, 513, 586)
#   * `prepare_inputs_for_generation` (4.51.3): with a cache, keep only the unprocessed tail of input_ids
#     (`input_ids[:, -len(cache_position):]` once cache_position has run past the ids, else `input_ids[:, cache_position]`);
#     `inputs_embeds` are used only when they cover exactly the positions in cache_position; position_ids =
#     cumsum(attention_mask) - 1 (1 where masked), cut to the current input length               (inference.py:466, 504, 577)
#   * `tie_weights(**kw)`: 5.5.0 passes `recompute_mapping=`; the reference's override takes no arguments (inference.py:113-131)
#
# `script_tokens(...)`: BASELINE.md section 3 scripts "diffusion x F, then EOS"; generate() discards a caller-supplied
# `logits_processor` (inference.py:375-377 overwrite it), so the script is injected where the reference itself constrains the
# scores -- after `VibeVoiceTokenConstraintProcessor.__call__` (inference.py:53-66) the scripted id is raised to +inf.
# ---------------------------------------------------------------------------------------------------------------------
_SCRIPT = {}


def script_tokens(initial_length=None, tokens=None):
    """Install (or clear, with no arguments) a per-row token script for the next reference generate() call."""
    _SCRIPT.clear()
    if tokens is not None:
        _SCRIPT.update(L0=int(initial_length), tokens=[list(t) for t in tokens])


def _legacy_cache_class():
    from transformers.cache_utils import DynamicCache

    class LegacyListCache(DynamicCache):
        @property
        def key_cache(self):
            return [layer.keys for layer in self.layers]

        @property
        def value_cache(self):
            return [layer.values for layer in self.layers]

    return LegacyListCache


def _patch_generation_class(cls, cache_config_of):
    """transformers-4.51.3 GenerationMixin glue (see the block comment above) installed on one reference inference class."""
    import torch

    if getattr(cls, "_vv_compat", False):
        return
    LegacyListCache = _legacy_cache_class()
    orig_tie = cls.tie_weights
    cls.tie_weights = lambda self, *a, **k: orig_tie(self)
    orig_pgc = cls._prepare_generation_config
    cls._prepare_generation_config = lambda self, gc, *flags, **kw: orig_pgc(self, gc, **kw)

    def prepare_cache(self, generation_config, model_kwargs, assistant_model, batch_size, max_cache_length, device=None):
        model_kwargs["past_key_values"] = LegacyListCache(config=cache_config_of(self))

    def update_kwargs(self, outputs, model_kwargs, is_encoder_decoder=False, num_new_tokens=1):
        model_kwargs["past_key_values"] = outputs.past_key_values
        am = model_kwargs["attention_mask"]
        model_kwargs["attention_mask"] = torch.cat([am, am.new_ones((am.shape[0], 1))], dim=-1)
        model_kwargs["cache_position"] = model_kwargs["cache_position"][-1:] + num_new_tokens
        return model_kwargs

    def prepare_inputs(self, input_ids, past_key_values=None, attention_mask=None, inputs_embeds=None, cache_position=None, **kwargs):
        mi = {"cache_position": cache_position}
        if past_key_values is not None:
            mi["past_key_values"] = past_key_values
            if inputs_embeds is not None and input_ids.shape[1] == 0:
                inputs_embeds = inputs_embeds[:, -cache_position.shape[0]:]
            elif inputs_embeds is not None or cache_position[-1] >= input_ids.shape[1]:
                input_ids = input_ids[:, -cache_position.shape[0]:]
            elif input_ids.shape[1] != cache_position.shape[0]:
                input_ids = input_ids[:, cache_position]
        if inputs_embeds is not None and len(cache_position) == inputs_embeds.shape[1]:
            mi["input_ids"], mi["inputs_embeds"] = None, inputs_embeds
        else:
            mi["input_ids"], mi["inputs_embeds"] = input_ids.clone(memory_format=torch.contiguous_format), None
        position_ids = kwargs.pop("position_ids", None)
        if attention_mask is not None and position_ids is None:
            position_ids = attention_mask.long().cumsum(-1) - 1
            position_ids.masked_fill_(attention_mask == 0, 1)
        if position_ids is not None:
            cur = mi["inputs_embeds"].shape[1] if mi["inputs_embeds"] is not None else mi["input_ids"].shape[1]
            mi["position_ids"] = position_ids[:, -cur:].clone(memory_format=torch.contiguous_format)
        if attention_mask is not None:
            mi["attention_mask"] = attention_mask
        for k, v in kwargs.items():
            mi.setdefault(k, v)
        mi.pop("labels", None)
        return mi

    cls._prepare_cache_for_generation = prepare_cache
    cls._update_model_kwargs_for_generation = update_kwargs
    cls.prepare_inputs_for_generation = prepare_inputs
    cls._vv_compat = True


def install_generate_compat():
    """Patch the imported reference inference class so that its generate() runs under transformers 5.5.0 (see above)."""
    load_reference()
    import importlib
    infer_mod = importlib.import_module("vibevoice.modular.modeling_vibevoice_inference")
    cls = infer_mod.VibeVoiceForConditionalGenerationInference
    if getattr(cls, "_vv_compat", False):
        return infer_mod
    _patch_generation_class(cls, lambda self: self.config.decoder_config)

    proc = infer_mod.VibeVoiceTokenConstraintProcessor
    orig_call = proc.__call__

    def constrained_then_scripted(self, input_ids, scores):
        scores = orig_call(self, input_ids, scores)
        if _SCRIPT:
            step = input_ids.shape[1] - _SCRIPT["L0"]
            for b, s in enumerate(_SCRIPT["tokens"]):
                scores[b, s[min(step, len(s) - 1)]] = float("inf")
        return scores

    proc.__call__ = constrained_then_scripted
    return infer_mod


def install_streaming_generate_compat():
    """Same glue for the streaming-0.5B inference class (modeling_vibevoice_streaming_inference.py:95-762).  Its four KV streams
    (lm / tts_lm and their negatives) are created by `_prepare_cache_for_generation` with no layer count of their own; the caller
    replaces them with the prefilled caches (`all_prefilled_outputs`, :517-534) before any forward, so an empty legacy-list cache
    is all that is needed here."""
    load_reference()
    import importlib
    mod = importlib.import_module("vibevoice.modular.modeling_vibevoice_streaming_inference")
    _patch_generation_class(mod.VibeVoiceStreamingForConditionalGenerationInference, lambda self: self.config.decoder_config)
    return mod


def legacy_cache(config):
    """An empty transformers-5.5.0 DynamicCache that also exposes the 4.x `.key_cache` / `.value_cache` lists."""
    return _legacy_cache_class()(config=config)
