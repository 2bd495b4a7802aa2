"""TEST INFRASTRUCTURE: the streaming oracle (`oracle/vv_streaming.generate_streaming`) started from `all_prefilled_outputs`, the cached
voice prompt format of the shipped presets (`demo/voices/streaming_model/*.pt`), instead of from prompt ids.

The four model outputs fill the oracle's `Streams`: each cache's per-layer K / V (keys stored rotated, as HF caches them) become the
lower-stack, TTS-LM and negative TTS-LM caches, and the last hidden states of the two TTS-LM outputs condition the first frame
(reference `modeling_vibevoice_streaming_inference.py:517-534`).  The loop itself is `generate_streaming`'s, unchanged: only its prompt
step is replaced, so the pinned oracle and what holds it to the reference stay as they are.
"""
from __future__ import annotations

from unittest import mock

import torch

from oracle import vv_streaming as VS


def cache_layers(cache):
    """[(k, v)] per layer, [1, kv_heads, L, head_dim] each, of a transformers-4.x DynamicCache (`key_cache` / `value_cache`, the shipped
    presets), a transformers-5.x cache (`layers`) or a tuple of (k, v) pairs."""
    if hasattr(cache, "key_cache"):
        return list(zip(cache.key_cache, cache.value_cache))
    if hasattr(cache, "layers"):
        return [(l.keys, l.values) for l in cache.layers if getattr(l, "keys", None) is not None]
    return [(kv[0], kv[1]) for kv in cache]


def _get(o, name):
    return o[name] if isinstance(o, dict) else getattr(o, name)


def fill_streams(st: VS.Streams, prefilled):
    for cache, name in ((st.lm, "lm"), (st.tts, "tts_lm"), (st.neg_tts, "neg_tts_lm")):
        kvs = cache_layers(_get(prefilled[name], "past_key_values"))
        if len(kvs) != len(cache.k):
            raise ValueError("%s has %d layers, expected %d" % (name, len(kvs), len(cache.k)))
        for j, (k, v) in enumerate(kvs):
            cache.preload(j, k[0].detach().float().cpu(), v[0].detach().float().cpu())
    st.h_pos = _get(prefilled["tts_lm"], "last_hidden_state")[0].detach().float().cpu()
    st.h_neg = _get(prefilled["neg_tts_lm"], "last_hidden_state")[0].detach().float().cpu()


def generate_from_prefilled(w, cfg, tts_layers: int, prefilled, tts_lm_input_ids: torch.Tensor, tts_text_ids: torch.Tensor,
                            cfg_scale: float = 1.5, num_steps: int = 5, max_new_tokens=None, kv_bf16: bool = False):
    """`generate_streaming` with the prompt state taken from `prefilled` (dict lm / tts_lm / neg_lm / neg_tts_lm of model outputs, or of
    dicts with `past_key_values` and `last_hidden_state`).  `tts_lm_input_ids` [L] is what `sequences` starts with and sets the length
    budget, as in the reference's generate()."""
    with mock.patch.object(VS, "prefill", lambda st, prompt_ids, neg_id: fill_streams(st, prefilled)):
        return VS.generate_streaming(w, cfg, tts_layers, tts_lm_input_ids.reshape(-1), tts_text_ids.reshape(-1), -1, cfg_scale=cfg_scale,
                                     num_steps=num_steps, max_new_tokens=max_new_tokens, kv_bf16=kv_bf16)
