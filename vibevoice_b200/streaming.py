"""Streaming-0.5B variant (SURVEY 8f-1): the reference's `VibeVoiceStreamingForConditionalGenerationInference`
(`vibevoice/modular/modeling_vibevoice_streaming_inference.py:95-762`) on the same engine as the multi-speaker model.

What differs from the multi-speaker loop (`modeling.py`), and how it maps onto the engine:
  * split LM (`modeling_vibevoice_streaming.py:134-146`): lower N-T layers = text-only stack without final norm, upper T layers = "TTS
    LM" with the final norm.  Both live in the engine's one layer array (lower first); `vv_lm_decode_range` runs one stack at a time.
    Each stack has its own KV sequences because their lengths differ (the upper stack also sees the speech positions):
        row 0 = TTS-LM positive stream, row 1 = lower text stack, row 2 = TTS-LM negative stream (max_batch = 2, row 3 unused);
    with `max_slots` = S > 1 the engine has max_batch = 2S and slot s uses rows s, S + s and 2S + s (`slot_rows`): the TTS-LM rows are
    the sampler's positive / negative pair (rows b and B + b), and the lower stack takes positive rows the sampler never activates;
  * every TTS-LM input gets a type embedding added (1 = text, 0 = speech; `:290-291`): `vv_tts_type_embed`;
  * no token selection: windows of 5 text tokens alternate with 6 speech frames (`:40-42, :568-614`); a binary classifier on the TTS-LM
    hidden state ends the utterance (`:691-696`): `vv_eos_prob`, whose result is the one host sync per speech frame;
  * no semantic tokenizer: the frame is sampler -> acoustic decoder -> acoustic connector (`:617-645`).  The engine is given zero
    semantic weights, for which its connector stage returns exactly `acoustic_connector(latent)` (RMSNorm(0) = 0), and the semantic
    encoder stage is simply never launched.
Batch size 1 per `generate()`, like the reference (`:511`); a multi-slot model runs it in slot 0, and `serving.StreamingRequestQueue`
serves up to `max_slots` requests at once.

The native `Engine` always runs the type embeddings and the EOS classifier on its sm_90a kernels (`vv_tts_type_embed`, `vv_eos_prob`),
and a checkpoint without their weights is refused.  An engine object that does not implement them (no `has_tts_heads`: the CPU
stand-in the host-logic tests drive this loop with, whose contract predates these kernels) gets the same two ops in fp32 PyTorch here.

STATUS: host logic held to fixtures from the reference's own streaming generate() on the CPU through the engine stand-in
(`tests/test_host_logic.py::test_streaming_product_host_logic_against_reference_fixture`); CUDA path vs the pinned oracle on the GPU
(`tests/test_gpu_parity.py::test_streaming_variant_vs_oracle`, sequences exact, audio 4e-6) and at the shipped 0.5B shapes (24 layers split
4 / 20, H = 896, 14 query / 2 KV heads, head_dim 64: `tests/test_gpu_scale.py::test_streaming_variant_real_05b_shapes_vs_oracle`); first-audio
latency harness: `python bench.py --model streaming-0.5b` (8 K cached prompt).
"""
from __future__ import annotations

from typing import Callable, Dict, Iterable, List, Optional, Tuple

import numpy as np
import torch

from . import _native as N
from .configuration import VibeVoiceConfig
from .engine import Engine
from .modeling import VibeVoiceGenerationOutput

TTS_TEXT_WINDOW_SIZE = 5      # :41
TTS_SPEECH_WINDOW_SIZE = 6    # :42
ROW_POS, ROW_TEXT, ROW_NEG = 0, 1, 2
LM, TTS = "model.language_model", "model.tts_language_model"
HEAD_NAMES = ("model.tts_input_types.weight", "tts_eos_classifier.fc1.weight", "tts_eos_classifier.fc1.bias", "tts_eos_classifier.fc2.weight",
              "tts_eos_classifier.fc2.bias")


def remap_streaming_state_dict(items: Iterable[Tuple[str, torch.Tensor]], config: VibeVoiceConfig, tts_layers: int):
    """Streaming checkpoint keys -> the engine's (multi-speaker) names; yields (name, tensor).  The streaming-only modules (type
    embeddings, EOS classifier) keep their names: the engine loads them as optional tensors."""
    low = config.decoder_config.num_hidden_layers - tts_layers
    for k, v in items:
        if k.startswith(TTS + ".layers."):
            parts = k.split(".")
            yield "%s.layers.%d.%s" % (LM, low + int(parts[3]), ".".join(parts[4:])), v
        elif k == TTS + ".norm.weight":
            yield LM + ".norm.weight", v
        elif k.startswith(TTS + ".embed_tokens") or k.startswith("model.acoustic_tokenizer.encoder") or "fix_std" in k:
            continue                                           # present in the checkpoint, unused by the loop (:139)
        else:
            yield k, v


class VibeVoiceStreamingForConditionalGenerationInference:
    def __init__(self, config: VibeVoiceConfig, tts_backbone_num_hidden_layers: int = 20, device: int = 0, max_diffusion_steps: int = 64,
                 max_slots: int = 1):
        """`max_slots` (1..4): requests the engine can hold at once (`serving.StreamingRequestQueue`); the engine has 2 * max_slots rows."""
        if not 1 <= int(max_slots) <= 4:
            raise ValueError("max_slots must be in [1, 4] (max_batch = 2 * max_slots <= 8), got %r" % (max_slots,))
        self.max_slots = int(max_slots)
        self.config = config
        self.tts_layers = int(tts_backbone_num_hidden_layers)
        self.low = config.decoder_config.num_hidden_layers - self.tts_layers
        if self.low < 1:
            raise ValueError("tts_backbone_num_hidden_layers must leave at least one lower layer")
        self._device_index, self._max_steps = device, max_diffusion_steps
        self.engine: Optional[Engine] = None
        self.ddpm_inference_steps = config.diffusion_head_config.ddpm_num_inference_steps
        self._host_heads: Optional[Dict[str, torch.Tensor]] = None   # only for engines without vv_tts_type_embed / vv_eos_prob

    def set_ddpm_inference_steps(self, num_steps=None):
        self.ddpm_inference_steps = num_steps or self.config.diffusion_head_config.ddpm_num_inference_steps

    @classmethod
    def from_pretrained(cls, path: str, torch_dtype=None, device_map=None, attn_implementation=None, **kw):
        """HF checkpoint directory (config.json of `VibeVoiceStreamingConfig` + *.safetensors), as
        `demo/streaming_inference_from_file.py:244-262` calls it.  `torch_dtype` / `attn_implementation` are accepted for drop-in
        compatibility (storage is bf16, attention is the built-in paged kernel); the split point comes from the config's
        `tts_backbone_num_hidden_layers` (`configuration_vibevoice_streaming.py:51, 90`)."""
        import glob
        import os
        from safetensors import safe_open
        cfg = VibeVoiceConfig.from_pretrained(path)
        dev = 0
        if isinstance(device_map, str) and device_map.startswith("cuda:"):
            dev = int(device_map.split(":")[1])
        elif device_map is not None and device_map not in ("cuda", "auto"):
            raise N.VVError("vibevoice_b200 runs on CUDA devices only (device_map=%r); there is no CPU path" % (device_map,))
        m = cls(cfg, tts_backbone_num_hidden_layers=int(getattr(cfg, "tts_backbone_num_hidden_layers", 20)), device=dev,
                max_diffusion_steps=int(kw.pop("max_diffusion_steps", 64)), max_slots=int(kw.pop("max_slots", 1)))
        files = sorted(glob.glob(os.path.join(path, "*.safetensors")))
        if not files:
            raise FileNotFoundError("no *.safetensors under %s" % path)

        def it():
            for f in files:
                with safe_open(f, framework="pt", device="cpu") as sf:
                    for k in sf.keys():
                        yield k, sf.get_tensor(k)
        m._attn_implementation = attn_implementation or "paged-split-kv"
        return m.load_state_dict(it())

    # the calls / attributes the demo touches between loading and generate() (`demo/streaming_inference_from_file.py:279-284`)
    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    @property
    def model(self):
        from types import SimpleNamespace
        return SimpleNamespace(language_model=SimpleNamespace(config=SimpleNamespace(
            _attn_implementation=getattr(self, "_attn_implementation", "paged-split-kv"))))

    def _new_engine(self):
        return Engine(self.config, [0, 1], 2 * self.max_slots, self._device_index, self._max_steps)   # no token constraint; ids are unused

    def slot_rows(self, slot: int) -> Tuple[int, int, int]:
        """(TTS-LM positive, lower text stack, TTS-LM negative) rows of `slot`; slot 0 of a one-slot model is (ROW_POS, ROW_TEXT, ROW_NEG)."""
        S = self.max_slots
        return slot, S + slot, 2 * S + slot

    def _mode(self, rows) -> List[int]:
        """row modes of `vv_set_row_mode` with exactly `rows` on"""
        return [1 if r in rows else 0 for r in range(4 * self.max_slots)]

    def load_state_dict(self, state_dict):
        eng = self.engine = self._new_engine()
        items = state_dict.items() if isinstance(state_dict, dict) else state_dict
        scale = bias = None
        seen_sem = False
        shapes: Dict[str, Tuple[torch.Size, torch.dtype]] = {}
        heads: Dict[str, torch.Tensor] = {}
        for name, t in remap_streaming_state_dict(items, self.config, self.tts_layers):
            if name == "model.speech_scaling_factor":
                scale = float(t)
            elif name == "model.speech_bias_factor":
                bias = float(t)
            elif name in HEAD_NAMES:
                heads[name] = t
            else:
                seen_sem |= name.startswith("model.semantic")
                eng.load_tensor(name, t)
        if not seen_sem:                                       # zero semantic encoder/connector: connector stage == acoustic connector only
            from .synth import param_specs
            for name, shape, _ in param_specs(self.config):
                if name.startswith("model.semantic"):
                    eng.load_tensor(name, torch.zeros(*shape, dtype=torch.bfloat16))
        native = hasattr(type(eng), "has_tts_heads")                # the engine implements the head kernels
        if native:
            for name, t in heads.items():
                eng.load_tensor(name, t)
        eng.finalize(scale, bias)
        if not (eng.has_tts_heads if native else len(heads) == len(HEAD_NAMES)):
            raise N.VVError("streaming checkpoint lacks model.tts_input_types / tts_eos_classifier")
        self._host_heads = None if native else {k: v.to(device=eng.device, dtype=torch.float32) for k, v in heads.items()}
        return self

    # ---- building blocks of the loop ----------------------------------------------------------------------------------
    def _lower_then_upper_text(self, token_ids: List[int], neg: bool = False):
        """One text token at a time: lower stack (row 1) -> upper stack (+ type 1) on the positive (or negative) TTS-LM row (:590-611)."""
        eng = self.engine
        pos, text, negr = self.slot_rows(0)
        up_row = negr if neg else pos
        for t in token_ids:
            toks = [0] * (4 * self.max_slots)
            toks[text] = int(t)
            eng.embed_tokens(toks, eng.embeds)
            eng.set_row_mode(self._mode([text]))
            eng.lm_decode_range(0, self.low, False)
            eng.kv_commit(self._mode([text]))
            self._type_embed(eng.hidden[text], 1, [up_row])
            eng.set_row_mode(self._mode([up_row]))
            eng.lm_decode_range(self.low, self.low + self.tts_layers, True)
            eng.kv_commit(self._mode([up_row]))

    def _speech_step(self, embed: torch.Tensor):
        """One TTS-LM step on both streams with the acoustic embedding (+ type 0) (:657-689)."""
        eng = self.engine
        pos, _, neg = self.slot_rows(0)
        self._type_embed(embed, 0, [pos, neg])
        eng.set_row_mode(self._mode([pos, neg]))
        eng.lm_decode_range(self.low, self.low + self.tts_layers, True)
        eng.kv_commit(self._mode([pos, neg]))

    def _type_embed(self, src: torch.Tensor, type_id: int, rows: List[int]):
        """`embeds[r] = src + tts_input_types[type_id]` for r in rows (:290-291); src may be one of those rows."""
        eng = self.engine
        if self._host_heads is None:
            eng.tts_type_embed(src, type_id, rows, eng.embeds)
            return
        with torch.cuda.stream(eng.stream):
            x = src + self._host_heads["model.tts_input_types.weight"][type_id]
            for r in rows:
                eng.embeds[r].copy_(x)

    def _eos_prob(self) -> float:
        """`sigmoid(tts_eos_classifier(h))` (:691; BinaryClassifier, modeling_vibevoice_streaming.py:42-53), one host sync."""
        eng = self.engine
        if self._host_heads is None:
            return eng.eos_prob(eng.hidden[ROW_POS])
        w = self._host_heads
        with torch.cuda.stream(eng.stream):
            x = torch.relu(w["tts_eos_classifier.fc1.weight"] @ eng.hidden[ROW_POS] + w["tts_eos_classifier.fc1.bias"])
            p = torch.sigmoid(w["tts_eos_classifier.fc2.weight"] @ x + w["tts_eos_classifier.fc2.bias"])
        eng.sync()
        return float(p[0])

    def _prefill_from_ids(self, input_ids: torch.Tensor, neg_id: int):
        """No cached prompt given: compute the four streams' prompt state through the decode kernels."""
        eng = self.engine
        _, text, neg = self.slot_rows(0)
        self._lower_then_upper_text([neg_id], neg=True)
        eng.kv_set_len(text, 0)                                # the negative text stack is not used again (:527-534 only keep its kwargs)
        with torch.cuda.stream(eng.stream):
            neg_hidden = eng.hidden[neg].clone()
        self._lower_then_upper_text(input_ids.tolist())
        with torch.cuda.stream(eng.stream):
            eng.hidden[neg].copy_(neg_hidden)                   # conditions of the first frame: last prompt position of both TTS-LM streams

    def _import_prefilled(self, outs, slot: int = 0):
        """`all_prefilled_outputs` (:517-534; the cached voice prompts of demo/streaming_inference_from_file.py:291 carry these four
        outputs): dict lm / tts_lm / neg_lm / neg_tts_lm of model outputs whose `past_key_values` expose per-layer key/value tensors
        [1, kv_heads, L, head_dim] (rotated keys, as HF caches them) and whose `last_hidden_state` is [1, L, H].  K/V go to the paged
        pool through `vv_kv_write`; the last hidden state of the two TTS-LM streams conditions the first frame."""
        eng = self.engine

        def layers_of(cache):
            if hasattr(cache, "key_cache"):                      # transformers 4.x DynamicCache
                return list(zip(cache.key_cache, cache.value_cache))
            if hasattr(cache, "layers"):                         # transformers 5.x
                return [(l.keys, l.values) for l in cache.layers if getattr(l, "keys", None) is not None]
            return [(kv[0], kv[1]) for kv in cache]              # legacy tuple-of-tuples

        def put(cache, seq: int, layer0: int, n_layers: int) -> int:
            kvs = layers_of(cache)
            if len(kvs) != n_layers:
                raise ValueError("prefilled cache has %d layers, expected %d" % (len(kvs), n_layers))
            L = int(kvs[0][0].shape[2])
            for j, (k, v) in enumerate(kvs):
                k = k[0].transpose(0, 1).to(device=eng.device, dtype=torch.bfloat16).contiguous()      # [L, kv_heads, head_dim]
                v = v[0].transpose(0, 1).to(device=eng.device, dtype=torch.bfloat16).contiguous()
                eng.kv_write(seq, layer0 + j, 0, k, v)
            eng.kv_set_len(seq, L)
            return L
        pos, text, neg = self.slot_rows(slot)
        put(outs["lm"].past_key_values, text, 0, self.low)
        put(outs["tts_lm"].past_key_values, pos, self.low, self.tts_layers)
        put(outs["neg_tts_lm"].past_key_values, neg, self.low, self.tts_layers)
        with torch.cuda.stream(eng.stream):
            eng.hidden[pos].copy_(outs["tts_lm"].last_hidden_state[0, -1].to(eng.device, torch.float32))
            eng.hidden[neg].copy_(outs["neg_tts_lm"].last_hidden_state[0, -1].to(eng.device, torch.float32))

    @torch.no_grad()
    def generate(self, inputs=None, tts_text_ids=None, cfg_scale: float = 1.0, audio_streamer=None, return_speech: bool = True,
                 stop_check_fn: Optional[Callable[[], bool]] = None, **kwargs) -> VibeVoiceGenerationOutput:
        """`:412-725`.  The prompt state comes from `all_prefilled_outputs` (the reference's cached-prompt format) when given, else it is
        computed from `input_ids` through the same decode kernels; the negative streams start from the single token `<|image_pad|>`
        (`:465, :475-482`)."""
        tokenizer = kwargs.pop("tokenizer", None)
        neg_id = kwargs.pop("neg_text_input_id", None)
        neg_id = int(tokenizer.convert_tokens_to_ids("<|image_pad|>") if neg_id is None else neg_id)           # :465
        input_ids = torch.as_tensor(kwargs["input_ids"] if "input_ids" in kwargs else inputs).cpu().long()
        if input_ids.dim() == 2:
            if input_ids.shape[0] != 1:
                raise ValueError("Currently only supports batch size == 1")                       # :511
            input_ids = input_ids[0]
        tts_ids = kwargs.pop("tts_lm_input_ids", None)          # the TTS-LM's view of the prompt (:468); equals input_ids for text prompts
        tts_ids = input_ids if tts_ids is None else torch.as_tensor(tts_ids).cpu().long().reshape(-1)
        kwargs.pop("tts_lm_attention_mask", None)
        text = torch.as_tensor(tts_text_ids).cpu().long().reshape(-1)
        eng = self.engine
        dc = self.config.decoder_config
        L0 = int(tts_ids.numel())
        if kwargs.get("max_new_tokens", None) is None:
            kwargs["max_new_tokens"] = dc.max_position_embeddings - L0                              # :472-473
        max_length = L0 + int(kwargs["max_new_tokens"])
        if eng.kv_pages == 0:
            eng.kv_init(4 * (max_length + 8))
        eng.set_diffusion_steps(int(self.ddpm_inference_steps))
        eng.codec_state_reset()
        for s in range(4 * self.max_slots):
            eng.kv_set_len(s, 0)
        # ---- prefill: what `all_prefilled_outputs` carries (lm / tts_lm and their negatives) ----
        prefilled = kwargs.pop("all_prefilled_outputs", None)
        if prefilled is not None:
            self._import_prefilled(prefilled)
        else:
            self._prefill_from_ids(input_ids, neg_id)

        neg_row = self.slot_rows(0)[2]
        seq: List[int] = tts_ids.tolist()
        chunks: List[torch.Tensor] = []
        finished, reach_max, win = False, False, 0
        vae = self.config.acoustic_vae_dim
        while True:
            if stop_check_fn is not None and stop_check_fn():                                       # :555-561
                if audio_streamer is not None:
                    audio_streamer.end()
                break
            if finished:                                                                           # :563-566
                break
            cur = text[win * TTS_TEXT_WINDOW_SIZE:(win + 1) * TTS_TEXT_WINDOW_SIZE]                  # :568-570
            win += 1
            if cur.numel() > 0:
                seq += cur.tolist()
                if len(seq) > max_length:                                                          # :576-582
                    reach_max = True
                    break
                with torch.cuda.stream(eng.stream):
                    neg_hidden = eng.hidden[neg_row].clone()
                self._lower_then_upper_text(cur.tolist())                                          # :590-611
                with torch.cuda.stream(eng.stream):
                    eng.hidden[neg_row].copy_(neg_hidden)       # the text window does not touch the negative stream
            for _ in range(TTS_SPEECH_WINDOW_SIZE):                                                # :614
                noise = torch.randn(2, vae)[:1]                                                    # :741, CPU global generator
                eng.upload_frame_inputs(noise, [0])
                eng.diffusion_sample(cfg_scale)                                                    # :617-621 (rows 0 and B + 0)
                eng.codec_decode()                                                                 # :624-632
                with torch.cuda.stream(eng.stream):
                    chunk = eng.audio[0:1].clone()
                if not finished:                                                                   # :634-638
                    chunks.append(chunk)
                if audio_streamer is not None:                                                     # :641-643
                    eng.sync()
                    audio_streamer.put(chunk.unsqueeze(1), torch.tensor([0]))
                with torch.cuda.stream(eng.stream):
                    eng.feat.zero_()
                eng.connect()                                                                      # :645 -> eng.embeds[0] (and [B])
                seq.append(1)                                                                      # :646
                if len(seq) > max_length:                                                          # :648-649
                    break
                self._speech_step(eng.embeds[ROW_POS])
                if self._eos_prob() > 0.5:                                                         # :691-696
                    finished = True
                    if audio_streamer is not None:
                        audio_streamer.end(torch.tensor([0]))
            if len(seq) > max_length:                                                              # :698-704
                reach_max = not finished
                break
        if audio_streamer is not None:
            audio_streamer.end()
        eng.sync()
        with torch.cuda.stream(eng.stream):
            out = torch.cat(chunks, dim=-1) if chunks else None
        eng.sync()
        return VibeVoiceGenerationOutput(sequences=torch.tensor([seq], dtype=torch.long), speech_outputs=[out] if return_speech else None,
                                         reach_max_step_sample=torch.tensor([reach_max]))
