"""`VibeVoiceForConditionalGenerationInference` -- the reference's public generation surface
(`vibevoice/modular/modeling_vibevoice_inference.py:68-717`) on top of the H100 engine.

Same constructor / `from_pretrained` / `set_ddpm_inference_steps` / `generate(**kwargs)` contract and the
same `VibeVoiceGenerationOutput`, so `demo/inference_from_file.py:280-431` runs against this class.  The loop
body keeps the reference's integer/boolean bookkeeping on the host, verbatim in meaning
(`:432-675`), and replaces every tensor op by one of five C-ABI calls:

    self(**model_inputs)            :480-482   -> Engine.lm_decode   (positive + negative rows, one weight pass)
    negative forward + KV shifting  :576-624   -> same call; vv_kv_commit advances the negative stream only on diffusion tokens
    sample_speech_tokens            :629-633 \\
    acoustic_tokenizer.decode       :637-643  |-> Engine.frame_tail (one captured CUDA graph)
    semantic_tokenizer.encode       :658-664  |
    connectors                      :667-672 /
"""
from __future__ import annotations

import glob
import json
import os
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Callable, Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _native as N
from .configuration import VibeVoiceConfig
from .engine import Engine


@dataclass
class VibeVoiceGenerationOutput:
    """`modeling_vibevoice_inference.py:38-51`."""
    sequences: torch.LongTensor = None
    speech_outputs: Optional[List[Optional[torch.Tensor]]] = None
    reach_max_step_sample: Optional[torch.BoolTensor] = None


class VoicePreset:
    """A voice prompt prefix (`system prompt + " Voice input:\\n" + speakers`) encoded once by `model.voice_preset()`.

    Holds the prefix ids [Lp], its embeddings [Lp, H] fp32 on the device (token rows with the connected voice frames in place), the voice
    noise it drew (`noise`, the `_voice_noise` a full-prompt `generate()` takes to reproduce it) and `shared = 64 * (Lp // 64)`: the
    positions whose K/V live in shared pages of the KV pool.  The first request that uses the preset after a pool (re)initialisation
    prefills them into its own sequence and makes them a prefix (`vv_kv_prefix_create`); later requests attach that prefix and prefill
    only from `shared` on.  `release()` gives the pages back; the next use builds them again."""

    def __init__(self, model, ids: torch.Tensor, embeds: torch.Tensor, noise):
        self.model, self.ids, self.embeds, self.noise = model, ids, embeds, noise
        self.shared = ids.numel() // 64 * 64
        self._eng, self._epoch, self._handle = None, -1, None

    @property
    def pages(self) -> int:
        return self.shared // 64

    def resident(self) -> bool:
        """whether the shared pages are in the model's current KV pool."""
        eng = self.model.engine
        return (self._handle is not None and eng is self._eng and eng.kv_epoch == self._epoch
                and eng.kv_prefix_tokens(self._handle) == self.shared)

    def _attach(self, seq: int) -> bool:
        if not self.resident():
            return False
        self._eng.kv_prefix_attach(self._handle, seq)
        return True

    def _adopt(self, seq: int):
        """the first `shared` positions of `seq` (prefilled from `embeds`) become the preset's pages."""
        eng = self.model.engine
        self._handle, self._eng, self._epoch = eng.kv_prefix_create(seq, self.shared), eng, eng.kv_epoch

    def release(self):
        """Give the shared pages back to the pool (sequences attached to them keep them until they are reset)."""
        if self.resident():
            self._eng.kv_prefix_release(self._handle)
        self._handle = self._eng = None


class ForcedTokenScript:
    """Accepted as (an element of) `logits_processor`: per-row token scripts that override the constrained argmax,
    e.g. "speech_diffusion x F then EOS" (BASELINE.md section 3).  The reference achieves the same with a
    `LogitsProcessor` that adds +inf to the wanted id; full-vocab logits do not exist on this path (only the
    4-5 ids that survive `VibeVoiceTokenConstraintProcessor`, :53-66, are ever computed)."""

    def __init__(self, scripts: Sequence[Sequence[int]]):
        self.scripts = [list(s) for s in scripts]

    def token(self, row: int, step: int) -> int:
        s = self.scripts[row]
        return s[min(step, len(s) - 1)]


def sample_valid_tokens(logits_valid, valid_ids, generator=None) -> np.ndarray:
    """Multinomial draw of the next token (reference modeling_vibevoice_inference.py:493-496, `do_sample=True`).

    The reference softmaxes the full-vocab scores after `VibeVoiceTokenConstraintProcessor` set every id outside the valid set to
    -inf (:55-66), so the distribution has support on the valid ids only; softmax over just those logits is the same distribution.
    `logits_valid` is [rows, n_valid] fp32 in `valid_ids` order.  The draw uses its own generator so that the CPU global RNG, which the
    reference consumes for the diffusion noise only (:701), sees the same sequence of calls in both modes."""
    lv = torch.as_tensor(np.asarray(logits_valid), dtype=torch.float32)
    probs = torch.softmax(lv, dim=-1)
    idx = torch.multinomial(probs, num_samples=1, generator=generator).squeeze(1)
    return np.asarray(valid_ids, dtype=np.int64)[idx.numpy()]


class _NegativeSlots:
    """Integer bookkeeping of ONE row of the CFG-negative stream when `refresh_negative=False`, exactly as the reference keeps it
    (modeling_vibevoice_inference.py:503-517, 594-624): a cache that only grows, an attention mask with one extra column for the incoming
    token, and an "undo" of non-diffusing rows done by shifting mask and cache one slot to the right from `correct_cnt`.  The two shift
    guards differ by one (:603 uses the mask length, :613 the cache length), so when the cache holds exactly correct_cnt + 2 entries the
    mask moves and the cache does not: the entry at `correct_cnt` is hidden for good and the NEWEST entry stays.  The paged pool holds the
    visible entries only (attention does not care about their order), so that case is one `vv_kv_delete_slot`."""

    def __init__(self):
        self.slots: List[int] = []          # physical slot -> entry id
        self.mask: List[int] = [1]          # len(slots) + 1 columns
        self.correct_cnt = 0
        self.n = 0

    def append(self) -> int:
        e = self.n
        self.n += 1
        self.slots.append(e)
        self.mask.append(1)
        return e

    def correct(self):
        s, n, L = self.correct_cnt, len(self.slots), len(self.mask)
        if s + 1 < L - 1:
            self.mask[s + 1:] = self.mask[s:-1]
        self.mask[s] = 0
        if s + 1 < n - 1:
            self.slots[s + 1:] = self.slots[s:-1]
        self.correct_cnt += 1

    def visible(self) -> List[int]:
        return [self.slots[i] for i in range(len(self.slots)) if self.mask[i]]


class WeightModule:
    """Stand-in for an `nn.Module` of the reference's module tree whose parameters live, packed, inside the engine:
    `model.model.prediction_head`, `.acoustic_connector`, `.semantic_connector`.  The reference's fine-tuning loader only ever calls
    `load_state_dict(sd, strict=False)` and `.to(device)` on them (`lora_loading.py:57-66, 104-112, 163-169`); both work here --
    a loaded state dict is folded into the checkpoint stream and the engine re-packs its weights.  PEFT wrapping (`PeftModel.from_pretrained`
    on these objects, lora_loading.py:88-91, 129-137) needs real `nn.Linear` modules and is served by `lora.load_lora_assets` instead,
    which merges the adapter pairs into the base matrices."""

    def __init__(self, owner: "VibeVoiceForConditionalGenerationInference", prefix: str):
        self._owner, self._prefix = owner, prefix

    def load_state_dict(self, state_dict, strict: bool = True):
        repl = {self._prefix + k: v for k, v in state_dict.items()}
        known = set(self._owner._tensor_names(self._prefix))
        unexpected = sorted(k[len(self._prefix):] for k in repl if k not in known)
        missing = sorted(k[len(self._prefix):] for k in known if k not in repl)
        if strict and (missing or unexpected):
            raise RuntimeError("Error(s) in loading state_dict: missing %s, unexpected %s" % (missing, unexpected))
        repl = {k: v for k, v in repl.items() if k in known}

        def transform(items):
            for name, t in items:
                yield name, (repl[name] if name in repl else t)
        self._owner._reload_with(transform)
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    def state_dict(self):
        return {k[len(self._prefix):]: v for k, v in self._owner._weights_source() if k.startswith(self._prefix)}

    def to(self, *a, **k):
        return self

    def eval(self):
        return self

    def parameters(self):
        return iter(())


class VibeVoiceForConditionalGenerationInference:
    def __init__(self, config: VibeVoiceConfig, tokenizer_ids=None, max_batch: int = 1, device: int = 0,
                 max_diffusion_steps: int = 64, torch_prefill: bool = False, prefill_impl: Optional[str] = None):
        if prefill_impl not in (None, "native"):
            raise ValueError("prefill_impl=%r: the model-level default can only be \"native\" (or None)" % (prefill_impl,))
        self.config = config
        self._prefill_impl = prefill_impl        # "native": generate() prefills prompts with vv_lm_prefill unless told otherwise
        self._torch_prefill = torch_prefill      # keep bf16 LM weights for the PyTorch prompt prefill (prefill.py)
        self._prefill = None
        self._lm_sd: Dict[str, torch.Tensor] = {}
        self._voice = None                       # voice-prompt encoder (a-9), set when the checkpoint has the acoustic encoder
        self._scale = self._bias = None
        self._tok = tokenizer_ids
        self._device_index = device
        self._max_batch = max_batch
        self._max_steps = max_diffusion_steps
        self.engine: Optional[Engine] = None
        self._pending: List[Tuple[str, torch.Tensor]] = []
        self._weights_source = None              # callable -> fresh (name, tensor) iterator, for adapter re-packing (lora.py)
        self.ddpm_inference_steps = config.diffusion_head_config.ddpm_num_inference_steps
        self.dtype = torch.bfloat16
        self._kv_tokens = 0
        # attribute surface other reference code pokes at (demo/inference_from_file.py:367-368, gradio_demo.py:142-146)
        self.model = SimpleNamespace(
            language_model=SimpleNamespace(config=config.decoder_config),
            noise_scheduler=None,
            prediction_head=WeightModule(self, "model.prediction_head."),
            acoustic_connector=WeightModule(self, "model.acoustic_connector."),
            semantic_connector=WeightModule(self, "model.semantic_connector."),
            speech_scaling_factor=torch.tensor(float("nan")), speech_bias_factor=torch.tensor(float("nan")))
        if not hasattr(config.decoder_config, "_attn_implementation"):
            try:
                config.decoder_config._attn_implementation = "b200_paged_split_kv"     # read at demo/inference_from_file.py:367-368
            except Exception:
                pass

    # ---- construction ---------------------------------------------------------------------------------
    def _ensure_engine(self, valid_ids):
        if self.engine is None:
            self.engine = Engine(self.config, valid_ids, self._max_batch, self._device_index, self._max_steps)
            self.model.noise_scheduler = self.engine.scheduler
        return self.engine

    def _tensor_names(self, prefix: str) -> List[str]:
        from .synth import param_specs
        return [n for n, _, _ in param_specs(self.config) if n.startswith(prefix)]

    def parameters(self):
        """`next(model.parameters()).device` is how the reference's adapter loader finds the device (lora_loading.py:160)."""
        yield torch.empty(0, dtype=self.dtype, device=self.device)

    @staticmethod
    def _valid_ids(tok) -> List[int]:
        v = [tok.speech_start_id, tok.speech_end_id, tok.speech_diffusion_id, tok.eos_token_id]   # :405-413
        if getattr(tok, "bos_token_id", None) is not None:
            v.append(tok.bos_token_id)
        return sorted(set(int(x) for x in v))

    def load_state_dict(self, state_dict, tokenizer_ids=None, strict: bool = True):
        """Same keys as the reference module tree (`modeling_vibevoice.py:119-142`)."""
        tok = tokenizer_ids or self._tok
        if tok is None:
            raise ValueError("tokenizer ids (speech_start/end/diffusion/eos) are needed before weights are packed")
        self._tok = tok
        eng = self._ensure_engine(self._valid_ids(tok))
        if isinstance(state_dict, dict):
            self._weights_source = lambda sd=state_dict: iter(sd.items())
        items = state_dict.items() if isinstance(state_dict, dict) else state_dict
        scale = bias = None
        has_encoder = False
        for name, t in items:
            if name == "model.speech_scaling_factor":
                scale = float(t); self.model.speech_scaling_factor = torch.tensor(scale)
            elif name == "model.speech_bias_factor":
                bias = float(t); self.model.speech_bias_factor = torch.tensor(bias)
            else:
                eng.load_tensor(name, t)
                has_encoder |= name.startswith("model.acoustic_tokenizer.encoder.")
                if self._torch_prefill and name.startswith("model.language_model."):
                    self._lm_sd[name] = t.to(device=eng.device, dtype=torch.bfloat16)
        eng.finalize(scale, bias)          # fails if only part of the acoustic encoder was loaded
        self._scale, self._bias = scale, bias
        self._voice = self._voice_prompt if has_encoder else None
        if self._torch_prefill:
            from .prefill import TorchPrefill
            self._prefill = TorchPrefill(self.config, self._lm_sd, eng.device)
        return self

    @torch.no_grad()
    def _voice_prompt(self, speech_tensors: torch.Tensor, speech_masks: torch.Tensor, scale: float, bias: float, noise=None,
                      generator: Optional[torch.Generator] = None) -> torch.Tensor:
        """Voice-prompt half of step 0 (`modeling_vibevoice_inference.py:149-163, 216-224`) on the engine (`vv_voice_encode`): acoustic
        tokenizer encoder over the padded reference wavs, Gaussian sampling (`modular_vibevoice_tokenizer.py:980-989`), (x + bias) * scale,
        `acoustic_connector`.  -> connected embeddings [sum(speech_masks), H] fp32 on the device, in row-major mask order.  The noise is
        drawn from the device RNG (or `generator`, a device generator) in the order PyTorch's sampling draws it (std_n [n], then
        eps [n, F, vae_dim]); `noise=(std_n, eps)` overrides both (tests)."""
        eng = self.engine
        if (float(scale), float(bias)) != (self._scale, self._bias):
            raise ValueError("speech scale / bias (%r, %r) differ from the checkpoint's (%r, %r), which the engine was built with"
                             % (scale, bias, self._scale, self._bias))
        tc, dev = self.config.acoustic_tokenizer_config, eng.device
        wavs = torch.as_tensor(speech_tensors)
        n, T = wavs.shape
        std_n, eps = self._draw_voice_noise(n, T, generator) if noise is None else noise
        if tc.std_dist_type == "gaussian":
            sigma = std_n.to(dev, torch.float32) * (float(tc.fix_std) / 0.8)
            eps = eps.to(dev, torch.float32)
        elif tc.std_dist_type == "fix":
            eps = eps.to(dev, torch.float32)
            sigma = torch.full((n,), float(tc.fix_std), device=dev)
        else:
            eps, sigma = None, torch.zeros(n, device=dev)
        emb = eng.voice_encode(wavs, sigma, eps)
        return emb[torch.as_tensor(speech_masks).to(dev).bool()]

    def _draw_voice_noise(self, n: int, T: int, generator: Optional[torch.Generator] = None):
        """(std_n [n], eps [n, F, vae_dim]) of `_voice_prompt` for n voices of T samples, in PyTorch's sampling order; a part the
        checkpoint's std_dist_type does not use is None and is not drawn."""
        tc, eng = self.config.acoustic_tokenizer_config, self.engine
        shape = (n, eng.voice_frames(T), self.config.acoustic_vae_dim)
        std_n = torch.randn(n, device=eng.device, generator=generator) if tc.std_dist_type == "gaussian" else None
        eps = torch.randn(shape, device=eng.device, generator=generator) if tc.std_dist_type in ("gaussian", "fix") else None
        return std_n, eps

    @torch.no_grad()
    def voice_preset(self, prefix_inputs, seed: Optional[int] = None, generator: Optional[torch.Generator] = None) -> "VoicePreset":
        """Encode a voice prompt prefix once (`VibeVoiceProcessor.voice_prefix`: ids, speech_input_mask, speech_tensors, speech_masks)
        for `generate(..., voice_preset=)` and `RequestQueue.submit(..., voice_preset=)`.  The voice noise comes from `generator` (a
        device generator), else a device generator seeded with `seed`, else the device RNG, and is kept (`VoicePreset.noise`), so a
        preset made with the same seed is the same.  The prefix's K/V is prefilled by the first request that uses it."""
        eng = self.engine
        if eng is None or not eng.finalized:
            raise N.VVError("weights not loaded")
        if self._voice is None:
            raise N.VVError("voice presets need the acoustic tokenizer encoder weights, which this checkpoint does not have")
        ids = torch.as_tensor(prefix_inputs["input_ids"]).cpu().long()
        sim = torch.as_tensor(prefix_inputs["speech_input_mask"]).cpu().bool()
        if ids.dim() == 2 and ids.shape[0] != 1 or sim.shape != ids.shape:
            raise ValueError("voice_preset: one prefix (input_ids %s, speech_input_mask %s)" % (tuple(ids.shape), tuple(sim.shape)))
        ids, sim = ids.reshape(-1), sim.reshape(-1)
        wavs, masks = torch.as_tensor(prefix_inputs["speech_tensors"]), torch.as_tensor(prefix_inputs["speech_masks"]).bool()
        if int(masks.sum()) != int(sim.sum()):
            raise ValueError("voice_preset: %d speech positions for %d voice frames" % (int(sim.sum()), int(masks.sum())))
        if generator is None and seed is not None:
            generator = torch.Generator(device=eng.device).manual_seed(int(seed))
        with torch.cuda.stream(eng.stream):
            noise = self._draw_voice_noise(wavs.shape[0], wavs.shape[1], generator)
            ve = self._voice(wavs, masks, self._scale, self._bias, noise=noise)
            e = eng.embed_gather(ids).clone()
            e[sim.to(e.device)] = ve.to(e.device, e.dtype)
        return VoicePreset(self, ids, e, noise)

    def _presets_of(self, voice_preset, b: int) -> List[Optional["VoicePreset"]]:
        ps = list(voice_preset) if isinstance(voice_preset, (list, tuple)) else [voice_preset] * b
        if len(ps) != b:
            raise ValueError("voice_preset: %d presets for %d rows" % (len(ps), b))
        for p in ps:
            if p is not None and (not isinstance(p, VoicePreset) or p.model is not self):
                raise ValueError("voice_preset: a preset made by model.voice_preset() of this model (or None)")
        return ps

    @staticmethod
    def _check_preset_row(p: "VoicePreset", ids: torch.Tensor, sim: Optional[torch.Tensor], what: str):
        """ids / sim: one row's unpadded prompt ids and speech mask (sim may be None)."""
        Lp = p.ids.numel()
        if ids.numel() <= Lp or not torch.equal(ids[:Lp], p.ids):
            raise ValueError("voice_preset: %s does not start with the preset's %d prefix ids (followed by the script)" % (what, Lp))
        if sim is not None and bool(sim[Lp:].any()):
            raise ValueError("voice_preset: %s has speech positions past the preset's prefix" % what)

    def _preset_embeds(self, p: "VoicePreset", ids: torch.Tensor) -> torch.Tensor:
        """[L, H] prompt embeddings of a row whose unpadded ids start with the preset's: its embeddings, then the rest gathered."""
        return torch.cat([p.embeds, self.engine.embed_gather(ids[p.ids.numel():])])

    def _preset_prefill(self, p: "VoicePreset", seq: int, embeds: torch.Tensor) -> torch.Tensor:
        """Native prefill of an empty sequence whose prompt starts with the preset: attach the shared pages, or prefill them and make
        them the preset's; then the rest from position `shared`.  -> final-norm hidden of the last row.  The caller sets the length."""
        eng = self.engine
        if p.shared and not p._attach(seq):
            eng.lm_prefill(seq, embeds[:p.shared])
            eng.kv_set_len(seq, p.shared)
            p._adopt(seq)
        return eng.lm_prefill(seq, embeds[p.shared:], pos0=p.shared)

    @classmethod
    def from_pretrained(cls, path: str, torch_dtype=None, device_map=None, attn_implementation=None, tokenizer=None,
                        max_batch: int = 1, **kw):
        """HF checkpoint directory (config.json + *.safetensors), as `demo/inference_from_file.py:295-332` calls it.
        `torch_dtype` / `attn_implementation` are accepted for drop-in compatibility; storage is bf16 and attention is
        the built-in paged split-KV kernel.  The prompt prefill is enabled by default; `torch_prefill=False` drops the second (bf16) copy of
        the LM weights that prefill keeps and leaves only token-by-token prompt ingestion through the decode kernels.  `prefill_impl="native"`
        makes the engine's own prefill kernels (`vv_lm_prefill`) the default of `generate()`; `torch_prefill` then defaults to False, so no
        second copy of the LM is kept unless asked for.  Voice prompts (the
        demo's `generate(**inputs, is_prefill=True)` with `speech_tensors`) run on the engine's acoustic encoder either way.
        Special-token ids come from the tokenizer files next to the checkpoint when there are any, else from the public Qwen2.5
        vocabulary (`modular_vibevoice_text_tokenizer.py:175-181`); `generate()` checks them against the tokenizer it is handed."""
        from safetensors import safe_open
        cfg = VibeVoiceConfig.from_pretrained(path)
        dev = 0
        if isinstance(device_map, str) and device_map.startswith("cuda:"):
            dev = int(device_map.split(":")[1])
        elif isinstance(device_map, str) and device_map not in ("cuda", "auto"):
            raise N.VVError("vibevoice_b200 runs on CUDA devices only (device_map=%r); there is no CPU path" % device_map)
        if tokenizer is None:
            tokenizer = cls._tokenizer_ids_from_dir(path, cfg.decoder_config.vocab_size)
        prefill_impl = kw.pop("prefill_impl", None)
        m = cls(cfg, tokenizer, max_batch=max_batch, device=dev, torch_prefill=bool(kw.pop("torch_prefill", prefill_impl != "native")),
                prefill_impl=prefill_impl)

        def it():
            files = sorted(glob.glob(os.path.join(path, "*.safetensors")))
            if not files:
                raise FileNotFoundError("no *.safetensors under %s" % path)
            for f in files:
                with safe_open(f, framework="pt", device="cpu") as sf:
                    for k in sf.keys():
                        yield k, sf.get_tensor(k)
        m._weights_source = it
        lora_dir = kw.pop("lora_dir", None)
        if lora_dir is not None:
            from .lora import collect_overrides, merged_state_dict
            deltas, repl, m.lora_report = collect_overrides(lora_dir)
            m.load_state_dict(merged_state_dict(it(), deltas, repl), tokenizer)
        else:
            m.load_state_dict(it(), tokenizer)
        return m

    @staticmethod
    def _tokenizer_ids_from_dir(path: str, vocab_size: int):
        if any(os.path.exists(os.path.join(path, f)) for f in ("tokenizer.json", "vocab.json", "tokenizer_config.json")):
            try:
                from transformers import AutoTokenizer
                t = AutoTokenizer.from_pretrained(path)
                ids = t.convert_tokens_to_ids
                return SimpleNamespace(speech_start_id=ids("<|vision_start|>"), speech_end_id=ids("<|vision_end|>"),
                                       speech_diffusion_id=ids("<|vision_pad|>"), pad_id=ids("<|image_pad|>"), pad_token_id=ids("<|image_pad|>"),
                                       eos_token_id=t.eos_token_id, bos_token_id=getattr(t, "bos_token_id", None))
            except Exception:
                pass
        from .synth import SynthTokenizer
        return SynthTokenizer(vocab_size)

    def _reload_with(self, transform):
        """Re-stream the weights through `transform` (an iterator -> iterator function) and pack them again; used by
        `lora.load_lora_assets`.  Generation state (KV pages, codec state) does not survive."""
        if self._weights_source is None:
            raise RuntimeError("weights were loaded from a one-shot iterator; build the model with from_pretrained(..., lora_dir=...) instead")
        user_sched = None
        if self.engine is not None:
            if self.model.noise_scheduler is not self.engine.scheduler:
                user_sched = self.model.noise_scheduler           # a scheduler the caller installed survives the re-pack
            self.engine.close()
        self.engine = None
        self._prefill = self._voice = None
        self._lm_sd = {}
        self._kv_tokens = 0
        src = self._weights_source
        self.load_state_dict(transform(src()), self._tok)
        self._weights_source = src
        if user_sched is not None:
            self.model.noise_scheduler = user_sched
        return self

    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    @property
    def device(self):
        return torch.device("cuda", self._device_index)

    def set_ddpm_inference_steps(self, num_steps=None):
        """`:146-147`."""
        self.ddpm_inference_steps = num_steps or self.config.diffusion_head_config.ddpm_num_inference_steps

    # ---- generate ----------------------------------------------------------------------------------------
    @staticmethod
    def _config_processors(gcfg: dict, do_sample: bool) -> list:
        """The generation-config-driven subset of HF `GenerationMixin._get_logits_processor` that acts per step on [B, vocab] scores:
        repetition penalty always; temperature -> top-k -> top-p when sampling.  HF's sampling defaults apply (top_k = 50 unless the
        caller sets it; pass top_k=0 to sample from the plain constrained softmax like `oracle/make_golden.py` does)."""
        out = []
        rp = gcfg.get("repetition_penalty")
        if rp is not None and float(rp) != 1.0:
            from transformers import RepetitionPenaltyLogitsProcessor
            out.append(RepetitionPenaltyLogitsProcessor(penalty=float(rp)))
        if do_sample:
            from transformers import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
            t = gcfg.get("temperature")
            if t is not None and float(t) != 1.0:
                out.append(TemperatureLogitsWarper(float(t)))
            k = gcfg.get("top_k", 50)
            if k is not None and int(k) != 0:
                out.append(TopKLogitsWarper(top_k=int(k), min_tokens_to_keep=1))
            tp = gcfg.get("top_p")
            if tp is not None and float(tp) < 1.0:
                out.append(TopPLogitsWarper(top_p=float(tp), min_tokens_to_keep=1))
        return out

    def _reserve_kv(self, total_tokens: int):
        eng = self.engine
        need_pages = (total_tokens + 63) // 64 + 4 * eng.B          # every sequence may hold one partially filled page
        held = sum((getattr(eng, "prefix_pages", None) or {}).values())     # voice presets' shared pages stay in the pool
        if eng.kv_pages - held < need_pages:
            eng.kv_init(total_tokens)                                # first call, or a later call that needs more: the pool is re-sized

    def _prefill_rows(self, b, input_ids, attention_mask, lens, use_voice, speech_tensors, speech_masks, speech_input_mask, voice_noise,
                      gather, run, presets=None) -> List[torch.Tensor]:
        """Whole-prompt prefill of rows 0..b-1, one call per row: `gather(ids)` embeds the unpadded ids, the voice embeddings are scattered
        at `speech_input_mask` (:216-224: acoustic encoder -> sample -> (x+bias)*scale -> connector), `run(r, embeds)` fills the K/V of
        sequence r and returns its last final-norm hidden state; the row's length is then set.  A row with a voice preset
        (`presets[r]`) takes the preset's embeddings and shared pages and the native prefill instead.  -> hidden states of the rows."""
        eng = self.engine
        hids = []
        with torch.cuda.stream(eng.stream):
            voice_embeds = None
            if use_voice:
                voice_embeds = self._voice(torch.as_tensor(speech_tensors), torch.as_tensor(speech_masks).bool(), self._scale, self._bias,
                                           noise=voice_noise)
                sim = torch.as_tensor(speech_input_mask).bool().cpu()
                counts = sim.sum(dim=-1).tolist()
                offs = [0]
                for c_ in counts:
                    offs.append(offs[-1] + int(c_))
            for r in range(b):
                keep = attention_mask[r].bool()
                if presets is not None and presets[r] is not None:
                    ids_r = input_ids[r][keep]
                    hids.append(self._preset_prefill(presets[r], r, self._preset_embeds(presets[r], ids_r)))
                    eng.kv_set_len(r, int(lens[r]))
                    continue
                e = gather(input_ids[r][keep])
                if voice_embeds is not None and counts[r]:
                    e = e.clone()
                    e[sim[r][keep].to(e.device)] = voice_embeds[offs[r]:offs[r + 1]].to(e.device, e.dtype)
                hids.append(run(r, e))
                eng.kv_set_len(r, int(lens[r]))
        return hids

    @torch.no_grad()
    def generate(self, inputs=None, generation_config=None, logits_processor=None, stopping_criteria=None,
                 prefix_allowed_tokens_fn=None, synced_gpus=None, assistant_model=None, audio_streamer=None,
                 negative_prompt_ids=None, negative_prompt_attention_mask=None, speech_tensors=None, speech_masks=None,
                 speech_input_mask=None, is_prefill: bool = True, return_speech: bool = True, cfg_scale: float = 1.0,
                 stop_check_fn: Optional[Callable[[], bool]] = None, tqdm_class=None, voice_preset=None, **kwargs) -> VibeVoiceGenerationOutput:
        """`modeling_vibevoice_inference.py:326-695`.

        `voice_preset`: a `VoicePreset` for every row, or a list with a preset or None per row.  A row with a preset must start with the
        preset's prefix ids and have no speech position after them; it runs no voice encoding (its speech inputs, if given, are not
        used) and is prefilled natively from the preset's shared pages on.  Rows without a preset carry no voice in such a batch."""
        tokenizer = kwargs.pop("tokenizer", None) or self._tok
        kwargs.pop("parsed_scripts", None); kwargs.pop("all_speakers_list", None)
        max_length_times = kwargs.pop("max_length_times", 2)
        verbose = kwargs.get("verbose", False)
        gcfg = {}
        if generation_config is not None:
            gcfg = dict(generation_config) if isinstance(generation_config, dict) else {k: v for k, v in vars(generation_config).items() if not k.startswith("_")}
        do_sample = bool(gcfg.get("do_sample", False))
        sample_gen = kwargs.get("sample_generator", None)          # torch.Generator for the token draw; never the noise RNG
        if do_sample and sample_gen is None:
            sample_gen = torch.Generator().manual_seed(torch.initial_seed())
        refresh_negative = bool(kwargs.get("refresh_negative", True))
        use_voice = bool(is_prefill and speech_tensors is not None)
        if use_voice and self._voice is None and voice_preset is None:
            raise N.VVError("voice-prompt prefill needs the acoustic tokenizer encoder weights, which this checkpoint does not have")
        forced: Optional[ForcedTokenScript] = None
        user_procs = []
        if logits_processor is not None:
            procs = logits_processor if isinstance(logits_processor, (list, tuple)) else [logits_processor]
            for p in procs:
                if isinstance(p, ForcedTokenScript):
                    forced = p
                else:
                    user_procs.append(p)
        # Score processors that rank the WHOLE vocabulary before the token constraint (`_get_logits_processor` from the generation config,
        # :310-319, then VibeVoiceTokenConstraintProcessor appended last, :415-418): they need full-vocabulary logits, which the default path
        # never materialises.  With any of them present every step computes them with one extra GEMV over the lm_head (vv_lm_logits_full).
        # NB the reference overwrites a caller-supplied `logits_processor` with the list built from the generation config (:375-377), i.e.
        # it silently ignores such objects; here they are applied (before the config-derived ones), which is what a caller expects.
        warpers = self._config_processors(gcfg, do_sample) + []
        full_vocab_procs = user_procs + warpers
        input_ids = kwargs["input_ids"] if "input_ids" in kwargs else inputs
        input_ids = torch.as_tensor(input_ids).cpu().long()
        attention_mask = kwargs.get("attention_mask", None)
        attention_mask = torch.ones_like(input_ids) if attention_mask is None else torch.as_tensor(attention_mask).cpu().long()
        eng = self.engine
        if eng is None or not eng.finalized:
            raise N.VVError("weights not loaded")
        dc = self.config.decoder_config
        b, L0 = input_ids.shape
        B = eng.B
        if b > B:
            raise ValueError("batch %d exceeds the engine's max_batch %d" % (b, B))
        tok = tokenizer
        start_id, end_id, diff_id, eos_id = tok.speech_start_id, tok.speech_end_id, tok.speech_diffusion_id, tok.eos_token_id
        if self._valid_ids(tok) != list(eng.valid_ids):
            # the lm_head rows and the constrained argmax were fixed when the weights were packed (:405-419 resolves them per call)
            raise ValueError("tokenizer special ids %s differ from the ids the engine was built with %s; load the model with this "
                             "tokenizer (from_pretrained(..., tokenizer=tok))" % (self._valid_ids(tok), list(eng.valid_ids)))
        presets = None
        if voice_preset is not None:
            if not is_prefill:
                raise ValueError("voice_preset needs the whole-prompt prefill (is_prefill=True)")
            if kwargs.get("prefill_impl") == "decode":
                raise ValueError("voice_preset: prefill_impl=\"decode\" cannot continue a prompt from shared K/V pages")
            presets = self._presets_of(voice_preset, b)
            sim_all = None if speech_input_mask is None else torch.as_tensor(speech_input_mask).bool().cpu()
            for r in range(b):
                keep = attention_mask[r].bool()
                sim_r = None if sim_all is None else sim_all[r][keep]
                if presets[r] is not None:
                    self._check_preset_row(presets[r], input_ids[r][keep], sim_r, "row %d" % r)
                elif sim_r is not None and bool(sim_r.any()):
                    raise ValueError("voice_preset: row %d has voice samples but no preset; give every voiced row a preset" % r)
            use_voice = False

        if kwargs.get("max_new_tokens", None) is None:
            kwargs["max_new_tokens"] = dc.max_position_embeddings - L0                      # :372-373
        max_length = L0 + int(kwargs["max_new_tokens"])
        init_len = attention_mask.sum(dim=-1)                                              # :402
        max_steps = min(max_length - L0, int(max_length_times * L0))                       # :421
        max_step_per_sample = torch.min(max_length - init_len, (max_length_times * init_len).long())   # :422
        self._reserve_kv(int(b * (L0 + max_steps + 2) + b * (max_steps + 2)))
        if self.model.noise_scheduler is not None and self.model.noise_scheduler is not eng.scheduler:
            eng.set_scheduler(self.model.noise_scheduler)      # `model.model.noise_scheduler = sched.from_config(...)`, gradio_demo.py:141-146
        eng.set_diffusion_steps(int(self.ddpm_inference_steps))
        step_noise_fn = kwargs.get("_step_noise_fn", None)      # test hook: i, n -> [2n,64]; default = device RNG like the reference
        eng.codec_state_reset()
        for s in range(2 * B):
            eng.kv_set_len(s, 0)

        neg_state = [_NegativeSlots() for _ in range(B)]        # refresh_negative=False only
        neg_pos: List[Dict[int, int]] = [dict() for _ in range(B)]   # entry id -> position in the pool
        finished = np.zeros(B, dtype=bool); finished[b:] = True
        reach_max = np.zeros(B, dtype=bool)
        seqs = [input_ids[i].tolist() for i in range(b)]
        audio_chunks: List[List[torch.Tensor]] = [[] for _ in range(b)]
        pad_tok = eos_id

        lens = init_len.tolist() + [0] * (B - b)
        Lmax = L0
        impl = kwargs.get("prefill_impl", self._prefill_impl or "auto")
        use_native_prefill = impl == "native"
        use_torch_prefill = not use_native_prefill and self._prefill is not None and impl != "decode"
        if presets is not None and not use_torch_prefill:
            use_native_prefill = True                            # preset rows continue from the pool; the others prefill as usual
        if use_torch_prefill or use_native_prefill:
            # ---- whole-prompt prefill (a-9 / f-2), K/V in the paged pool: library kernels (TorchPrefill) or the engine's (vv_lm_prefill) -----
            if use_torch_prefill:
                embw = self._lm_sd["model.language_model.embed_tokens.weight"]
                gather, run = (lambda ids_r: embw[ids_r.to(eng.device)]), (lambda r, e: self._prefill.run(eng, r, e))
            else:
                gather, run = eng.embed_gather, (lambda r, e: eng.lm_prefill(r, e))
            hids = self._prefill_rows(b, input_ids, attention_mask, lens, use_voice, speech_tensors, speech_masks, speech_input_mask,
                                      kwargs.get("_voice_noise"), gather, run, presets)
            eng.embed_tokens([pad_tok] * B + [start_id] * B, eng.embeds)     # negative rows: [<speech_start>] at pos 0 (:379-386)
            eng.lm_decode()
            with torch.cuda.stream(eng.stream):
                for r in range(b):
                    eng.hidden[r].copy_(hids[r])
            eng.lm_head(eng.hidden)
            pending_adv_pos = [0] * B
        else:
            # ---- prompt prefill through the decode kernel (left-padded rows start late) ----------------------------------
            adv = [0] * B
            voice_embeds, sim, nxt = None, None, [0] * b
            if use_voice:         # voice rows take the connected embeddings in mask order, same offsets as above
                with torch.cuda.stream(eng.stream):
                    voice_embeds = self._voice(torch.as_tensor(speech_tensors), torch.as_tensor(speech_masks).bool(), self._scale, self._bias,
                                               noise=kwargs.get("_voice_noise"))
                sim = torch.as_tensor(speech_input_mask).bool().cpu()
                counts = sim.sum(dim=-1).tolist()
                for r in range(1, b):
                    nxt[r] = nxt[r - 1] + int(counts[r - 1])
            for t in range(Lmax):
                toks, adv = [], []
                for r in range(B):
                    live = r < b and t >= Lmax - lens[r] and bool(attention_mask[r, t])
                    toks.append(int(input_ids[r, t]) if live else pad_tok)
                    adv.append(1 if live else 0)
                last = t == Lmax - 1
                eng.embed_tokens(toks + ([start_id] * B if last else toks), eng.embeds)      # neg rows: [<speech_start>] at pos 0
                if voice_embeds is not None:
                    with torch.cuda.stream(eng.stream):
                        for r in range(b):
                            if adv[r] and sim[r, t]:
                                eng.embeds[r].copy_(voice_embeds[nxt[r]])
                                nxt[r] += 1
                eng.lm_decode()
                if not last:
                    eng.kv_commit(adv + [0] * B)
            pending_adv_pos = adv                                                           # committed once tokens are known

        iterator = range(max_steps)
        if kwargs.get("show_progress_bar", False):
            from tqdm import tqdm
            iterator = (tqdm_class or tqdm)(iterator, desc="Generating", leave=False)
        step_done = False
        pending_audio = None

        def flush_audio():
            """hand the previous frame's chunk to the streamer: its copy into the pinned ring was enqueued before the LM step whose
            tokens the loop has just read back, so no extra synchronisation happens here"""
            nonlocal pending_audio
            if pending_audio is not None:
                ticket, rows = pending_audio
                pending_audio = None
                audio_streamer.put(eng.fetch_audio(ticket).unsqueeze(1), torch.as_tensor(rows))

        for step in iterator:
            if stop_check_fn is not None and stop_check_fn():                               # :434-440
                if audio_streamer is not None:
                    flush_audio()
                    audio_streamer.end()
                break
            if audio_streamer is not None and hasattr(audio_streamer, "finished_flags") and any(audio_streamer.finished_flags):
                break                                                                       # :443-447
            if finished[:b].all():                                                          # :449-452
                break
            if len(seqs[0]) >= max_length:                                                  # :454-459
                reach_max[:b] |= ~finished[:b]
                break
            if step > 0:
                eng.lm_decode()                                                             # :480-482 (+ speculative negative rows)
            toks_dev, logits_valid = eng.read_tokens()
            if audio_streamer is not None:
                flush_audio()
            next_tokens = toks_dev.astype(np.int64).copy()
            if full_vocab_procs:                                                              # :488-498 on full-vocabulary scores
                scores = eng.lm_logits_full()[:b].clone()
                cur_ids = torch.tensor([s_ for s_ in seqs], dtype=torch.long, device=scores.device)
                for p_ in full_vocab_procs:
                    scores = p_(cur_ids, scores)
                sv = scores[:, eng.valid_ids].float().cpu()                                   # the constraint keeps these ids only (:55-66)
                if do_sample:
                    next_tokens[:b] = sample_valid_tokens(sv.numpy(), eng.valid_ids, sample_gen)
                else:
                    next_tokens[:b] = np.asarray(eng.valid_ids, dtype=np.int64)[sv.argmax(dim=-1).numpy()]
            elif do_sample:
                next_tokens[:b] = sample_valid_tokens(logits_valid[:b], eng.valid_ids, sample_gen)                   # :493-496
            if forced is not None:
                for r in range(b):
                    next_tokens[r] = forced.token(r, step)
            next_tokens[finished] = eos_id                                                   # :500
            for r in range(b):
                seqs[r].append(int(next_tokens[r]))                                          # :501
            new_eos = (next_tokens == eos_id) & ~finished                                    # :519-528
            if new_eos.any():
                finished |= new_eos
                if verbose:
                    print(f"Samples {np.nonzero(new_eos)[0].tolist()} reached EOS token at step {step + 1}.", flush=True)
                if audio_streamer is not None:
                    audio_streamer.end(torch.as_tensor(np.nonzero(new_eos)[0]))
            mlr = np.zeros(B, dtype=bool)
            mlr[:b] = (step >= max_step_per_sample.numpy()) & ~finished[:b]                  # :531-539
            if mlr.any():
                finished |= mlr; reach_max |= mlr
                if audio_streamer is not None:
                    audio_streamer.end(torch.as_tensor(np.nonzero(mlr)[0]))
            end_rows = np.nonzero(next_tokens[:b] == end_id)[0]                               # :542-546
            if end_rows.size:
                eng.codec_state_zero(end_rows.tolist())
            start_rows = np.nonzero(~finished[:b] & (next_tokens[:b] == start_id))[0]         # :549-565
            diff_mask = np.zeros(B, dtype=bool)
            diff_mask[:b] = ~finished[:b] & (next_tokens[:b] == diff_id)                      # :573
            diff_rows = np.nonzero(diff_mask)[0]
            # KV bookkeeping: positive rows always keep their entry; negative rows only when the token is a diffusion token
            adv_pos = pending_adv_pos if step == 0 else [1] * b + [0] * (B - b)
            if refresh_negative:
                eng.kv_commit(list(adv_pos) + [1 if diff_mask[r] else 0 for r in range(B)])
                for r in start_rows.tolist():
                    eng.kv_set_len(B + r, 0)                                                  # negative stream restarts at [<speech_start>]
            else:
                # :503-517, 594-624: every step's input enters the negative stream; when some row diffuses, the rows that do not get
                # their step undone by the reference's mask / cache shift.  Mirror its bookkeeping and bring the pool to the same set.
                neg_adv = [0] * B
                deletes = []
                for r in range(b):
                    if finished[r]:
                        continue                                   # its stream is never read again
                    st = neg_state[r]
                    e_new = st.append()
                    if diff_rows.size and not diff_mask[r]:
                        st.correct()
                    vis = st.visible()
                    if len(set(vis)) != len(vis):
                        raise NotImplementedError("the reference's cache shift left a duplicated visible entry; not representable")
                    vis = set(vis)
                    neg_adv[r] = 1 if e_new in vis else 0
                    deletes += [(r, e) for e in neg_pos[r] if e not in vis]
                    if neg_adv[r]:
                        neg_pos[r][e_new] = len(neg_pos[r])
                eng.kv_commit(list(adv_pos) + neg_adv)
                for r, e_old in deletes:                           # an OLDER entry was hidden: the last entry takes its place in the pool
                    p_old = neg_pos[r].pop(e_old)
                    n_after = len(neg_pos[r])
                    for e, ppos in neg_pos[r].items():
                        if ppos == n_after:
                            neg_pos[r][e] = p_old
                            break
                    eng.kv_delete(B + r, p_old)
            tl = [int(t) for t in next_tokens]
            eng.embed_tokens(tl + tl, eng.embeds)                                             # :569 (negative rows see the same input, :579-581)
            if diff_rows.size:
                n = int(diff_rows.size)
                noise = torch.randn(2 * n, self.config.acoustic_vae_dim)[:n]                  # CPU global RNG, rows [:n] used (:701-704)
                eng.upload_frame_inputs(noise, diff_rows.tolist())
                if eng.sde:                                                                   # dpm_solver.py:993-997, one draw per step
                    draw = (lambda i: step_noise_fn(i, n)) if step_noise_fn is not None else \
                        (lambda i: torch.randn(2 * n, self.config.acoustic_vae_dim, device=eng.device))
                    eng.upload_step_noise(draw, diff_rows.tolist())
                eng.frame_tail(cfg_scale)                                                     # :626-672
                with torch.cuda.stream(eng.stream):
                    chunk = eng.audio[diff_rows.tolist()].clone()                              # [n, 3200]
                for i, r in enumerate(diff_rows.tolist()):
                    audio_chunks[r].append(chunk[i:i + 1])                                    # :646-650
                if audio_streamer is not None:                                                 # :653-655, one frame behind (no sync here):
                    pending_audio = (eng.stage_audio(diff_rows.tolist()), diff_rows.copy())   # pinned ring, delivered after the next read-back
        if audio_streamer is not None:
            flush_audio()
            audio_streamer.end()                                                              # :677-678
        eng.sync()
        outs: List[Optional[torch.Tensor]] = []
        with torch.cuda.stream(eng.stream):
            for ch in audio_chunks:
                outs.append(torch.cat(ch, dim=-1) if ch else None)                            # :680-689
        eng.sync()
        L = max(len(s) for s in seqs)
        sequences = torch.tensor([s + [pad_tok] * (L - len(s)) for s in seqs], dtype=torch.long)
        return VibeVoiceGenerationOutput(sequences=sequences, speech_outputs=outs if return_speech else None,
                                         reach_max_step_sample=torch.as_tensor(reach_max[:b].copy()))
