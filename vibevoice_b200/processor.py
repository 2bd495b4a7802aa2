"""`VibeVoiceProcessor` -- script + voice samples -> model inputs, and `save_audio`; `VibeVoiceStreamingProcessor` -- text + a cached
voice prompt -> the streaming-0.5B model's inputs.

Same call surface and output keys as the reference (`vibevoice/processor/vibevoice_processor.py:163-244, 374-404, 677-696`):
`input_ids, attention_mask, speech_input_mask, speech_tensors, speech_masks, parsed_scripts, all_speakers_list`, left-padded
with `tokenizer.pad_id`.  Runs once per request on the host (not part of the accelerated path); re-implemented here so that
`demo/inference_from_file.py` has everything it imports, without `librosa`/`soundfile` (absent in this image): wav I/O goes through
`scipy.io.wavfile` + polyphase resampling to 24 kHz.

Prompt layout (`_process_single`, :246-304; `_create_voice_prompt`, :406-467):
    <system prompt> [" Voice input:\\n" (" Speaker i:" <speech_start> <speech_diffusion> x ceil(len/3200) <speech_end> "\\n")*]
    " Text input:\\n" (" Speaker i:<text>\\n")* " Speech output:\\n" <speech_start>
"""
from __future__ import annotations

import json
import math
import os
import re
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

SYSTEM_PROMPT = (" Transform the text provided by various speakers into speech output, utilizing the distinct voice of each "
                 "respective speaker.\n")


class BatchEncoding(dict):
    """dict with attribute access and `.to(device)` (the slice of HF `BatchEncoding` the demos use)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def to(self, device):
        for k, v in self.items():
            if torch.is_tensor(v):
                self[k] = v.to(device)
        return self


class AudioNormalizer:
    """-25 dBFS RMS normalisation then peak protection (`vibevoice_tokenizer_processor.py:19-87`)."""

    def __init__(self, target_dB_FS: float = -25, eps: float = 1e-6):
        self.target_dB_FS, self.eps = target_dB_FS, eps

    def __call__(self, audio: np.ndarray) -> np.ndarray:
        rms = np.sqrt(np.mean(audio ** 2))
        audio = audio * (10 ** (self.target_dB_FS / 20) / (rms + self.eps))
        peak = np.max(np.abs(audio))
        return audio / (peak + self.eps if peak > 1.0 else 1.0)


def load_wav_24k(path: str, target_sr: int = 24000) -> np.ndarray:
    """mono float32 at 24 kHz (the reference uses `librosa.load(sr=24000, mono=True)`)."""
    from scipy.io import wavfile
    from scipy.signal import resample_poly
    sr, x = wavfile.read(path)
    if x.dtype.kind == "i":
        x = x.astype(np.float32) / float(np.iinfo(x.dtype).max + 1)
    elif x.dtype.kind == "u":
        x = (x.astype(np.float32) - 128.0) / 128.0
    else:
        x = x.astype(np.float32)
    if x.ndim > 1:
        x = x.mean(axis=1)
    if sr != target_sr:
        g = math.gcd(int(sr), target_sr)
        x = resample_poly(x, target_sr // g, int(sr) // g).astype(np.float32)
    return x


def convert_to_16_bit_wav(data) -> np.ndarray:
    """`demo/gradio_demo.py:1058-1072`: tensor / array -> int16 PCM, peak-normalised only when the signal exceeds [-1, 1]."""
    if torch.is_tensor(data):
        data = data.detach().float().cpu().numpy()
    data = np.array(data)
    peak = np.max(np.abs(data)) if data.size else 0.0
    if peak > 1.0:
        data = data / peak
    return (data * 32767).astype(np.int16)


def _set_speech_token_ids(tokenizer):
    """The special-token ids the VibeVoice tokenizers expose as attributes (`modular_vibevoice_text_tokenizer.py:163-181`)."""
    ids = tokenizer.convert_tokens_to_ids
    tokenizer.speech_start_id, tokenizer.speech_end_id = ids("<|vision_start|>"), ids("<|vision_end|>")
    tokenizer.speech_diffusion_id, tokenizer.pad_id = ids("<|vision_pad|>"), ids("<|image_pad|>")
    return tokenizer


class VibeVoiceProcessor:
    def __init__(self, tokenizer=None, audio_processor=None, speech_tok_compress_ratio: int = 3200, db_normalize: bool = True, **kwargs):
        self.tokenizer = tokenizer
        self.audio_processor = audio_processor
        self.speech_tok_compress_ratio = speech_tok_compress_ratio
        self.db_normalize = db_normalize
        self.audio_normalizer = AudioNormalizer() if db_normalize else None
        self.system_prompt = SYSTEM_PROMPT
        self.sampling_rate = 24000

    @classmethod
    def from_pretrained(cls, path: str, tokenizer=None, **kwargs):
        cfg = {}
        f = os.path.join(path, "preprocessor_config.json")
        if os.path.exists(f):
            cfg = json.load(open(f))
        if tokenizer is None:
            try:   # a Qwen2.5 tokenizer next to the checkpoint (the reference resolves `language_model_pretrained_name` on the hub)
                from transformers import AutoTokenizer
                tokenizer = _set_speech_token_ids(AutoTokenizer.from_pretrained(path))
            except Exception as e:
                raise FileNotFoundError("no tokenizer files under %s (offline image): pass tokenizer=... explicitly" % path) from e
        return cls(tokenizer=tokenizer, speech_tok_compress_ratio=cfg.get("speech_tok_compress_ratio", 3200),
                   db_normalize=cfg.get("db_normalize", True))

    # ---- script ------------------------------------------------------------------------------------------------------
    @staticmethod
    def _parse_script(script: str) -> List[Tuple[int, str]]:
        out = []
        for line in script.strip().split("\n"):
            m = re.match(r"^Speaker\s+(\d+)\s*:\s*(.*)$", line.strip(), re.IGNORECASE) if line.strip() else None
            if m:
                out.append((int(m.group(1)), " " + m.group(2).strip()))
        if not out:
            raise ValueError("No valid speaker lines found in script")
        if min(s for s, _ in out) > 0:                       # 1-based scripts are shifted to 0-based
            out = [(s - 1, t) for s, t in out]
        return out

    def _text_file_to_script(self, path: str) -> str:
        """`.json` = [{"speaker": "1", "text": "..."}]; `.txt` = "Speaker N: text" lines, bare lines go to Speaker 1 (:519-602)."""
        lines = []
        if path.endswith(".json"):
            data = json.load(open(path, encoding="utf-8"))
            if not isinstance(data, list):
                raise ValueError("JSON file must contain a list of speaker entries")
            for item in data:
                if not isinstance(item, dict) or item.get("speaker") is None or item.get("text") is None:
                    continue
                try:
                    spk = int(item["speaker"])
                except (ValueError, TypeError):
                    continue
                if item["text"].strip():
                    lines.append(f"Speaker {spk}: {item['text'].strip()}")
            if not lines:
                raise ValueError("No valid entries found in JSON file")
            return "\n".join(lines)
        for raw in open(path, encoding="utf-8").read().split("\n"):
            raw = raw.strip()
            if not raw:
                continue
            m = re.match(r"^Speaker\s+(\d+)\s*:\s*(.*)$", raw, re.IGNORECASE)
            if m:
                if m.group(2).strip():
                    lines.append(f"Speaker {int(m.group(1))}: {m.group(2).strip()}")
            else:
                lines.append(f"Speaker 1: {raw}")
        if not lines:
            raise ValueError("No valid content found in text file")
        return "\n".join(lines)

    def _enc(self, text: str, special: bool = False) -> List[int]:
        return list(self.tokenizer.encode(text) if special else self.tokenizer.encode(text, add_special_tokens=False))

    def _voice_prompt(self, samples: Sequence[Union[str, np.ndarray, dict]]):
        tok = self.tokenizer
        ids = self._enc(" Voice input:\n")
        mask = [False] * len(ids)
        wavs = []
        for i, a in enumerate(samples):
            if isinstance(a, str):
                wav = load_wav_24k(a)
            elif isinstance(a, dict):
                key = "array" if "array" in a else "audio"
                if key not in a:
                    raise ValueError("Dictionary audio input must have 'array' or 'audio' key")
                wav = np.array(a[key], dtype=np.float32)
            else:
                wav = np.array(a, dtype=np.float32)
            if self.audio_normalizer is not None:
                wav = self.audio_normalizer(wav)
            n = math.ceil(wav.shape[0] / self.speech_tok_compress_ratio)
            pre, nl = self._enc(f" Speaker {i}:"), self._enc("\n")
            ids += pre + [tok.speech_start_id] + [tok.speech_diffusion_id] * n + [tok.speech_end_id] + nl
            mask += [False] * (len(pre) + 1) + [True] * n + [False] * (1 + len(nl))
            wavs.append(wav)
        return ids, wavs, mask

    def _process_single(self, text, voice_samples=None) -> Dict[str, Any]:
        if isinstance(text, str) and text.endswith((".json", ".txt")) and os.path.exists(text):
            text = self._text_file_to_script(text)
        if not isinstance(text, str):
            raise ValueError(f"Could not process input text: {text}")
        parsed = self._parse_script(text)
        speakers = list(set(s for s, _ in parsed))
        ids = self._enc(self.system_prompt, special=True)
        mask = [False] * len(ids)
        wavs = []
        if voice_samples:
            v_ids, wavs, v_mask = self._voice_prompt(voice_samples[: len(speakers)])
            ids += v_ids
            mask += v_mask
        t = self._enc(" Text input:\n")
        ids += t
        mask += [False] * len(t)
        for spk, txt in parsed:
            t = self._enc(f" Speaker {spk}:{txt}\n")
            ids += t
            mask += [False] * len(t)
        t = self._enc(" Speech output:\n") + [self.tokenizer.speech_start_id]
        ids += t
        mask += [False] * len(t)
        return dict(input_ids=ids, speech_inputs=wavs or None, speech_input_mask=mask, parsed_script=parsed, all_speakers=speakers)

    def voice_prefix(self, voice_samples) -> BatchEncoding:
        """The prompt prefix `system prompt + " Voice input:\\n" + speakers` of `voice_samples` as tensors: `input_ids` [1, Lp],
        `speech_input_mask` [1, Lp], `speech_tensors` and `speech_masks` -- exactly the first Lp ids and the speech inputs that
        `self(text=script, voice_samples=voice_samples)` gives for any script, provided the script has as many speakers as there are
        voices (the processor keeps the first `len(speakers)` voices).  The input of `model.voice_preset`."""
        if not voice_samples:
            raise ValueError("voice_prefix needs at least one voice sample")
        ids = self._enc(self.system_prompt, special=True)
        v_ids, wavs, v_mask = self._voice_prompt(voice_samples)
        sp = self.prepare_speech_inputs(wavs, return_tensors="pt")
        return BatchEncoding(input_ids=torch.tensor([ids + v_ids], dtype=torch.long),
                             speech_input_mask=torch.tensor([[False] * len(ids) + v_mask], dtype=torch.bool),
                             speech_tensors=sp["padded_speeches"], speech_masks=sp["speech_masks"])

    def prepare_speech_inputs(self, speech_inputs: List[np.ndarray], return_tensors=None, device=None, dtype=None) -> Dict[str, Any]:
        if not speech_inputs:
            return {"padded_speeches": None, "speech_masks": None}
        r = self.speech_tok_compress_ratio
        n_tok = [math.ceil(s.shape[0] / r) for s in speech_inputs]
        padded = np.zeros((len(speech_inputs), max(s.shape[0] for s in speech_inputs)), dtype=np.float32)
        masks = np.zeros((len(speech_inputs), max(n_tok)), dtype=np.bool_)
        for i, (s, n) in enumerate(zip(speech_inputs, n_tok)):
            padded[i, : len(s)] = s
            masks[i, :n] = True
        if return_tensors == "pt":
            return {"padded_speeches": torch.tensor(padded, device=device, dtype=dtype or torch.float32),
                    "speech_masks": torch.tensor(masks, device=device, dtype=torch.bool)}
        return {"padded_speeches": padded, "speech_masks": masks}

    def __call__(self, text=None, voice_samples=None, padding=True, truncation=False, max_length=None, return_tensors=None,
                 return_attention_mask: bool = True, **kwargs) -> BatchEncoding:
        single = isinstance(text, str) or (isinstance(text, list) and len(text) > 0 and not isinstance(text[0], str))
        texts = [text] if single else list(text)
        if voice_samples is None:
            voices = [None] * len(texts)
        elif single or isinstance(voice_samples[0], (str, np.ndarray)):
            voices = [voice_samples]
        else:
            voices = voice_samples
        encs = [self._process_single(t, v) for t, v in zip(texts, voices)]
        ids_l, mask_l = [e["input_ids"] for e in encs], [e["speech_input_mask"] for e in encs]
        pad = padding is True or (isinstance(padding, str) and padding not in ("do_not_pad", "False"))
        att = [[1] * len(i) for i in ids_l]
        if pad:
            L = max_length if (padding == "max_length" and max_length is not None) else max(len(i) for i in ids_l)
            for j in range(len(ids_l)):
                if truncation and len(ids_l[j]) > L:
                    ids_l[j], mask_l[j] = ids_l[j][:L], mask_l[j][:L]
                n = L - len(ids_l[j])
                att[j] = [0] * n + [1] * len(ids_l[j])
                ids_l[j] = [self.tokenizer.pad_id] * n + ids_l[j]            # LEFT padding (:351-353)
                mask_l[j] = [False] * n + mask_l[j]
        out = BatchEncoding()
        if return_tensors is not None:
            out["input_ids"] = torch.tensor(ids_l, dtype=torch.long)
            if return_attention_mask:
                out["attention_mask"] = torch.tensor(att, dtype=torch.long)
            out["speech_input_mask"] = torch.tensor(mask_l, dtype=torch.bool)
        else:
            out["input_ids"] = ids_l
            if return_attention_mask:
                out["attention_mask"] = att
            out["speech_input_mask"] = mask_l
        all_wavs = [w for e in encs if e["speech_inputs"] is not None for w in e["speech_inputs"]]
        sp = self.prepare_speech_inputs(all_wavs, return_tensors=return_tensors)
        out["speech_tensors"], out["speech_masks"] = sp["padded_speeches"], sp["speech_masks"]
        out["parsed_scripts"] = [e["parsed_script"] for e in encs]
        out["all_speakers_list"] = [e["all_speakers"] for e in encs]
        return out

    # ---- output ------------------------------------------------------------------------------------------------------
    def save_audio(self, audio, output_path: str = "output.wav", sampling_rate: Optional[int] = None, normalize: bool = False,
                   batch_prefix: str = "audio_") -> Union[str, List[str]]:
        """`vibevoice_tokenizer_processor.py:352-457`: one tensor/array -> one 24 kHz wav; a list -> `batch_prefix{i}.wav` files."""
        from scipy.io import wavfile
        sr = sampling_rate or self.sampling_rate

        def to_np(a):
            a = a.detach().float().cpu().numpy() if torch.is_tensor(a) else np.asarray(a, dtype=np.float32)
            a = a.reshape(-1) if a.ndim <= 2 and (a.ndim == 1 or a.shape[0] == 1) else a.squeeze()
            if normalize and np.max(np.abs(a)) > 0:
                a = a / np.max(np.abs(a))
            return a.astype(np.float32)

        if isinstance(audio, (list, tuple)):
            d = output_path if os.path.isdir(output_path) or not output_path.endswith(".wav") else os.path.dirname(output_path) or "."
            os.makedirs(d, exist_ok=True)
            paths = []
            for i, a in enumerate(audio):
                p = os.path.join(d, f"{batch_prefix}{i}.wav")
                wavfile.write(p, sr, to_np(a))
                paths.append(p)
            return paths
        os.makedirs(os.path.dirname(os.path.abspath(output_path)), exist_ok=True)
        wavfile.write(output_path, sr, to_np(audio))
        return output_path

    def batch_decode(self, *a, **k):
        return self.tokenizer.batch_decode(*a, **k)

    def decode(self, *a, **k):
        return self.tokenizer.decode(*a, **k)


class VibeVoiceStreamingProcessor:
    """Inputs of the streaming-0.5B model (`VibeVoiceStreamingForConditionalGenerationInference.generate`) from one text and a cached
    voice prompt: the `all_prefilled_outputs` dict of a shipped preset (`demo/voices/streaming_model/*.pt`), whose four model outputs
    already hold the voice's K/V.  Same surface and output keys as the reference's `vibevoice/processor/vibevoice_streaming_processor.py`;
    the prompt positions are represented by `tokenizer.pad_id` placeholders, one per cached position of each stack."""

    def __init__(self, tokenizer=None, audio_processor=None, speech_tok_compress_ratio: int = 3200, db_normalize: bool = True, **kwargs):
        self.tokenizer = tokenizer
        self.audio_processor = audio_processor
        self.speech_tok_compress_ratio = speech_tok_compress_ratio
        self.db_normalize = db_normalize
        self.audio_normalizer = AudioNormalizer() if db_normalize else None
        self.sampling_rate = 24000

    @classmethod
    def from_pretrained(cls, path: str, tokenizer=None, **kwargs):
        """`path/preprocessor_config.json` (defaults when absent).  The tokenizer is, in order: `tokenizer=`; tokenizer files in `path`;
        `language_model_pretrained_name` (config, else keyword) from the local Hugging Face cache only.  Nothing is downloaded."""
        cfg = {}
        f = os.path.join(path, "preprocessor_config.json")
        if os.path.exists(f):
            with open(f) as fh:
                cfg = json.load(fh)
        if tokenizer is None:
            from transformers import AutoTokenizer
            name = cfg.get("language_model_pretrained_name") or kwargs.get("language_model_pretrained_name")
            errors = []
            for src in ([path] if os.path.isdir(path) else []) + ([name] if name else []):
                try:
                    tokenizer = _set_speech_token_ids(AutoTokenizer.from_pretrained(src, local_files_only=True))
                    break
                except Exception as e:   # no tokenizer files there / not in the local cache
                    errors.append("%s: %s" % (src, e))
            if tokenizer is None:
                raise FileNotFoundError("no tokenizer found offline for %s (tried %s): pass tokenizer=... explicitly"
                                        % (path, "; ".join(errors) or "nothing"))
        return cls(tokenizer=tokenizer, speech_tok_compress_ratio=cfg.get("speech_tok_compress_ratio", 3200),
                   db_normalize=cfg.get("db_normalize", True))

    def save_pretrained(self, save_directory: str, **kwargs):
        """Writes `preprocessor_config.json` in the reference's format (what `from_pretrained` reads back)."""
        os.makedirs(save_directory, exist_ok=True)
        ap = self.audio_processor
        cfg = {"processor_class": "VibeVoiceStreamingProcessor", "speech_tok_compress_ratio": self.speech_tok_compress_ratio,
               "db_normalize": self.db_normalize,
               "audio_processor": {"feature_extractor_type": "VibeVoiceTokenizerProcessor",
                                   "sampling_rate": getattr(ap, "sampling_rate", self.sampling_rate),
                                   "normalize_audio": getattr(ap, "normalize_audio", True),
                                   "target_dB_FS": getattr(ap, "target_dB_FS", -25), "eps": getattr(ap, "eps", 1e-6)}}
        with open(os.path.join(save_directory, "preprocessor_config.json"), "w") as fh:
            json.dump(cfg, fh, indent=2)

    def __call__(self, *args, **kwargs):
        raise NotImplementedError("VibeVoiceStreamingProcessor.__call__ is not implemented. "
                                  "Use process_input_with_cached_prompt for streaming inputs.")

    def process_input_with_cached_prompt(self, text: Optional[str] = None, cached_prompt: Optional[Dict[str, Any]] = None, padding=True,
                                         truncation=False, max_length: Optional[int] = None, return_tensors=None,
                                         return_attention_mask: bool = True, **kwargs) -> BatchEncoding:
        """One text and its cached prompt -> `input_ids` / `tts_lm_input_ids` (`pad_id` placeholders as long as the prompt's `lm` /
        `tts_lm` outputs), `tts_text_ids` = `encode(text.strip() + "\\n")` without special tokens, the two attention masks (all ones),
        `speech_input_mask` (all False) and `speech_tensors = speech_masks = None`.  A batch of one: `padding`, `truncation` and
        `max_length` have nothing to act on."""
        tok = self.tokenizer
        text_ids = tok.encode(text.strip() + "\n", add_special_tokens=False)
        n_lm = int(cached_prompt["lm"]["last_hidden_state"].size(1))
        n_tts = int(cached_prompt["tts_lm"]["last_hidden_state"].size(1))
        cols = {"input_ids": [[tok.pad_id] * n_lm], "tts_lm_input_ids": [[tok.pad_id] * n_tts], "tts_text_ids": [list(text_ids)]}
        if return_attention_mask:
            cols["attention_mask"] = [[1] * n_lm]
            cols["tts_lm_attention_mask"] = [[1] * n_tts]
        out = BatchEncoding()
        for k, v in cols.items():
            out[k] = torch.tensor(v, dtype=torch.long) if return_tensors is not None else v
        out["speech_input_mask"] = torch.zeros(1, n_tts, dtype=torch.bool) if return_tensors is not None else [[False] * n_tts]
        out["speech_tensors"] = out["speech_masks"] = None
        return out

    save_audio = VibeVoiceProcessor.save_audio
    batch_decode = VibeVoiceProcessor.batch_decode
    decode = VibeVoiceProcessor.decode
