"""CPU ORACLE (TEST INFRASTRUCTURE) for the streaming-0.5B variant -- SURVEY 8f-1, the first "next" row.

Restates `VibeVoiceStreamingForConditionalGenerationInference.generate`
(reference vibevoice/modular/modeling_vibevoice_streaming_inference.py:412-725) on a flat state dict with the reference's key
names, reusing the arithmetic of `vv_oracle` (Qwen2 stack, diffusion head + DPM-Solver++, streaming acoustic decoder, connector).
Pinned against the reference's own generate() on a synthetic checkpoint: `tests/golden/streaming.pt` (`oracle/make_golden.py::
gen_streaming`), held by `tests/test_oracle_golden.py::test_streaming_generate_matches_the_reference`.

Model (modeling_vibevoice_streaming.py:108-160): the Qwen2 stack is split -- `language_model` = lower N-T layers, no final norm
(text only); `tts_language_model` = upper T layers + final norm; `tts_input_types` [2,H] is added to every TTS-LM input (1 = text,
0 = speech); `tts_eos_classifier` = Linear-ReLU-Linear on the last TTS-LM hidden state; no semantic tokenizer, no lm_head.

Loop (:553-702), batch 1: per window of 5 text tokens (:40-41) run the lower stack on the tokens, then the upper stack on the lower
stack's outputs (+ type 1); then 6 speech frames (:42): CFG sampler conditioned on the last TTS-LM hidden state of the positive and
the negative stream -> acoustic decoder frame -> connector -> one TTS-LM step (+ type 0) on both streams -> EOS classifier.
Frames computed after EOS fired inside a window are not kept (:630-634).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
from torch import Tensor

from . import vv_oracle as O

TEXT_WINDOW, SPEECH_WINDOW = 5, 6                      # TTS_TEXT_WINDOW_SIZE, TTS_SPEECH_WINDOW_SIZE (:40-42)
LM, TTS = "model.language_model", "model.tts_language_model"


def streaming_state_dict(base: Dict[str, Tensor], cfg, tts_layers: int, seed: int = 99, eos_bias: float = -0.3) -> Dict[str, Tensor]:
    """Synthetic streaming checkpoint from a synthetic multi-speaker one (`vibevoice_b200.synth.synth_state_dict`): same tensors
    under the streaming model's key names (lower layers -> language_model, upper -> tts_language_model, final norm -> the upper
    stack), semantic parts dropped, plus the three streaming-only modules drawn from `seed`."""
    nl = cfg.decoder_config.num_hidden_layers
    low = nl - tts_layers
    H = cfg.decoder_config.hidden_size
    sd: Dict[str, Tensor] = {}
    for k, v in base.items():
        if k.startswith("model.semantic") or k.startswith("lm_head"):
            continue
        if k.startswith(LM + ".layers."):
            parts = k.split(".")
            i, rest = int(parts[3]), ".".join(parts[4:])
            sd[f"{LM}.layers.{i}.{rest}" if i < low else f"{TTS}.layers.{i - low}.{rest}"] = v
        elif k == LM + ".norm.weight":
            sd[TTS + ".norm.weight"] = v
        else:
            sd[k] = v
    g = torch.Generator().manual_seed(seed)
    sd[TTS + ".embed_tokens.weight"] = base[LM + ".embed_tokens.weight"].clone()      # present in the checkpoint, unused (:139)
    sd["model.tts_input_types.weight"] = torch.randn(2, H, generator=g) * 0.05
    sd["tts_eos_classifier.fc1.weight"] = torch.randn(H, H, generator=g) * 0.05
    sd["tts_eos_classifier.fc1.bias"] = torch.randn(H, generator=g) * 0.05
    sd["tts_eos_classifier.fc2.weight"] = torch.randn(1, H, generator=g) * 0.05
    sd["tts_eos_classifier.fc2.bias"] = torch.full((1,), float(eos_bias))
    return sd


def eos_logit(w, h: Tensor) -> Tensor:
    """`BinaryClassifier.forward` (modeling_vibevoice_streaming.py:42-53)."""
    x = torch.relu(h.float() @ w["tts_eos_classifier.fc1.weight"].float().T + w["tts_eos_classifier.fc1.bias"].float())
    return x @ w["tts_eos_classifier.fc2.weight"].float().T + w["tts_eos_classifier.fc2.bias"].float()


class Streams:
    """The four KV streams of the loop (`all_prefilled_outputs`, :517-534) and the last hidden state of the two TTS-LM streams."""

    def __init__(self, w, cfg, tts_layers: int, kv_bf16: bool = False):
        self.w, self.dc, self.t = w, cfg.decoder_config, tts_layers
        self.low = self.dc.num_hidden_layers - tts_layers
        mk = lambda n: O.KVCache(n, kv_bf16)
        self.lm, self.tts, self.neg_tts = mk(self.low), mk(tts_layers), mk(tts_layers)
        self.types = w["model.tts_input_types.weight"].float()
        self.h_pos: Optional[Tensor] = None
        self.h_neg: Optional[Tensor] = None

    def forward_lm(self, ids: Tensor, cache: O.KVCache) -> Tensor:                    # :178-238
        e = self.w[LM + ".embed_tokens.weight"][ids].float()
        return O.qwen2_forward(self.w, self.dc, e, cache, len(cache), p=LM, n_layers=self.low, final_norm=False)

    def forward_tts(self, x: Tensor, type_id: int, cache: O.KVCache) -> Tensor:       # :240-318 (inputs fully replaced by x, + type)
        return O.qwen2_forward(self.w, self.dc, x.float() + self.types[type_id], cache, len(cache), p=TTS, n_layers=self.t)


def prefill(st: Streams, prompt_ids: Tensor, neg_id: int):
    """What `all_prefilled_outputs` holds for a text-only prompt (the shipped voices carry these four outputs pre-computed,
    demo/streaming_inference_from_file.py:291): lower stack over the prompt, upper stack over its outputs (type 1); the negative
    streams see the single token <|image_pad|> (:475, :476-482)."""
    st.h_pos = st.forward_tts(st.forward_lm(prompt_ids, st.lm), 1, st.tts)
    neg_lm = O.KVCache(st.low, st.lm.kv_bf16)
    st.h_neg = st.forward_tts(st.forward_lm(torch.tensor([neg_id]), neg_lm), 1, st.neg_tts)


def generate_streaming(w, cfg, tts_layers: int, prompt_ids: Tensor, tts_text_ids: Tensor, neg_id: int, cfg_scale: float = 1.5,
                       num_steps: int = 5, max_new_tokens: Optional[int] = None, kv_bf16: bool = False) -> O.GenerateResult:
    """prompt_ids [L0], tts_text_ids [T] (one sample).  Returns sequences = `tts_lm_input_ids` (prompt, text windows, a 1 per speech
    frame, :643), the concatenated waveform, and the max-length flag."""
    dc, hc = cfg.decoder_config, cfg.diffusion_head_config
    st = Streams(w, cfg, tts_layers, kv_bf16)
    prefill(st, prompt_ids, neg_id)
    L0 = int(prompt_ids.numel())
    if max_new_tokens is None:
        max_new_tokens = dc.max_position_embeddings - L0                              # :472-473
    max_length = L0 + max_new_tokens                                                  # tts_lm_generation_config.max_length
    scale, bias = float(w["model.speech_scaling_factor"]), float(w["model.speech_bias_factor"])
    a_state = O.StreamState(1)
    row = torch.tensor([0])
    seq: List[int] = prompt_ids.tolist()
    chunks: List[Tensor] = []
    finished, reach_max, win = False, False, 0
    while True:
        if finished:                                                                  # :563-566
            break
        cur = tts_text_ids[win * TEXT_WINDOW:(win + 1) * TEXT_WINDOW]                  # :568-570
        win += 1
        if cur.numel() > 0:
            seq += cur.tolist()
            if len(seq) > max_length:                                                 # :576-582
                reach_max = True
                break
            st.h_pos = st.forward_tts(st.forward_lm(cur, st.lm), 1, st.tts)            # :590-611
        for _ in range(SPEECH_WINDOW):                                                # :614
            noise = torch.randn(2, cfg.acoustic_vae_dim)                              # :741 (CPU global generator)
            lat = O.sample_speech_tokens(w, st.h_pos[-1:], st.h_neg[-1:], cfg_scale, num_steps, noise, hc.head_layers, hc.rms_norm_eps)
            audio = O.decoder_frame(w, cfg.acoustic_tokenizer_config, (lat / scale - bias)[:, None, :], a_state, row)   # :624-632
            if not finished:                                                          # :634-638
                chunks.append(audio[0])
            emb = O.connector(w, "model.acoustic_connector", lat)                     # :645
            seq.append(1)                                                             # :646
            if len(seq) > max_length:                                                 # :648-649
                break
            st.h_pos = st.forward_tts(emb, 0, st.tts)                                 # :657-667
            st.h_neg = st.forward_tts(emb, 0, st.neg_tts)                             # :677-689
            if torch.sigmoid(eos_logit(w, st.h_pos[-1:]))[0, 0].item() > 0.5:          # :691-696
                finished = True
        if len(seq) > max_length:                                                     # :698-704
            reach_max = not finished
            break
    out = torch.cat(chunks, dim=-1) if chunks else None
    return O.GenerateResult(torch.tensor([seq]), [out], torch.tensor([reach_max]))
