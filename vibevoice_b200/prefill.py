"""Prompt prefill (SURVEY a-9 / f-2): the one-time, tensor-core-bound part of `generate()` step 0
(`modeling_vibevoice_inference.py:467-482`), kept on PyTorch library kernels for now (cuBLAS GEMMs + SDPA)
exactly as SURVEY 8(a-9) scopes it; the per-frame loop never touches this module.

It runs the Qwen2 stack over the whole prompt in bf16 (what the CUDA reference does, `demo/inference_from_file.py:288`),
hands each layer's K/V to the engine's paged pool through `vv_kv_write`, and returns the final-norm hidden state of the
last prompt token of every row so the first token decision uses the same `vv_lm_head` kernel as every later step.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

LM = "model.language_model"


class TorchPrefill:
    def __init__(self, config, state_dict: Dict[str, torch.Tensor], device):
        self.dc = config.decoder_config
        self.device = device
        self.w = {k: v.to(device=device, dtype=torch.bfloat16) for k, v in state_dict.items() if k.startswith(LM + ".")}

    def _rms(self, x, w, eps):
        xf = x.float()
        return (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).to(x.dtype) * w

    @torch.no_grad()
    def run(self, engine, seq: int, embeds: torch.Tensor, chunk: int = 1 << 30) -> torch.Tensor:
        """embeds [L, H] (any float dtype, on device) for ONE row -> writes KV for positions [0, L) of sequence `seq`,
        returns final-norm hidden of the last position, fp32 [H]."""
        dc, w = self.dc, self.w
        L = embeds.shape[0]
        nh, nkv, hd = dc.num_attention_heads, dc.num_key_value_heads, dc.head_dim
        x = embeds.to(torch.bfloat16)
        inv_freq = 1.0 / (dc.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float() / hd)).to(self.device)
        pos = torch.arange(L, device=self.device)
        ang = pos.float()[:, None] * inv_freq[None]
        emb = torch.cat([ang, ang], -1)
        cos, sin = emb.cos().to(torch.bfloat16)[:, None, :], emb.sin().to(torch.bfloat16)[:, None, :]

        def rope(t):
            t1, t2 = t[..., : hd // 2], t[..., hd // 2:]
            return t * cos + torch.cat([-t2, t1], -1) * sin

        for l in range(dc.num_hidden_layers):
            p = f"{LM}.layers.{l}"
            h = self._rms(x, w[f"{p}.input_layernorm.weight"], dc.rms_norm_eps)
            q = F.linear(h, w[f"{p}.self_attn.q_proj.weight"], w[f"{p}.self_attn.q_proj.bias"]).view(L, nh, hd)
            k = F.linear(h, w[f"{p}.self_attn.k_proj.weight"], w[f"{p}.self_attn.k_proj.bias"]).view(L, nkv, hd)
            v = F.linear(h, w[f"{p}.self_attn.v_proj.weight"], w[f"{p}.self_attn.v_proj.bias"]).view(L, nkv, hd)
            q, k = rope(q), rope(k)
            engine.kv_write(seq, l, 0, k.contiguous(), v.contiguous())
            out = torch.empty(L, nh, hd, dtype=torch.bfloat16, device=self.device)
            kt, vt = k.transpose(0, 1)[None], v.transpose(0, 1)[None]          # [1, nkv, L, hd]
            for s in range(0, L, chunk):
                e = min(L, s + chunk)
                qc = q[s:e].transpose(0, 1)[None]                               # [1, nh, c, hd]
                if s == 0:
                    o = F.scaled_dot_product_attention(qc, kt[:, :, :e], vt[:, :, :e], is_causal=True, enable_gqa=True)
                else:
                    m = pos[s:e, None] >= pos[None, :e]
                    o = F.scaled_dot_product_attention(qc, kt[:, :, :e], vt[:, :, :e], attn_mask=m, enable_gqa=True)
                out[s:e] = o[0].transpose(0, 1)
            x = x + F.linear(out.reshape(L, nh * hd), w[f"{p}.self_attn.o_proj.weight"])
            h = self._rms(x, w[f"{p}.post_attention_layernorm.weight"], dc.rms_norm_eps)
            g = F.silu(F.linear(h, w[f"{p}.mlp.gate_proj.weight"])) * F.linear(h, w[f"{p}.mlp.up_proj.weight"])
            x = x + F.linear(g, w[f"{p}.mlp.down_proj.weight"])
        last = x[-1:].float()
        last = last * torch.rsqrt(last.pow(2).mean(-1, keepdim=True) + dc.rms_norm_eps) * w[f"{LM}.norm.weight"].float()
        return last[0]


class TorchVoicePrompt:
    """Voice-prompt half of step 0 (`modeling_vibevoice_inference.py:149-163, 216-224`): acoustic tokenizer ENCODER over the 24 kHz
    reference wavs (non-streaming `TokenizerEncoder.forward`, `modular_vibevoice_tokenizer.py:384-418, 776-813`), Gaussian sampling
    (`:980-989`: std = randn(n)*fix_std/0.8, x = mean + std*randn_like(mean)), (x + bias)*scale, `acoustic_connector`
    (`modeling_vibevoice.py:58-69`).  PyTorch library kernels, fp32 -- once per request."""

    ENC = "model.acoustic_tokenizer.encoder"
    CON = "model.acoustic_connector"

    def __init__(self, config, state_dict: Dict[str, torch.Tensor], device):
        self.tc = config.acoustic_tokenizer_config
        self.device = device
        self.w = {k: v.to(device=device, dtype=torch.float32) for k, v in state_dict.items()
                  if k.startswith(self.ENC + ".") or k.startswith(self.CON + ".")}
        if not any(k.startswith(self.ENC) for k in self.w):
            raise ValueError("voice-prompt prefill needs the acoustic tokenizer encoder weights in the checkpoint")

    def _conv(self, name, x, stride=1, groups=1):
        wt, bs = self.w[name + ".conv.conv.weight"], self.w[name + ".conv.conv.bias"]
        k = wt.shape[-1]
        pad_total = (k - 1) - (stride - 1)
        length = x.shape[-1]
        n_frames = (length - k + pad_total) / stride + 1
        ideal = (math.ceil(n_frames) - 1) * stride + (k - pad_total)
        return F.conv1d(F.pad(x, (pad_total, ideal - length)), wt, bs, stride=stride, groups=groups)

    @staticmethod
    def _rms_c(x, w, eps):
        y = x.transpose(1, 2)
        y = y * torch.rsqrt(y.pow(2).mean(-1, keepdim=True) + eps) * w
        return y.transpose(1, 2)

    @torch.no_grad()
    def encode_mean(self, wavs: torch.Tensor) -> torch.Tensor:
        """wavs [n, T] -> latent means [n, ceil(T/3200), vae_dim]"""
        # cuDNN may run fp32 convolutions in TF32 unless told otherwise; the encoder is meant to be fp32
        cd = torch.backends.cudnn
        with cd.flags(enabled=cd.enabled, benchmark=cd.benchmark, deterministic=cd.deterministic, allow_tf32=False):
            return self._encode_mean(wavs)

    def _encode_mean(self, wavs: torch.Tensor) -> torch.Tensor:
        tc, p, w = self.tc, self.ENC, self.w
        x = wavs.to(self.device, torch.float32)[:, None, :]
        depths, ratios = tc.encoder_depth_list, list(reversed(tc.encoder_ratios))
        for i in range(len(depths)):
            x = self._conv(f"{p}.downsample_layers.{i}.0", x, stride=1 if i == 0 else ratios[i - 1])
            for j in range(depths[i]):
                q = f"{p}.stages.{i}.{j}"
                y = self._conv(f"{q}.mixer.conv", self._rms_c(x, w[f"{q}.norm.weight"], tc.layernorm_eps), groups=x.shape[1])
                x = x + y * w[f"{q}.gamma"][None, :, None]
                y = self._rms_c(x, w[f"{q}.ffn_norm.weight"], tc.layernorm_eps).permute(0, 2, 1)
                y = F.gelu(F.linear(y, w[f"{q}.ffn.linear1.weight"], w[f"{q}.ffn.linear1.bias"]))
                y = F.linear(y, w[f"{q}.ffn.linear2.weight"], w[f"{q}.ffn.linear2.bias"]).permute(0, 2, 1)
                x = x + y * w[f"{q}.ffn_gamma"][None, :, None]
        return self._conv(f"{p}.head", x).permute(0, 2, 1)

    @torch.no_grad()
    def __call__(self, speech_tensors: torch.Tensor, speech_masks: torch.Tensor, scale: float, bias: float, noise=None):
        """-> connected embeddings [sum(speech_masks), H] in row-major mask order.  `noise=(std_noise [n], eps [n,F,D])` overrides the
        device RNG draws (tests)."""
        mean = self.encode_mean(speech_tensors)
        n = mean.shape[0]
        value = float(self.tc.fix_std) / 0.8
        if self.tc.std_dist_type == "gaussian":
            std_n = torch.randn(n, device=self.device) if noise is None else noise[0].to(self.device)
            eps = torch.randn_like(mean) if noise is None else noise[1].to(self.device)
            x = mean + (std_n * value)[:, None, None] * eps
        elif self.tc.std_dist_type == "fix":
            eps = torch.randn_like(mean) if noise is None else noise[1].to(self.device)
            x = mean + float(self.tc.fix_std) * eps
        else:
            x = mean
        feat = (x + bias) * scale
        c = self.CON
        y = F.linear(feat, self.w[f"{c}.fc1.weight"], self.w[f"{c}.fc1.bias"])
        y = y * torch.rsqrt(y.pow(2).mean(-1, keepdim=True) + 1e-6) * self.w[f"{c}.norm.weight"]
        y = F.linear(y, self.w[f"{c}.fc2.weight"], self.w[f"{c}.fc2.bias"])
        return y[speech_masks.to(self.device)]
