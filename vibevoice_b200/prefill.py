"""Prompt prefill (SURVEY a-9 / f-2): the one-time, tensor-core-bound part of `generate()` step 0
(`modeling_vibevoice_inference.py:467-482`), kept on PyTorch library kernels for now (cuBLAS GEMMs + SDPA)
exactly as SURVEY 8(a-9) scopes it; the per-frame loop never touches this module.

It runs the Qwen2 stack over the whole prompt in bf16 (what the CUDA reference does, `demo/inference_from_file.py:288`),
hands each layer's K/V to the engine's paged pool through `vv_kv_write`, and returns the final-norm hidden state of the
last prompt token of every row so the first token decision uses the same `vv_lm_head` kernel as every later step.
"""
from __future__ import annotations

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
