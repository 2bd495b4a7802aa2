"""Device engine: owns one `vv_ctx` (C ABI, `include/vibevoice_b200.h`), the persistent I/O buffers the
captured CUDA graphs are bound to, and the stream they run on.  Pure plumbing -- all arithmetic is in
`csrc/` (hand-written sm_90a kernels).  PyTorch is used for device memory and streams only.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Iterable, Optional, Tuple

import numpy as np
import torch

from . import _native as N
from .configuration import VibeVoiceConfig
from .schedule import DPMSolverMultistepScheduler

_DT = {torch.bfloat16: N.VV_DT_BF16, torch.float32: N.VV_DT_F32, torch.float16: N.VV_DT_F16}


def _desc_from_config(cfg: VibeVoiceConfig, valid_ids, max_batch: int, max_steps: int) -> N.ModelDesc:
    dc, hc = cfg.decoder_config, cfg.diffusion_head_config
    ac, sc = cfg.acoustic_tokenizer_config, cfg.semantic_tokenizer_config
    d = N.ModelDesc()
    d.hidden_size, d.intermediate_size, d.num_layers = dc.hidden_size, dc.intermediate_size, dc.num_hidden_layers
    d.num_q_heads, d.num_kv_heads, d.head_dim, d.vocab_size = dc.num_attention_heads, dc.num_key_value_heads, dc.head_dim, dc.vocab_size
    d.max_position_embeddings, d.tie_word_embeddings = dc.max_position_embeddings, int(bool(dc.tie_word_embeddings))
    d.rms_norm_eps, d.rope_theta = dc.rms_norm_eps, dc.rope_theta
    d.head_layers, d.head_ffn_dim, d.latent_size = hc.head_layers, int(hc.hidden_size * hc.head_ffn_ratio), hc.latent_size
    d.head_rms_eps = hc.rms_norm_eps
    dec_depths, enc_depths = ac.decoder_depth_list, sc.encoder_depth_list
    if len(dec_depths) != len(enc_depths) or list(ac.decoder_ratios) != list(sc.encoder_ratios):
        raise ValueError("acoustic decoder and semantic encoder must share the stage / ratio structure")
    d.n_stages = len(dec_depths)
    for i, r in enumerate(ac.decoder_ratios):
        d.dec_ratios[i] = r
    for i, r in enumerate(sc.encoder_ratios):
        d.enc_ratios[i] = r
    for i, v in enumerate(dec_depths):
        d.dec_depths[i] = v
    for i, v in enumerate(enc_depths):
        d.enc_depths[i] = v
    d.dec_n_filters, d.enc_n_filters = ac.decoder_n_filters, sc.encoder_n_filters
    d.acoustic_vae_dim, d.semantic_vae_dim, d.codec_eps = ac.vae_dim, sc.vae_dim, ac.layernorm_eps
    if ac.layernorm_eps != sc.layernorm_eps:
        raise ValueError("codec eps mismatch")
    valid_ids = sorted(set(int(v) for v in valid_ids))
    d.n_valid_ids = len(valid_ids)
    for i, v in enumerate(valid_ids):
        d.valid_ids[i] = v
    d.max_batch, d.max_diffusion_steps = max_batch, max_steps
    return d


class Engine:
    """One GPU's worth of VibeVoice: weights, paged KV, codec state, per-frame programs."""

    def __init__(self, config: VibeVoiceConfig, valid_ids, max_batch: int = 1, device: int = 0, max_diffusion_steps: int = 64):
        if not torch.cuda.is_available():
            raise N.VVError("vibevoice_b200 needs a CUDA device (sm_90a); there is no CPU path")
        self.lib = N.load_library()
        if self.lib.vv_abi_version() != 1:
            raise N.VVError("ABI mismatch")
        self.config = config
        self.B = max_batch
        self.device = torch.device("cuda", device)
        self.valid_ids = sorted(set(int(v) for v in valid_ids))
        self.desc = _desc_from_config(config, valid_ids, max_batch, max_diffusion_steps)
        h = C.c_void_p()
        N.check(self.lib.vv_create(C.byref(self.desc), device, C.byref(h)), "vv_create")
        self.h = h
        self.finalized = False
        self.kv_pages = 0
        self.stream = torch.cuda.Stream(device=self.device)
        H, B = config.decoder_config.hidden_size, max_batch
        dev = self.device
        with torch.cuda.device(dev):
            self.embeds = torch.zeros(2 * B, H, dtype=torch.float32, device=dev)
            self.hidden = torch.zeros(2 * B, H, dtype=torch.float32, device=dev)
            self.logits = torch.zeros(B, len(self.valid_ids), dtype=torch.float32, device=dev)
            self.tokens = torch.zeros(B, dtype=torch.int32, device=dev)
            self.noise = torch.zeros(B, 64, dtype=torch.float32, device=dev)
            self.active = torch.zeros(B, dtype=torch.int32, device=dev)
            self.latent = torch.zeros(B, 64, dtype=torch.float32, device=dev)
            self.audio = torch.zeros(B, 3200, dtype=torch.float32, device=dev)
            self.feat = torch.zeros(B, config.semantic_vae_dim, dtype=torch.float32, device=dev)
        self.tokens_h = torch.zeros(B, dtype=torch.int32).pin_memory()
        self.logits_h = torch.zeros(B, len(self.valid_ids), dtype=torch.float32).pin_memory()
        self.noise_h = torch.zeros(B, 64, dtype=torch.float32).pin_memory()
        self.active_h = torch.zeros(B, dtype=torch.int32).pin_memory()
        self.n_steps = 0
        self.step_noise = None
        self.scheduler = DPMSolverMultistepScheduler(
            num_train_timesteps=config.diffusion_head_config.ddpm_num_steps,
            beta_schedule=config.diffusion_head_config.ddpm_beta_schedule,
            prediction_type=config.diffusion_head_config.prediction_type)

    # ---- lifetime -------------------------------------------------------------------------------
    def close(self):
        if getattr(self, "h", None) is not None and self.h:
            torch.cuda.synchronize(self.device)
            self.lib.vv_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def s(self):
        return C.c_void_p(self.stream.cuda_stream)

    # ---- weights ----------------------------------------------------------------------------------
    def load_tensor(self, name: str, t: torch.Tensor) -> int:
        if t.dtype not in _DT:
            t = t.float()
        t = t.contiguous()
        shape = (C.c_int64 * max(t.dim(), 1))(*t.shape)
        rc = self.lib.vv_load_tensor(self.h, name.encode(), C.c_void_p(t.data_ptr()), _DT[t.dtype], shape, t.dim())
        return N.check(rc, "vv_load_tensor(%s)" % name)

    def load_state_dict(self, items: Iterable[Tuple[str, torch.Tensor]]):
        n = 0
        for name, t in items:
            self.load_tensor(name, t)
            n += 1
        return n

    def finalize(self, speech_scaling_factor: Optional[float] = None, speech_bias_factor: Optional[float] = None):
        if speech_scaling_factor is not None:
            N.check(self.lib.vv_set_speech_factors(self.h, float(speech_scaling_factor), float(speech_bias_factor)))
        N.check(self.lib.vv_finalize_weights(self.h), "vv_finalize_weights")
        self.finalized = True
        # Qwen2RotaryEmbedding.inv_freq exactly as torch computes it (fp32)
        dc = self.config.decoder_config
        inv = 1.0 / (dc.rope_theta ** (torch.arange(0, dc.head_dim, 2, dtype=torch.int64).float() / dc.head_dim))
        inv = inv.contiguous()
        N.check(self.lib.vv_set_rope_inv_freq(self.h, C.c_void_p(inv.data_ptr()), inv.numel()))

    def weight_bytes(self) -> Dict[str, int]:
        names = ["lm", "head_step", "cond_proj", "decoder", "semantic", "connectors"]
        return {n: int(self.lib.vv_weight_bytes(self.h, i)) for i, n in enumerate(names)}

    # ---- a-9 voice prompts ------------------------------------------------------------------------------
    def voice_frames(self, n_samples: int) -> int:
        """latent frames the acoustic encoder makes of `n_samples` (one per hop of prod(ratios) samples, the last one partial)."""
        hop = int(np.prod(self.config.acoustic_tokenizer_config.encoder_ratios))
        return -(-int(n_samples) // hop)

    def voice_workspace_bytes(self, n_voices: int, n_samples: int) -> int:
        """minimum workspace of `voice_encode`; raises if the checkpoint had no acoustic encoder."""
        return N.check(int(self.lib.vv_voice_encode_workspace(self.h, int(n_voices), int(n_samples))), "vv_voice_encode_workspace")

    def voice_encode(self, wavs: torch.Tensor, sigma: torch.Tensor, eps: Optional[torch.Tensor], mean_out: Optional[torch.Tensor] = None,
                     workspace_bytes: Optional[int] = None) -> torch.Tensor:
        """wavs [n, T], sigma [n], eps [n, F, vae_dim] or None -> connected embeddings [n, F, H] fp32 on the device (`vv_voice_encode`).
        The default workspace fits every voice at once plus 256 MB of GEMM scratch, within 2 GB unless the minimum is larger."""
        n, T = wavs.shape
        need = self.voice_workspace_bytes(n, T)
        ws = int(workspace_bytes) if workspace_bytes is not None else min(need * n + (256 << 20), max(need, 2 << 30))
        F, H = self.voice_frames(T), self.config.decoder_config.hidden_size
        cur = torch.cuda.current_stream(self.device)
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            wavs = wavs.to(self.device, torch.float32).contiguous()
            sigma = sigma.to(self.device, torch.float32).contiguous()
            eps = None if eps is None else eps.to(self.device, torch.float32).contiguous()
            out = torch.empty(n, F, H, dtype=torch.float32, device=self.device)
            work = torch.empty(max(ws, 1), dtype=torch.uint8, device=self.device)
            P = lambda t: C.c_void_p(None if t is None else t.data_ptr())
            N.check(self.lib.vv_voice_encode(self.h, P(wavs), n, T, P(sigma), P(eps), P(mean_out), P(out), P(work), ws, self.s),
                    "vv_voice_encode")
        cur.wait_stream(self.stream)
        return out

    def voice_taps(self, wavs: torch.Tensor, sigma: torch.Tensor, eps: Optional[torch.Tensor], workspace_bytes: Optional[int] = None):
        """`voice_encode` with every stage boundary copied out (`vv_debug_voice_taps`, tests), on `voice_encode`'s default workspace unless
        one is given.  Returns ([(meta, tap)], embeds): meta = (kind, stage, index, T, C), tap = [n, T, C] fp32 on the device (a 10 s voice
        at full width has about 0.8 GB of taps); embeds [n, F, H]."""
        n, T = wavs.shape
        need = self.voice_workspace_bytes(n, T)
        ws = int(workspace_bytes) if workspace_bytes is not None else min(need * n + (256 << 20), max(need, 2 << 30))
        F, H = self.voice_frames(T), self.config.decoder_config.hidden_size
        P = lambda t: C.c_void_p(None if t is None else t.data_ptr())
        call = lambda w, s, e, out, work, taps, nt, meta, st: self.lib.vv_debug_voice_taps(self.h, w, n, T, s, e, out, work, ws, taps, nt, meta, st)
        k = N.check(call(None, None, None, None, None, None, 0, None, None), "vv_debug_voice_taps")
        meta = np.zeros((k, 5), dtype=np.int32)
        N.check(call(None, None, None, None, None, None, 0, N.iptr(meta), None), "vv_debug_voice_taps")
        sizes = [n * int(t) * int(c) for t, c in meta[:, 3:]]
        cur = torch.cuda.current_stream(self.device)
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            wavs = wavs.to(self.device, torch.float32).contiguous()
            sigma = sigma.to(self.device, torch.float32).contiguous()
            eps = None if eps is None else eps.to(self.device, torch.float32).contiguous()
            out = torch.empty(n, F, H, dtype=torch.float32, device=self.device)
            work = torch.empty(max(ws, 1), dtype=torch.uint8, device=self.device)
            taps = torch.empty(sum(sizes), dtype=torch.float32, device=self.device)
            N.check(call(P(wavs), P(sigma), P(eps), P(out), P(work), P(taps), taps.numel(), None, self.s), "vv_debug_voice_taps")
        cur.wait_stream(self.stream)
        res, off = [], 0
        for m, sz in zip(meta.tolist(), sizes):
            res.append((tuple(m), taps[off:off + sz].view(n, m[3], m[4])))
            off += sz
        return res, out

    # ---- f-2 native prompt prefill ---------------------------------------------------------------------
    def lm_prefill_workspace_bytes(self, n_tokens: int) -> int:
        """minimum workspace of `lm_prefill` (one 64-row chunk)."""
        return N.check(int(self.lib.vv_lm_prefill_workspace(self.h, int(n_tokens))), "vv_lm_prefill_workspace")

    def lm_prefill(self, seq: int, embeds: torch.Tensor, pos0: int = 0, workspace_bytes: Optional[int] = None) -> torch.Tensor:
        """embeds [n, H] (prompt rows of sequence `seq` at positions pos0..pos0+n) -> final-norm hidden of the last row, fp32 [H] on the device
        (`vv_lm_prefill`).  K/V land in the paged pool; the caller sets the length with `kv_set_len`.  The default workspace fits the whole
        prompt in one chunk, within 2 GB unless the minimum is larger (the `voice_encode` rule)."""
        n = int(embeds.shape[0])
        need = self.lm_prefill_workspace_bytes(n)
        ws = int(workspace_bytes) if workspace_bytes is not None else min(need * ((n + 63) // 64), max(need, 2 << 30))
        cur = torch.cuda.current_stream(self.device)
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            e = embeds.to(self.device, torch.float32).contiguous()
            out = torch.empty(self.config.decoder_config.hidden_size, dtype=torch.float32, device=self.device)
            work = torch.empty(max(ws, 1), dtype=torch.uint8, device=self.device)
            N.check(self.lib.vv_lm_prefill(self.h, int(seq), int(pos0), n, C.c_void_p(e.data_ptr()), C.c_void_p(out.data_ptr()),
                                           C.c_void_p(work.data_ptr()), ws, self.s), "vv_lm_prefill")
        cur.wait_stream(self.stream)
        return out

    def prefill_taps(self, seq: int, layer: int, x: torch.Tensor, pos0: int = 0, workspace_bytes: Optional[int] = None):
        """Decoder layer `layer` of `lm_prefill` alone on the residual input x [n, H] at positions pos0..pos0+n of sequence `seq`, with each
        kernel's output copied out (`vv_debug_prefill_taps`, tests).  K/V land in the pool as in `lm_prefill`; the default workspace is
        `lm_prefill`'s.  Returns ([(meta, tap)], hidden_last): meta = (kind, bytes per element, cols), tap = [n, cols] bf16 / fp32 on the
        device; hidden_last [H] = the final-norm hidden state of the last output row."""
        n = int(x.shape[0])
        need = self.lm_prefill_workspace_bytes(n)
        ws = int(workspace_bytes) if workspace_bytes is not None else min(need * ((n + 63) // 64), max(need, 2 << 30))
        P = lambda t: C.c_void_p(None if t is None else t.data_ptr())
        call = lambda xin, hl, work, w, taps, tb, meta, s: self.lib.vv_debug_prefill_taps(self.h, int(seq), int(pos0), n, int(layer), xin, hl, work,
                                                                                          w, taps, tb, meta, s)
        k = N.check(call(None, None, None, 0, None, 0, None, None), "vv_debug_prefill_taps")
        meta = np.zeros((k, 3), dtype=np.int32)
        N.check(call(None, None, None, 0, None, 0, N.iptr(meta), None), "vv_debug_prefill_taps")
        sizes = [n * int(b) * int(c) for _, b, c in meta.tolist()]
        cur = torch.cuda.current_stream(self.device)
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            e = x.to(self.device, torch.float32).contiguous()
            hl = torch.empty(self.config.decoder_config.hidden_size, dtype=torch.float32, device=self.device)
            work = torch.empty(max(ws, 1), dtype=torch.uint8, device=self.device)
            taps = torch.empty(sum(sizes), dtype=torch.uint8, device=self.device)
            N.check(call(P(e), P(hl), P(work), ws, P(taps), taps.numel(), None, self.s), "vv_debug_prefill_taps")
        cur.wait_stream(self.stream)
        out, off = [], 0
        for m, sz in zip(meta.tolist(), sizes):
            out.append((tuple(m), taps[off:off + sz].view(torch.bfloat16 if m[1] == 2 else torch.float32).view(n, m[2])))
            off += sz
        return out, hl

    def embed_gather(self, ids) -> torch.Tensor:
        """token ids (any count) -> embedding rows [n, H] fp32 on the device (`vv_embed_gather`)."""
        ids = torch.as_tensor(ids).reshape(-1)
        V = self.config.decoder_config.vocab_size
        if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= V):
            raise ValueError("token id outside [0, %d)" % V)
        cur = torch.cuda.current_stream(self.device)
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            d = ids.to(self.device, torch.int32).contiguous()
            out = torch.empty(d.numel(), self.config.decoder_config.hidden_size, dtype=torch.float32, device=self.device)
            N.check(self.lib.vv_embed_gather(self.h, C.c_void_p(d.data_ptr()), d.numel(), C.c_void_p(out.data_ptr()), self.s), "vv_embed_gather")
        cur.wait_stream(self.stream)
        return out

    def kv_read(self, seq: int, layer: int, pos0: int, n: int):
        """K, V [n, kv_heads, head_dim] bf16 of positions [pos0, pos0 + n) of (seq, layer) (`vv_debug_kv_read`, tests)."""
        dc = self.config.decoder_config
        with torch.cuda.stream(self.stream):
            k = torch.empty(n, dc.num_key_value_heads, dc.head_dim, dtype=torch.bfloat16, device=self.device)
            v = torch.empty_like(k)
            N.check(self.lib.vv_debug_kv_read(self.h, int(seq), int(layer), int(pos0), int(n), C.c_void_p(k.data_ptr()), C.c_void_p(v.data_ptr()),
                                              self.s), "vv_debug_kv_read")
        self.stream.synchronize()
        return k, v

    # ---- KV -----------------------------------------------------------------------------------------
    def kv_init(self, total_tokens: int):
        pages = (total_tokens + 63) // 64 + 2 * self.B * 2
        N.check(self.lib.vv_kv_init(self.h, pages), "vv_kv_init")
        self.kv_pages = pages

    def kv_len(self, seq: int) -> int:
        return int(self.lib.vv_kv_len(self.h, seq))

    def kv_set_len(self, seq: int, n: int):
        N.check(self.lib.vv_kv_set_len(self.h, seq, n, self.s), "vv_kv_set_len")

    def kv_delete(self, seq: int, pos: int):
        """forget the committed entry at `pos` (the last entry takes its place)."""
        N.check(self.lib.vv_kv_delete_slot(self.h, seq, pos, self.s), "vv_kv_delete_slot")

    def kv_commit(self, advance):
        a = N.i32(advance)
        N.check(self.lib.vv_kv_commit(self.h, N.iptr(a), self.s), "vv_kv_commit")

    def kv_write(self, seq: int, layer: int, pos0: int, k: torch.Tensor, v: torch.Tensor):
        assert k.dtype == torch.bfloat16 and k.is_contiguous() and v.is_contiguous()
        N.check(self.lib.vv_kv_write(self.h, seq, layer, pos0, k.shape[0], C.c_void_p(k.data_ptr()), C.c_void_p(v.data_ptr()),
                                     self.s), "vv_kv_write")

    # ---- programs -------------------------------------------------------------------------------------
    @property
    def sde(self) -> bool:
        return getattr(self.scheduler.config, "algorithm_type", "dpmsolver++") == "sde-dpmsolver++"

    def set_scheduler(self, scheduler):
        """`model.model.noise_scheduler = scheduler.from_config(...)` (demo/gradio_demo.py:141-146) lands here."""
        self.scheduler = scheduler
        self.n_steps = 0                          # tables are rebuilt on the next set_diffusion_steps

    def set_diffusion_steps(self, n_steps: int):
        if n_steps == self.n_steps:
            return
        self.scheduler.set_timesteps(n_steps)
        ts = np.ascontiguousarray(self.scheduler.timesteps.numpy().astype(np.float32))
        coef = np.ascontiguousarray(self.scheduler.coef)
        if self.sde:
            if self.step_noise is None or self.step_noise.shape[0] < n_steps:
                with torch.cuda.device(self.device):
                    self.step_noise = torch.zeros(max(n_steps, 8), self.B, 64, dtype=torch.float32, device=self.device)
            N.check(self.lib.vv_set_diffusion_steps_sde(self.h, n_steps, N.iptr(ts), N.iptr(coef), self.s), "vv_set_diffusion_steps_sde")
            N.check(self.lib.vv_set_step_noise(self.h, C.c_void_p(self.step_noise.data_ptr())), "vv_set_step_noise")
        else:
            N.check(self.lib.vv_set_diffusion_steps(self.h, n_steps, N.iptr(ts), N.iptr(coef), self.s), "vv_set_diffusion_steps")
        self.n_steps = n_steps

    def upload_step_noise(self, draw, active_rows):
        """sde-dpmsolver++: the reference draws randn_tensor([2n,64]) once per solver step on the model's device (dpm_solver.py:993-997)
        and only rows [:n] reach the latent (:703-706); `draw(i)` returns that [2n,64] block for step i."""
        n = len(active_rows)
        rows = torch.as_tensor(list(active_rows), dtype=torch.long, device=self.step_noise.device)
        with torch.cuda.stream(self.stream):
            for i in range(self.n_steps):
                self.step_noise[i].index_copy_(0, rows, draw(i)[:n].to(self.step_noise.device, torch.float32))

    def embed_tokens(self, tokens, out: torch.Tensor):
        a = N.i32(tokens)
        N.check(self.lib.vv_embed_tokens(self.h, N.iptr(a), len(a), C.c_void_p(out.data_ptr()), self.s), "vv_embed_tokens")

    def lm_decode(self):
        """embeds -> hidden, logits, tokens (all persistent buffers)."""
        N.check(self.lib.vv_lm_decode(self.h, C.c_void_p(self.embeds.data_ptr()), C.c_void_p(self.hidden.data_ptr()),
                                      C.c_void_p(self.logits.data_ptr()), C.c_void_p(self.tokens.data_ptr()), self.s), "vv_lm_decode")

    def set_row_mode(self, modes):
        """rows (2B) with mode 0 neither read nor append KV in the next decode calls (include/vibevoice_b200.h: vv_set_row_mode)."""
        a = N.i32(modes)
        N.check(self.lib.vv_set_row_mode(self.h, N.iptr(a), self.s), "vv_set_row_mode")

    def lm_decode_range(self, layer_begin: int, layer_end: int, final_norm: bool, out: Optional[torch.Tensor] = None):
        """embeds -> `out` (default: hidden) through decoder layers [layer_begin, layer_end) only (streaming-0.5B split stack)."""
        out = self.hidden if out is None else out
        N.check(self.lib.vv_lm_decode_range(self.h, C.c_void_p(self.embeds.data_ptr()), int(layer_begin), int(layer_end), int(bool(final_norm)),
                                            C.c_void_p(out.data_ptr()), self.s), "vv_lm_decode_range")

    def lm_head(self, hidden: torch.Tensor):
        N.check(self.lib.vv_lm_head(self.h, C.c_void_p(hidden.data_ptr()), C.c_void_p(self.logits.data_ptr()),
                                    C.c_void_p(self.tokens.data_ptr()), self.s), "vv_lm_head")

    def lm_logits_full(self) -> torch.Tensor:
        """[B, vocab] fp32 logits of the positive rows from the current `hidden` (device tensor, valid after the call returns)."""
        if getattr(self, "_logits_full", None) is None:
            with torch.cuda.device(self.device):
                self._logits_full = torch.zeros(self.B, self.config.decoder_config.vocab_size, dtype=torch.float32, device=self.device)
        N.check(self.lib.vv_lm_logits_full(self.h, C.c_void_p(self.hidden.data_ptr()), C.c_void_p(self._logits_full.data_ptr()), self.s),
                "vv_lm_logits_full")
        self.stream.synchronize()
        return self._logits_full

    def read_tokens(self):
        """device -> pinned host, synchronising the engine stream (the one host sync per frame)."""
        with torch.cuda.stream(self.stream):
            self.tokens_h.copy_(self.tokens, non_blocking=True)
            self.logits_h.copy_(self.logits, non_blocking=True)
        self.stream.synchronize()
        return self.tokens_h.numpy(), self.logits_h.numpy()

    def upload_frame_inputs(self, noise_rows: torch.Tensor, active_rows):
        self.noise_h.zero_()
        self.active_h.zero_()
        for i, b in enumerate(active_rows):
            self.noise_h[b] = noise_rows[i]
            self.active_h[b] = 1
        with torch.cuda.stream(self.stream):
            self.noise.copy_(self.noise_h, non_blocking=True)
            self.active.copy_(self.active_h, non_blocking=True)

    # ---- zero-sync audio hand-off (SURVEY 8f-4): frames leave through a pinned ring, one frame behind the loop -------------------
    AUDIO_RING = 8

    def stage_audio(self, rows):
        """Enqueue an asynchronous copy of this frame's audio rows into the next slot of a pinned host ring (no synchronisation).
        Returns a ticket for `fetch_audio`; the data is valid after ANY later synchronisation of the engine stream (the loop's
        per-step token read-back already is one), so the streamer hand-off costs no sync of its own."""
        if getattr(self, "_ring_h", None) is None:
            self._ring_h = torch.zeros(self.AUDIO_RING, self.B, 3200, dtype=torch.float32).pin_memory()
            self._ring_ev = [torch.cuda.Event() for _ in range(self.AUDIO_RING)]
            self._ring_n = 0
        slot = self._ring_n % self.AUDIO_RING
        self._ring_n += 1
        with torch.cuda.stream(self.stream):
            self._ring_h[slot].copy_(self.audio, non_blocking=True)
            self._ring_ev[slot].record(self.stream)
        return slot, list(rows)

    def fetch_audio(self, ticket) -> torch.Tensor:
        """[n, 3200] CPU tensor of a staged frame (waits on that frame's event only -- already complete in the steady-state loop)."""
        slot, rows = ticket
        self._ring_ev[slot].synchronize()
        return self._ring_h[slot][rows].clone()

    def frame_tail(self, cfg_scale: float):
        P = lambda t: C.c_void_p(t.data_ptr())
        N.check(self.lib.vv_frame_tail(self.h, P(self.hidden), P(self.noise), P(self.active), float(cfg_scale), P(self.latent),
                                       P(self.audio), P(self.embeds), self.s), "vv_frame_tail")

    # individual stages (tests / profiling)
    def diffusion_sample(self, cfg_scale: float):
        P = lambda t: C.c_void_p(t.data_ptr())
        N.check(self.lib.vv_diffusion_sample(self.h, P(self.hidden), P(self.noise), P(self.active), float(cfg_scale), P(self.latent), self.s))

    def codec_decode(self):
        P = lambda t: C.c_void_p(t.data_ptr())
        N.check(self.lib.vv_codec_decode_frame(self.h, P(self.latent), P(self.active), P(self.audio), self.s))

    def semantic_encode(self):
        P = lambda t: C.c_void_p(t.data_ptr())
        N.check(self.lib.vv_semantic_encode_frame(self.h, P(self.audio), P(self.active), P(self.feat), self.s))

    def connect(self):
        P = lambda t: C.c_void_p(t.data_ptr())
        N.check(self.lib.vv_connect(self.h, P(self.latent), P(self.feat), P(self.active), P(self.embeds), self.s))

    def codec_state_zero(self, rows):
        a = N.i32(rows)
        if len(a):
            N.check(self.lib.vv_codec_state_zero(self.h, N.iptr(a), len(a), self.s))

    def codec_state_reset(self):
        N.check(self.lib.vv_codec_state_reset(self.h, self.s))

    def codec_taps(self, which: int, rows):
        """One decoder (which = 0: `latent` -> `audio`) or semantic-encoder (which = 1: `audio` -> `feat`) pass with every stage boundary
        copied out (`vv_debug_codec_taps`, tests).  `rows` become the active set and commit their history, as in `codec_decode` /
        `semantic_encode`.  Returns [(meta, tap)]: meta = (kind, stage, index, T, C), tap = [B, T, C] fp32 CPU tensor."""
        src, dst = (self.latent, self.audio) if which == 0 else (self.audio, self.feat)
        n = N.check(self.lib.vv_debug_codec_taps(self.h, int(which), None, None, None, None, 0, None, None), "vv_debug_codec_taps")
        meta = np.zeros((n, 5), dtype=np.int32)
        N.check(self.lib.vv_debug_codec_taps(self.h, int(which), None, None, None, None, 0, N.iptr(meta), None), "vv_debug_codec_taps")
        sizes = [self.B * int(t) * int(c) for t, c in meta[:, 3:]]
        self.active_h.zero_()
        for r in rows:
            self.active_h[r] = 1
        with torch.cuda.stream(self.stream):
            self.active.copy_(self.active_h, non_blocking=True)
            taps = torch.empty(sum(sizes), dtype=torch.float32, device=self.device)
            N.check(self.lib.vv_debug_codec_taps(self.h, int(which), C.c_void_p(src.data_ptr()), C.c_void_p(self.active.data_ptr()),
                                                 C.c_void_p(dst.data_ptr()), C.c_void_p(taps.data_ptr()), taps.numel(), None, self.s),
                    "vv_debug_codec_taps")
        taps = taps.cpu()
        out, off = [], 0
        for m, sz in zip(meta.tolist(), sizes):
            out.append((tuple(m), taps[off:off + sz].view(self.B, m[3], m[4])))
            off += sz
        return out

    def sampler_taps(self, cfg_scale: float):
        """`diffusion_sample` (`hidden` -> `latent`, with `noise`) with every solver block's result copied out (`vv_debug_sampler_taps`,
        tests).  Returns [(meta, tap)]: meta = (kind, step, layer, rows, cols, kernel, split), tap = [rows, cols] fp32 CPU tensor."""
        P = lambda t: C.c_void_p(t.data_ptr())
        call = lambda taps, n, meta, s: self.lib.vv_debug_sampler_taps(self.h, P(self.hidden), P(self.noise), float(cfg_scale), P(self.latent),
                                                                        taps, n, meta, s)
        n = N.check(call(None, 0, None, None), "vv_debug_sampler_taps")
        meta = np.zeros((n, 7), dtype=np.int32)
        N.check(call(None, 0, N.iptr(meta), None), "vv_debug_sampler_taps")
        sizes = [int(r) * int(c) for r, c in meta[:, 3:5]]
        with torch.cuda.stream(self.stream):
            taps = torch.empty(sum(sizes), dtype=torch.float32, device=self.device)
            N.check(call(P(taps), taps.numel(), N.iptr(meta), self.s), "vv_debug_sampler_taps")
        taps = taps.cpu()
        out, off = [], 0
        for m, sz in zip(meta.tolist(), sizes):
            out.append((tuple(m), taps[off:off + sz].view(m[3], m[4])))
            off += sz
        return out

    def launch_count(self) -> int:
        return int(self.lib.vv_launch_count(self.h))

    def sync(self):
        self.stream.synchronize()
