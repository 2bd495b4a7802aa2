"""ctypes binding of `csrc/libvibevoice_b200.so` (C ABI declared in `include/vibevoice_b200.h`).

No CPU fallback: if the shared library is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libvibevoice_b200.so")

VV_DT_BF16, VV_DT_F32, VV_DT_F16 = 0, 1, 2
PRO_NONE, PRO_RMSNORM, PRO_ADALN, PRO_SILU = 0, 1, 2, 3
EPI_NONE, EPI_RESID, EPI_GATED_RESID, EPI_GAMMA_RESID, EPI_SWIGLU, EPI_GELU, EPI_SILU = 0, 2, 3, 4, 5, 6, 7


class VVError(RuntimeError):
    pass


class ModelDesc(C.Structure):
    _fields_ = [
        ("hidden_size", C.c_int32), ("intermediate_size", C.c_int32), ("num_layers", C.c_int32),
        ("num_q_heads", C.c_int32), ("num_kv_heads", C.c_int32), ("head_dim", C.c_int32), ("vocab_size", C.c_int32),
        ("max_position_embeddings", C.c_int32), ("tie_word_embeddings", C.c_int32),
        ("rms_norm_eps", C.c_float), ("rope_theta", C.c_float),
        ("head_layers", C.c_int32), ("head_ffn_dim", C.c_int32), ("latent_size", C.c_int32), ("head_rms_eps", C.c_float),
        ("n_stages", C.c_int32), ("dec_ratios", C.c_int32 * 8), ("dec_depths", C.c_int32 * 8), ("dec_n_filters", C.c_int32),
        ("enc_ratios", C.c_int32 * 8), ("enc_depths", C.c_int32 * 8), ("enc_n_filters", C.c_int32),
        ("acoustic_vae_dim", C.c_int32), ("semantic_vae_dim", C.c_int32), ("codec_eps", C.c_float),
        ("n_valid_ids", C.c_int32), ("valid_ids", C.c_int32 * 8),
        ("max_batch", C.c_int32), ("max_diffusion_steps", C.c_int32),
    ]


# every symbol include/vibevoice_b200.h declares: (restype, argtypes)
_P, _I, _L, _F = C.c_void_p, C.c_int, C.c_int64, C.c_float
SYMBOLS = {
    "vv_abi_version": (_I, []),
    "vv_last_error": (C.c_char_p, []),
    "vv_create": (_I, [C.POINTER(ModelDesc), _I, C.POINTER(_P)]),
    "vv_destroy": (None, [_P]),
    "vv_load_tensor": (_I, [_P, C.c_char_p, _P, _I, C.POINTER(_L), _I]),
    "vv_set_speech_factors": (_I, [_P, _F, _F]),
    "vv_finalize_weights": (_I, [_P]),
    "vv_weight_bytes": (_L, [_P, _I]),
    "vv_kv_init": (_I, [_P, _L]),
    "vv_kv_reserve": (_I, [_P, _I, _L, _P]),
    "vv_kv_set_len": (_I, [_P, _I, _L, _P]),
    "vv_kv_write": (_I, [_P, _I, _I, _L, _L, _P, _P, _P]),
    "vv_kv_delete_slot": (_I, [_P, _I, _L, _P]),
    "vv_kv_pages_free": (_L, [_P]),
    "vv_kv_pages_total": (_L, [_P]),
    "vv_set_rope_inv_freq": (_I, [_P, _P, _I]),
    "vv_set_row_mode": (_I, [_P, _P, _P]),
    "vv_lm_decode": (_I, [_P, _P, _P, _P, _P, _P]),
    "vv_lm_head": (_I, [_P, _P, _P, _P, _P]),
    "vv_lm_logits_full": (_I, [_P, _P, _P, _P]),
    "vv_lm_decode_range": (_I, [_P, _P, _I, _I, _I, _P, _P]),
    "vv_kv_commit": (_I, [_P, _P, _P]),
    "vv_kv_len": (_L, [_P, _I]),
    "vv_embed_tokens": (_I, [_P, _P, _I, _P, _P]),
    "vv_set_diffusion_steps": (_I, [_P, _I, _P, _P, _P]),
    "vv_set_diffusion_steps_sde": (_I, [_P, _I, _P, _P, _P]),
    "vv_set_step_noise": (_I, [_P, _P]),
    "vv_diffusion_sample": (_I, [_P, _P, _P, _P, _F, _P, _P]),
    "vv_codec_decode_frame": (_I, [_P, _P, _P, _P, _P]),
    "vv_semantic_encode_frame": (_I, [_P, _P, _P, _P, _P]),
    "vv_connect": (_I, [_P, _P, _P, _P, _P, _P]),
    "vv_codec_state_zero": (_I, [_P, _P, _I, _P]),
    "vv_codec_state_reset": (_I, [_P, _P]),
    "vv_frame_tail": (_I, [_P, _P, _P, _P, _F, _P, _P, _P, _P]),
    "vv_voice_encode_workspace": (_L, [_P, _I, _L]),
    "vv_voice_encode": (_I, [_P, _P, _I, _L, _P, _P, _P, _P, _P, _L, _P]),
    "vv_lm_prefill_workspace": (_L, [_P, _L]),
    "vv_lm_prefill": (_I, [_P, _I, _L, _L, _P, _P, _P, _L, _P]),
    "vv_embed_gather": (_I, [_P, _P, _L, _P, _P]),
    "vv_debug_kv_read": (_I, [_P, _I, _I, _L, _L, _P, _P, _P]),
    "vv_launch_count": (_L, [_P]),
    "vv_debug_barrier_bench": (_I, [_P, _I, _I, C.POINTER(C.c_float)]),
    "vv_debug_gemv": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P, _F, _I, _P]),
    "vv_debug_gemv2": (_I, [_P, _P, _P, _P, _L, _I, _L, _P, _L, _P, _L, _I, _I, _I, _I, _P, _F, _I, _P, _L, _P, _P]),
    "vv_debug_codec_taps": (_I, [_P, _I, _P, _P, _P, _P, _L, _P, _P]),
    "vv_debug_sampler_taps": (_I, [_P, _P, _P, _F, _P, _P, _L, _P, _P]),
    "vv_debug_prefill_taps": (_I, [_P, _I, _L, _L, _I, _P, _P, _P, _L, _P, _L, _P, _P]),
    "vv_debug_voice_taps": (_I, [_P, _P, _I, _L, _P, _P, _P, _P, _L, _P, _L, _P, _P]),
    "vv_debug_stream_gemv": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P, _F, _I, _P, _I, _P]),
    "vv_debug_stream_gemv2": (_I, [_P, _P, _P, _P, _L, _P, _L, _I, _I, _I, _I, _P, _F, _P, _P, _L, _I, _P, _L, _I, _L, _P]),
    "vv_stream_diag": (_I, [_P, _P]),
    "vv_stream_trace_read": (_I, [_P, _P, _P, _I, C.c_char_p]),
    "vv_stream_trace_read2": (_I, [_P, _P, _I]),
}

_lib = None


def load_library(path: Optional[str] = None):
    """dlopen the C-ABI library and bind every declared symbol.  Works without a GPU (no CUDA call is made)."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise VVError("libvibevoice_b200.so not built (%s). Run `python -c 'import __graft_entry__ as g; g.build()'`; "
                      "there is no CPU fallback." % p)
    lib = C.CDLL(p)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)          # AttributeError if the export is missing
        fn.restype, fn.argtypes = res, args
    if path is None:
        _lib = lib
    return lib


def check(rc: int, what: str = ""):
    if rc < 0:
        msg = load_library().vv_last_error().decode("utf-8", "replace")
        raise VVError("%s failed (%d): %s" % (what or "vibevoice_b200 call", rc, msg))
    return rc


def iptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def i32(seq: Sequence[int]) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(seq, dtype=np.int32))
