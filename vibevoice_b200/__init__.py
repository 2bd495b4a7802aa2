"""vibevoice_b200 -- H100-native implementation of VibeVoice's autoregressive generation hot path.

Host side (this package) mirrors the reference's Python surface
(`vibevoice/modular/modeling_vibevoice_inference.py:68`, `vibevoice/processor/vibevoice_processor.py`)
and drives hand-written sm_90a kernels through the C-ABI library `csrc/libvibevoice_b200.so`
(declared in `include/vibevoice_b200.h`).  There is no CPU fallback: importing the package is
cheap, but any compute call raises if the library is missing.
"""
from .configuration import (  # noqa: F401
    VibeVoiceConfig,
    VibeVoiceAcousticTokenizerConfig,
    VibeVoiceSemanticTokenizerConfig,
    VibeVoiceDiffusionHeadConfig,
    Qwen2DecoderConfig,
    preset_config,
)

__version__ = "0.1.0"
