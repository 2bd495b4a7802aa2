"""`vibevoice/modular/modeling_vibevoice_inference.py` import path -> H100 implementation."""
from vibevoice_b200.modeling import ForcedTokenScript, VibeVoiceForConditionalGenerationInference, VibeVoiceGenerationOutput  # noqa: F401

__all__ = ["VibeVoiceForConditionalGenerationInference"]
