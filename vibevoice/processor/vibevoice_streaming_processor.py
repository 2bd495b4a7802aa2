from vibevoice_b200.processor import AudioNormalizer, VibeVoiceStreamingProcessor  # noqa: F401

__all__ = ["VibeVoiceStreamingProcessor"]
