from vibevoice_b200.processor import VibeVoiceProcessor, VibeVoiceStreamingProcessor  # noqa: F401
