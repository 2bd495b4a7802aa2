"""Drop-in import paths of vibevoice-community/VibeVoice for the generation path, served by `vibevoice_b200`.

`demo/inference_from_file.py:26-28` imports
    vibevoice.modular.modeling_vibevoice_inference.VibeVoiceForConditionalGenerationInference
    vibevoice.processor.vibevoice_processor.VibeVoiceProcessor
and `demo/gradio_demo.py` additionally `vibevoice.modular.streamer.AudioStreamer`; those names resolve here to the H100
implementations; `vibevoice.modular.modeling_vibevoice_streaming_inference` and
`vibevoice.processor.vibevoice_streaming_processor.VibeVoiceStreamingProcessor` serve the streaming-0.5B variant the same way
(`demo/streaming_inference_from_file.py`).  Training and conversion modules of the reference are out of scope (SURVEY section 2)."""
