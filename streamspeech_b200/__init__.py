"""H100-native streaming speech-to-speech inference path behind the StreamSpeech agent API.

`from streamspeech_b200 import Engine` needs the in-tree CUDA library (libstreamspeech_b200.so,
built by `__graft_entry__.build()` / `make -C streamspeech_b200/csrc`) and a CUDA device at
construction time; nothing here falls back to the CPU.
"""
from .config import ModelConfig, VocoderConfig  # noqa: F401

__all__ = ["ModelConfig", "VocoderConfig"]
