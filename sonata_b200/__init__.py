"""sonata_b200 — H100-native drop-in for sonata's Piper/VITS phoneme -> waveform hot path.

Public surface mirrors the reference crates on that path:
  sonata_core   -> core.py   (SonataError, Phonemes, Audio, AudioSamples, AudioInfo)
  sonata_piper  -> piper.py  (from_config_path, VitsModel, VitsStreamingModel, PiperSynthesisConfig)
  sonata_synth  -> synth.py  (SonataSpeechSynthesizer: lazy / parallel / realtime schedulers)
All arithmetic runs in sonata_b200/lib/libsonata_b200.so (hand-written sm_90a CUDA, C ABI in
include/sonata_b200.h).  There is no CPU path.
"""
from .core import (Audio, AudioInfo, AudioSamples, FailedToLoadResource, OperationError, PhonemeAlignment, Phonemes,
                   PhonemizationError, SonataError)
from .synth import AudioOutputConfig, RealtimeBatch, SonataSpeechSynthesizer
from .piper import (AdaptiveMelChunker, PiperSynthesisConfig, SpeechStreamer, StreamBatch, VitsModel,
                    VitsStreamingModel, from_config_path)

__all__ = ["Audio", "AudioInfo", "AudioSamples", "FailedToLoadResource", "OperationError", "PhonemeAlignment", "Phonemes",
           "PhonemizationError", "SonataError", "AdaptiveMelChunker", "PiperSynthesisConfig", "SpeechStreamer",
           "StreamBatch", "VitsModel", "VitsStreamingModel", "from_config_path", "AudioOutputConfig",
           "SonataSpeechSynthesizer", "RealtimeBatch"]
