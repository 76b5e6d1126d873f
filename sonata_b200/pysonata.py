"""`pysonata`-shaped binding (SURVEY §8f row N4): the classes and method names of the reference's pyo3 module
(crates/frontends/python/src/lib.rs:43-457) over the H100 engine, so a script written against `pysonata` runs
with `import sonata_b200.pysonata as pysonata`.

    Sonata.with_piper(PiperModel(cfg)).synthesize_parallel(text, AudioOutputConfig(volume=80))  -> WaveSamples ...

Same edges as the rest of the package: `text` is phonemes, one sentence per line (the espeak-ng front-end is
outside this repository, so `phonemize_text` raises `SonataException`); rate / pitch other than neutral raise.
"""
from __future__ import annotations

import os
from typing import Dict, Iterator, Optional

from . import piper as _piper
from .core import Audio, AudioSamples, SonataError
from .synth import AudioOutputConfig as _AudioOutputConfig, SonataSpeechSynthesizer

SonataException = SonataError        # python/src/lib.rs:21-41: every SonataError surfaces as SonataException


class AudioInfo:
    """python/src/lib.rs:43-67 (pyo3 name "AudioInfo")"""

    def __init__(self, info):
        self._i = info

    sample_rate = property(lambda s: s._i.sample_rate)
    num_channels = property(lambda s: s._i.num_channels)
    sample_width = property(lambda s: s._i.sample_width)


class AudioOutputConfig(_AudioOutputConfig):
    """python/src/lib.rs:69-96: AudioOutputConfig(rate=None, volume=None, pitch=None, appended_silence_ms=None)"""


class WaveSamples:
    """python/src/lib.rs:98-134: one synthesized sentence"""

    def __init__(self, audio: Audio):
        self._a = audio

    def get_wave_bytes(self) -> bytes:
        return self._a.as_wave_bytes()

    def save_to_file(self, filename: str) -> None:
        self._a.save_to_file(filename)

    sample_rate = property(lambda s: s._a.info.sample_rate)
    num_channels = property(lambda s: s._a.info.num_channels)
    sample_width = property(lambda s: s._a.info.sample_width)
    inference_ms = property(lambda s: s._a.inference_ms)
    duration_ms = property(lambda s: s._a.duration_ms())
    real_time_factor = property(lambda s: s._a.real_time_factor())


class _Stream:
    def __init__(self, it: Iterator):
        self._it = iter(it)

    def __iter__(self):
        return self


class LazySpeechStream(_Stream):
    """python/src/lib.rs:136-165"""

    def __next__(self) -> WaveSamples:
        return WaveSamples(next(self._it))


class ParallelSpeechStream(LazySpeechStream):
    """python/src/lib.rs:167-196"""


class RealtimeSpeechStream(_Stream):
    """python/src/lib.rs:198-217: yields raw 16-bit PCM bytes per chunk"""

    def __next__(self) -> bytes:
        chunk: AudioSamples = next(self._it)
        return chunk.as_wave_bytes()


class PiperScales:
    """python/src/lib.rs:219-239"""

    def __init__(self, length_scale: float, noise_scale: float, noise_w: float):
        self.length_scale, self.noise_scale, self.noise_w = float(length_scale), float(noise_scale), float(noise_w)

    def __repr__(self):
        return f"PiperScales(length_scale={self.length_scale}, noise_scale={self.noise_scale}, noise_w={self.noise_w})"


class PiperModel:
    """python/src/lib.rs:241-326: PiperModel(config_path); `speaker` property, get_scales / set_scales"""

    def __init__(self, config_path: str, device: Optional[int] = None):
        dev = int(os.environ.get("SONATA_B200_DEVICE", "0")) if device is None else device
        self._m = _piper.from_config_path(config_path, device=dev)

    @property
    def speaker(self) -> Optional[str]:
        cfg = self._m.get_fallback_synthesis_config()
        if cfg.speaker is None:
            return None
        return (self._m.get_speakers() or {}).get(int(cfg.speaker))

    @speaker.setter
    def speaker(self, name: str) -> None:
        sid = self._m.speaker_name_to_id(name)
        if sid is None:
            raise SonataException(f"A speaker with the given name `{name}` was not found")
        cfg = self._m.get_fallback_synthesis_config()
        self._m.set_fallback_synthesis_config(_piper.PiperSynthesisConfig(sid, cfg.noise_scale, cfg.length_scale, cfg.noise_w))

    def get_scales(self) -> PiperScales:
        c = self._m.get_fallback_synthesis_config()
        return PiperScales(c.length_scale, c.noise_scale, c.noise_w)

    def set_scales(self, length_scale: float, noise_scale: float, noise_w: float) -> None:
        c = self._m.get_fallback_synthesis_config()
        self._m.set_fallback_synthesis_config(_piper.PiperSynthesisConfig(c.speaker, noise_scale, length_scale, noise_w))


class Sonata:
    """python/src/lib.rs:328-406"""

    def __init__(self, synth: SonataSpeechSynthesizer):
        self._s = synth

    @staticmethod
    def with_piper(vits_model: PiperModel) -> "Sonata":
        return Sonata(SonataSpeechSynthesizer(vits_model._m))

    def synthesize(self, text: str, audio_output_config: Optional[AudioOutputConfig] = None) -> LazySpeechStream:
        return self.synthesize_lazy(text, audio_output_config)

    def synthesize_lazy(self, text: str, audio_output_config: Optional[AudioOutputConfig] = None) -> LazySpeechStream:
        return LazySpeechStream(self._s.synthesize_lazy(text, audio_output_config))

    def synthesize_parallel(self, text: str, audio_output_config: Optional[AudioOutputConfig] = None) -> ParallelSpeechStream:
        return ParallelSpeechStream(self._s.synthesize_parallel(text, audio_output_config))

    def synthesize_streamed(self, text: str, audio_output_config: Optional[AudioOutputConfig] = None,
                            chunk_size: Optional[int] = None, chunk_padding: Optional[int] = None) -> RealtimeSpeechStream:
        return RealtimeSpeechStream(self._s.synthesize_streamed(text, audio_output_config, chunk_size or 45,
                                                                chunk_padding or 3))          # defaults :379-380

    def synthesize_to_file(self, filename: str, text: str, audio_output_config: Optional[AudioOutputConfig] = None) -> None:
        self._s.synthesize_to_file(filename, text, audio_output_config)

    @property
    def language(self) -> Optional[str]:
        return self._s.model.get_language()

    @property
    def speakers(self) -> Optional[Dict[int, str]]:
        return self._s.model.get_speakers()

    def get_audio_output_info(self) -> AudioInfo:
        return AudioInfo(self._s.audio_output_info())


def phonemize_text(text: str, language: str, phoneme_separator: Optional[str] = None,
                   remove_lang_switch_flags: Optional[bool] = None, remove_stress: Optional[bool] = None,
                   use_tashkeel: Optional[bool] = None):
    """python/src/lib.rs:408-442 calls espeak-ng (and libtashkeel for Arabic): text front-ends before the hot path,
    outside this repository (SURVEY §2 rows 8-9)."""
    raise SonataException("phonemize_text needs the espeak-ng front-end of the reference (crates/text/espeak-phonemizer); "
                          "sonata_b200 takes phonemes")
