"""Host-side mirror of `sonata-core` + the `audio-ops` output types the hot path returns.

Reference: crates/sonata/core/src/lib.rs (SonataError :19-24, Phonemes :53-79, trait SonataModel
:82-131) and crates/audio/ops/src/samples.rs (AudioInfo :9-14, AudioSamples :16-18, to_i16_vec
:51-75, as_wave_bytes :76-78, crossfade :144-157, Audio :208-271).  Same names, argument meaning
and error behaviour, so the parity tests read like the reference's own.
"""
from __future__ import annotations

import math
import struct
import wave
from dataclasses import dataclass
from typing import Optional

import numpy as np


class SonataError(Exception):
    """enum SonataError (core/src/lib.rs:19-24); FFI codes from capi/libsonata.h:10-14."""
    code = 19

    @staticmethod
    def from_code(code: int, message: str) -> "SonataError":
        cls = {17: FailedToLoadResource, 18: PhonemizationError, 19: OperationError}.get(code, OperationError)
        e = cls(message)
        e.code = code
        return e


class FailedToLoadResource(SonataError):
    code = 17

    def __str__(self):  # Display impl, core/src/lib.rs:35-37
        return f"Failed to load resource from. Error `{self.args[0]}`"


class PhonemizationError(SonataError):
    code = 18


class OperationError(SonataError):
    code = 19


class Phonemes:
    """struct Phonemes(Vec<String>) (core/src/lib.rs:53-79)."""

    def __init__(self, sentences):
        self._s = list(sentences)

    def sentences(self):
        return self._s

    def to_vec(self):
        return list(self._s)

    def num_sentences(self):
        return len(self._s)

    def __str__(self):
        return " ".join(self._s)


@dataclass
class PhonemeAlignment:
    """When one phoneme of an utterance is spoken: `num_samples` samples of its audio from `start_sample` on."""
    phoneme: str
    start_sample: int
    num_samples: int


@dataclass
class AudioInfo:
    sample_rate: int
    num_channels: int = 1
    sample_width: int = 2


_F32_EPS = float(np.finfo(np.float32).eps)

# G.711 encodings a result can be delivered in: the C ABI's law codes (SB200_G711_MULAW / _ALAW), the byte of silence
# (sample 0) and the WAV format tag (WAVE_FORMAT_MULAW = 7, WAVE_FORMAT_ALAW = 6).
ENCODINGS = ("mulaw", "alaw")
G711_LAW = {"mulaw": 0, "alaw": 1}
G711_SILENCE = {"mulaw": 0xFF, "alaw": 0xD5}
G711_WAVE_TAG = {"mulaw": 7, "alaw": 6}


def check_encoding(encoding, who: str = "") -> Optional[str]:
    """`encoding` when it is None, "mulaw" or "alaw"; otherwise OperationError prefixed by `who` (e.g. "utterance 3: ")."""
    if encoding is None or (isinstance(encoding, str) and encoding in ENCODINGS):
        return encoding
    raise OperationError(f"{who}encoding {encoding!r} is neither 'mulaw' nor 'alaw' (or None for linear PCM)")


def g711_encode(x: np.ndarray, encoding: str) -> np.ndarray:
    """G.711 bytes (uint8) of 16-bit samples, as CPython's audioop.lin2ulaw / lin2alaw compute them (the Sun g711.c
    lineage); the library's encoders compute the same bytes on the device."""
    check_encoding(encoding)
    if encoding is None:
        raise OperationError("encoding None is neither 'mulaw' nor 'alaw'")
    v = np.asarray(x, dtype=np.int16).astype(np.int32).reshape(-1)
    if encoding == "mulaw":
        v = v >> 2                                            # 14 bits, arithmetic shift
        mask = np.where(v < 0, 0x7F, 0xFF)
        v = np.minimum(np.abs(v), 8159) + 33                  # 33 .. 8192
        seg = (v[:, None] >= (0x40 << np.arange(8))).sum(axis=1)
        code = np.where(seg >= 8, 0x7F, (np.minimum(seg, 7) << 4) | ((v >> (np.minimum(seg, 7) + 1)) & 0xF))
    else:
        v = v >> 3                                            # 13 bits
        mask = np.where(v < 0, 0x55, 0xD5)
        v = np.where(v < 0, -v - 1, v)                        # 0 .. 4095
        seg = (v[:, None] >= (0x20 << np.arange(8))).sum(axis=1)
        code = (seg << 4) | ((v >> np.maximum(seg, 1)) & 0xF)
    return (code ^ mask).astype(np.uint8)


def g711_wave_bytes(data: bytes, encoding: str, sample_rate: int) -> bytes:
    """A mono 8-bit G.711 WAV file holding `data`: an 18-byte `fmt ` chunk (WAVE_FORMAT_MULAW or WAVE_FORMAT_ALAW,
    block align 1, cbSize 0), a `fact` chunk with the sample count, and the `data` chunk (padded to an even length).
    Python's `wave` module writes PCM only."""
    check_encoding(encoding)
    n = len(data)
    fmt = struct.pack("<HHIIHHH", G711_WAVE_TAG[encoding], 1, int(sample_rate), int(sample_rate), 1, 8, 0)
    body = (b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"fact" + struct.pack("<II", 4, n)
            + b"data" + struct.pack("<I", n) + bytes(data) + (b"\0" if n % 2 else b""))
    return b"RIFF" + struct.pack("<I", len(body)) + body


# FLAC is a whole-file format: its STREAMINFO holds the stream's length and frame sizes, so it is written whole (files,
# batches, jobs) and never handed out piece by piece.
FLAC = "flac"


def refuse_flac(encoding, where: str) -> None:
    """OperationError when `encoding` is "flac" in `where`, a mode that hands out audio piece by piece."""
    if isinstance(encoding, str) and encoding == FLAC:
        raise OperationError(f"{where} cannot deliver 'flac': a FLAC stream is one whole file (STREAMINFO holds its "
                             "length and frame sizes); use synthesize_to_file, infer_batch_flac / speak_batch_flac or "
                             "SynthesisJob.fetch_flac")


def flac_encode(samples_i16: np.ndarray, sample_rate: int, device: int = 0) -> bytes:
    """A complete FLAC stream (RFC 9639 streamable subset: mono, 16 bits, blocks of 4096, MD5 left zero) of the 1-D
    int16 array `samples_i16` at `sample_rate` (one of piper.OUTPUT_RATES), encoded on CUDA device `device` by the
    library's kernels; nothing is encoded on the host.  Zero samples give the 42-byte header-only stream."""
    import ctypes as C
    from . import _native as N
    from .piper import OUTPUT_RATES, _check
    if not isinstance(samples_i16, np.ndarray) or samples_i16.dtype != np.int16 or samples_i16.ndim != 1:
        raise OperationError("flac_encode takes a 1-D numpy array of int16 samples")
    if isinstance(sample_rate, bool) or not isinstance(sample_rate, (int, np.integer)) or int(sample_rate) not in OUTPUT_RATES:
        raise OperationError(f"FLAC: sample rate {sample_rate!r} is not one of the output rates {OUTPUT_RATES}")
    if isinstance(device, bool) or not isinstance(device, (int, np.integer)) or int(device) < 0:
        raise OperationError(f"device {device!r} is not a CUDA device index")
    x = np.ascontiguousarray(samples_i16)
    out, n, err = C.POINTER(C.c_uint8)(), C.c_size_t(), N.sb200_error()
    lib = N.lib()
    _check(lib.sb200_flac_encode(int(device), x.ctypes.data_as(C.POINTER(C.c_int16)), x.size, int(sample_rate),
                                 C.byref(out), C.byref(n), C.byref(err)), err)
    try:
        return C.string_at(out, n.value)
    finally:
        lib.sb200_bytes_free(out)


class AudioSamples:
    """struct AudioSamples(Vec<f32>) (audio/ops/src/samples.rs:16-18)."""

    def __init__(self, samples=()):
        self._v = np.asarray(samples, dtype=np.float32).reshape(-1).copy()

    @classmethod
    def _wrap(cls, array: np.ndarray) -> "AudioSamples":
        """Adopt `array` without copying (used for the library's pinned result buffers)."""
        self = cls.__new__(cls)
        self._v = array
        return self

    def as_slice(self) -> np.ndarray:
        return self._v

    def into_vec(self) -> np.ndarray:
        return self._v

    def __len__(self):
        return int(self._v.shape[0])

    def is_empty(self) -> bool:
        return len(self) == 0

    def to_i16_vec(self) -> np.ndarray:
        """samples.rs:51-75: per-buffer peak normalisation to +-32767, clamp, truncating cast."""
        if self.is_empty():
            return np.zeros(0, dtype=np.int16)
        v = self._v
        abs_max = np.float32(max(abs(float(v.max())), abs(float(v.min())), _F32_EPS))
        scale = np.float32(32767.0) / abs_max
        y = np.clip(v * scale, np.float32(-32768.0), np.float32(32767.0))
        return np.trunc(y).astype(np.int16)

    def to_i16_fixed(self) -> np.ndarray:
        """trunc(clamp(x * 32767, -32768, 32767)): 16-bit PCM at a fixed scale, which keeps a loudness-normalised
        buffer's level (the library's i16 conversion of an utterance with a loudness target)."""
        y = np.clip(self._v * np.float32(32767.0), np.float32(-32768.0), np.float32(32767.0))
        return np.trunc(y).astype(np.int16)

    def as_wave_bytes(self, fixed_scale: bool = False) -> bytes:
        """16-bit little-endian PCM, peak-normalised (to_i16_vec), or at the fixed scale (to_i16_fixed)."""
        return (self.to_i16_fixed() if fixed_scale else self.to_i16_vec()).astype("<i2").tobytes()

    def as_g711_bytes(self, law: str, fixed_scale: bool = False) -> bytes:
        """G.711 ("mulaw" or "alaw") of the 16-bit samples as_wave_bytes holds, one byte per sample: what the library's
        G.711 results are, computed here on the host."""
        check_encoding(law)
        if law is None:
            raise OperationError("law None is neither 'mulaw' nor 'alaw'")
        return g711_encode(self.to_i16_fixed() if fixed_scale else self.to_i16_vec(), law).tobytes()

    def merge(self, other: "AudioSamples") -> None:
        self._v = np.concatenate([self._v, other._v])

    def _own(self) -> None:
        if not self._v.flags.writeable or self._v.base is not None:
            self._v = self._v.copy()

    def crossfade(self, fade_samples: int) -> None:
        """samples.rs:144-157: quarter-sine fade on both ends, f(i) = sin(i/(n-1) * pi/2)."""
        length = len(self)
        n = min(fade_samples, length // 2)
        if n <= 0:
            return
        self._own()
        att = np.float32(n - 1)
        i = np.arange(n, dtype=np.float32)
        with np.errstate(divide="ignore", invalid="ignore"):
            f = np.sin((i / att) * np.float32(math.pi) / np.float32(2.0)).astype(np.float32)
        self._v[:n] *= f
        self._v[length - 1 - np.arange(n)] *= f


class Audio:
    """struct Audio {samples, info, inference_ms} (audio/ops/src/samples.rs:208-271)."""

    def __init__(self, samples, sample_rate: int, inference_ms: Optional[float] = None):
        self.samples = samples if isinstance(samples, AudioSamples) else AudioSamples(samples)
        self.info = AudioInfo(sample_rate=sample_rate, num_channels=1, sample_width=2)
        self.inference_ms = inference_ms

    def into_vec(self):
        return self.samples.into_vec()

    def as_wave_bytes(self) -> bytes:
        return self.samples.as_wave_bytes()

    def __len__(self):
        return len(self.samples)

    def is_empty(self):
        return self.samples.is_empty()

    def duration_ms(self) -> float:
        return (len(self) / self.info.sample_rate) * 1000.0

    def real_time_factor(self) -> Optional[float]:
        """inference_ms / duration_ms — lower is better (samples.rs:253-260)."""
        if self.inference_ms is None:
            return None
        d = self.duration_ms()
        return 0.0 if d == 0.0 else self.inference_ms / d

    def save_to_file(self, filename, fixed_scale: bool = False) -> None:
        """A 16-bit WAV file, peak-normalised, or at the fixed scale (see AudioSamples.as_wave_bytes)."""
        with wave.open(str(filename), "wb") as w:
            w.setnchannels(self.info.num_channels)
            w.setsampwidth(self.info.sample_width)
            w.setframerate(self.info.sample_rate)
            w.writeframes(self.samples.as_wave_bytes(fixed_scale))
