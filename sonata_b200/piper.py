"""Host-side mirror of `sonata-piper` (crates/sonata/models/piper/src/lib.rs) over libsonata_b200.

`from_config_path` / `VitsModel` / `VitsStreamingModel` / `PiperSynthesisConfig` keep the reference's
names and semantics; the arithmetic behind `speak_*` is the CUDA library, never Python.  The integer
host logic that the reference keeps in Rust around `session.run` (the streaming chunk scheduler,
crossfade, one-shot rule) is restated here because it lives on the host side of the FFI boundary
in the reference too.
"""
from __future__ import annotations

import ctypes as C
import math
import numbers
from dataclasses import dataclass
from typing import Iterator, List, Optional, Sequence, Tuple

import numpy as np

from . import _native as N
from .core import (G711_LAW, Audio, AudioInfo, AudioSamples, OperationError, PhonemeAlignment, Phonemes,
                   PhonemizationError, SonataError, check_encoding, refuse_flac)

MIN_CHUNK_SIZE = 44      # piper/src/lib.rs:18
MAX_CHUNK_SIZE = 1024    # piper/src/lib.rs:19
HOP = 256                # piper/src/lib.rs:910
OUTPUT_RATES = (8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000)    # rates results can be resampled to


@dataclass
class PiperSynthesisConfig:
    """piper/src/lib.rs:160-166"""
    speaker: Optional[int] = None
    noise_scale: float = 0.667
    length_scale: float = 1.0
    noise_w: float = 0.8


def _config_array(configs: Optional[Sequence["PiperSynthesisConfig"]], n: int):
    """The C image of per-utterance synthesis configs (None stays None: the voice's fallback config for everyone)."""
    if configs is None:
        return None
    configs = list(configs)
    if len(configs) != n:
        raise OperationError(f"Invalid configuration for Vits Model: {len(configs)} configs for {n} utterances")
    arr = (N.sb200_synth_config * n)()
    for i, c in enumerate(configs):
        if not isinstance(c, PiperSynthesisConfig):
            raise OperationError(f"Invalid configuration for Vits Model (utterance {i})")
        arr[i] = N.sb200_synth_config(c.speaker or 0, 0 if c.speaker is None else 1, c.noise_scale, c.length_scale,
                                      c.noise_w)
    return arr


def _per_utterance(values, n: int, what: str) -> list:
    if isinstance(values, (str, bytes)) or not hasattr(values, "__len__"):
        raise OperationError(f"Invalid {what}: expected one entry (or None) per utterance")
    values = list(values)
    if len(values) != n:
        raise OperationError(f"Invalid {what}: {len(values)} entries for {n} utterances")
    return values


def _scale_value(x, b: int, i: int, unit: str = "id") -> float:
    if isinstance(x, bool) or not isinstance(x, numbers.Real):
        raise OperationError(f"utterance {b}, {unit} {i}: duration scale {x!r} is not a number")
    x = float(x)
    if not (math.isfinite(x) and x >= 0.0):
        raise OperationError(f"utterance {b}, {unit} {i}: duration scale {x} is not a finite value >= 0")
    return x


def _numeric(v, kinds):
    """v as a 1-D numpy array when its dtype kind is one of `kinds` (the vectorised checks), else None."""
    a = v if isinstance(v, np.ndarray) else np.asarray(v) if not isinstance(v, (str, bytes)) else None
    return a.reshape(-1) if a is not None and a.dtype.kind in kinds and a.ndim <= 1 else None


def _duration_arrays(lens: Sequence[int], duration_scales=None, durations=None):
    """The packed C images of per-id duration controls, checked as the library checks them: (scales f32, frames i32),
    each None when not given.  duration_scales[b] / durations[b] hold one value per id of utterance b, or None for an
    utterance without that control (scale 1.0, frames -1: its plain result).  Numeric arrays are checked in one
    vectorised pass; anything else element by element, which also names the first bad element."""
    n = len(lens)
    total = int(sum(lens))
    scales = frames = None
    if duration_scales is not None:
        scales = np.ones(total, np.float32)
        pos = 0
        for b, v in enumerate(_per_utterance(duration_scales, n, "duration scales")):
            if v is not None:
                a = _numeric(v, "fiu")
                if a is None:
                    v = list(v)
                    a = np.array([_scale_value(x, b, i) for i, x in enumerate(v)] if len(v) == lens[b] else v)
                if a.size != lens[b]:
                    raise OperationError(f"utterance {b}: {a.size} duration scales for {lens[b]} ids")
                f = a.astype(np.float32)
                bad = np.nonzero(~(np.isfinite(f) & (f >= 0)))[0]
                if bad.size:
                    _scale_value(float(f[bad[0]]), b, int(bad[0]))
                scales[pos:pos + lens[b]] = f
            pos += lens[b]
    if durations is not None:
        frames = np.full(total, -1, np.int32)
        pos = 0
        for b, v in enumerate(_per_utterance(durations, n, "durations")):
            if v is not None:
                a = _numeric(v, "iu")
                if a is None:
                    v = list(v)
                    if len(v) == lens[b]:
                        for i, x in enumerate(v):
                            if isinstance(x, bool) or not isinstance(x, numbers.Integral):
                                raise OperationError(f"utterance {b}, id {i}: fixed duration {x!r} is not an integer")
                    a = np.array([int(x) for x in v], dtype=object)
                if a.size != lens[b]:
                    raise OperationError(f"utterance {b}: {a.size} durations for {lens[b]} ids")
                bad = np.nonzero((a < -1) | (a > 2**31 - 1))[0]
                if bad.size:
                    raise OperationError(f"utterance {b}, id {int(bad[0])}: fixed duration {int(a[bad[0]])} is neither "
                                         "-1 (predicted) nor a frame count >= 0")
                frames[pos:pos + lens[b]] = a.astype(np.int64)
            pos += lens[b]
    return scales, frames


def _seed_arrays(seeds, n: int):
    """The C image of per-utterance noise seeds: (seeds u64, seeded i32), or (None, None) when `seeds` is None or holds
    no seed.  seeds[b] is an int in [0, 2**64) or None (utterance b keeps its positional noise)."""
    if seeds is None:
        return None, None
    vals = np.zeros(n, np.uint64)
    flags = np.zeros(n, np.int32)
    for b, s in enumerate(_per_utterance(seeds, n, "noise seeds")):
        if s is None:
            continue
        if isinstance(s, bool) or not isinstance(s, numbers.Integral):
            raise OperationError(f"utterance {b}: noise seed {s!r} is not an integer")
        if not 0 <= int(s) < 2**64:
            raise OperationError(f"utterance {b}: noise seed {int(s)} is not in [0, 2**64)")
        vals[b], flags[b] = int(s), 1
    if not flags.any():
        return None, None
    return vals, flags


def _rate_array(rates, n: int):
    """The C image of per-utterance output rates (u32), or None when `rates` is None.  rates[b] is one of OUTPUT_RATES,
    or None / 0 for the voice's own rate; the library also treats the voice's own rate as no resampling."""
    if rates is None:
        return None
    out = np.zeros(n, np.uint32)
    for b, r in enumerate(_per_utterance(rates, n, "output rates")):
        if r is None:
            continue
        if isinstance(r, bool) or not isinstance(r, numbers.Integral) or (int(r) != 0 and int(r) not in OUTPUT_RATES):
            raise OperationError(f"utterance {b}: output rate {r!r} Hz is not supported "
                                 f"({', '.join(map(str, OUTPUT_RATES))}, or 0 / None for the voice's rate)")
        out[b] = int(r)
    return out


def _loudness_array(targets, n: int):
    """The C image of per-utterance loudness targets (f32, NaN for none), or None when `targets` is None or holds no
    target.  targets[b] is a LUFS value, finite and in [-70, 0], or None / NaN (utterance b is measured only)."""
    if targets is None:
        return None
    out = np.full(n, np.nan, np.float32)
    for b, t in enumerate(_per_utterance(targets, n, "loudness targets")):
        if t is None:
            continue
        if isinstance(t, bool) or not isinstance(t, numbers.Real):
            raise OperationError(f"utterance {b}: loudness target {t!r} is not a number")
        if math.isnan(float(t)):
            continue
        if not (math.isfinite(float(t)) and -70.0 <= float(t) <= 0.0):
            raise OperationError(f"utterance {b}: loudness target {float(t)} LUFS is not a finite value in [-70, 0]")
        out[b] = float(t)
    return None if np.isnan(out).all() else out


PITCH_RANGE = (0.5, 2.0)     # pitch ratios a result can be shifted by
TEMPO_RANGE = (0.25, 4.0)    # tempo ratios a result can be played at


def _ratio_array(values, n: int, what: str, lo: float, hi: float):
    if values is None:
        return None
    out = np.full(n, np.nan, np.float32)
    for b, v in enumerate(_per_utterance(values, n, f"{what} ratios")):
        if v is None:
            continue
        if isinstance(v, bool) or not isinstance(v, numbers.Real):
            raise OperationError(f"utterance {b}: {what} ratio {v!r} is not a number")
        if math.isnan(float(v)) or float(v) == 1.0:
            continue
        if not (math.isfinite(float(v)) and lo <= float(v) <= hi):
            raise OperationError(f"utterance {b}: {what} ratio {float(v)} is not a finite value in [{lo}, {hi}]")
        out[b] = float(v)
    return None if np.isnan(out).all() else out


def _prosody_arrays(pitches, tempos, n: int):
    """The C images of per-utterance pitch and tempo ratios: (pitch f32, tempo f32), NaN for none, each None when not
    given or when no utterance asks.  pitches[b] is a ratio in PITCH_RANGE, tempos[b] one in TEMPO_RANGE, or None / NaN /
    1.0 for an utterance that keeps its samples."""
    return _ratio_array(pitches, n, "pitch", *PITCH_RANGE), _ratio_array(tempos, n, "tempo", *TEMPO_RANGE)


def _prosody_kwargs(pitches, tempos) -> dict:
    out = {} if pitches is None else {"pitches": pitches}
    if tempos is not None:
        out["tempos"] = tempos
    return out


def refuse_prosody(pitch, tempo, where: str) -> None:
    """OperationError when `where`, a mode that hands out a sentence chunk by chunk, is asked for a pitch or tempo
    ratio."""
    if any(a is not None for a in _prosody_arrays([pitch], [tempo], 1)):
        raise OperationError(f"{where} cannot shift pitch or tempo: the time stretch walks a whole sentence frame by "
                             "frame, and this mode hands out a sentence's first chunk before its last one is decoded "
                             "(use the lazy, parallel or file modes, speak_batch or a SynthesisJob)")


def _encoding_list(law, n: int) -> list:
    """One G.711 encoding ("mulaw" / "alaw") per utterance from `law`: one encoding for all, or one per utterance.  A bad
    entry raises OperationError naming the utterance."""
    laws = [law] * n if law is None or isinstance(law, str) else _per_utterance(law, n, "encodings")
    for b, e in enumerate(laws):
        if e is None or check_encoding(e, f"utterance {b}: ") is None:
            raise OperationError(f"utterance {b}: encoding {e!r} is neither 'mulaw' nor 'alaw'")
    return laws


def _gain_array(gains, n: int):
    """The C image of per-utterance linear gains (f32), or None when `gains` is None (1 for every utterance)."""
    if gains is None:
        return None
    out = np.ones(n, np.float32)
    for b, g in enumerate(_per_utterance(gains, n, "gains")):
        if g is None:
            continue
        if isinstance(g, bool) or not isinstance(g, numbers.Real) or not math.isfinite(float(g)):
            raise OperationError(f"utterance {b}: gain {g!r} is not a finite number")
        out[b] = float(g)
    return out


def rate_ratio(in_rate: int, out_rate: Optional[int]) -> Tuple[int, int]:
    """(up, down): out_rate / in_rate reduced, (1, 1) for no resampling (None, 0 or the same rate)."""
    if not out_rate or int(out_rate) == int(in_rate):
        return 1, 1
    g = math.gcd(int(in_rate), int(out_rate))
    return int(out_rate) // g, int(in_rate) // g


def _ptr(a, ctype):
    return None if a is None else a.ctypes.data_as(C.POINTER(ctype))


def _alignment(phonemes: str, src_char: Sequence[int], frames: Sequence[int], n_samples: int,
               up: int = 1, down: int = 1, warped: bool = False) -> List[PhonemeAlignment]:
    """Groups per-id frame counts by the character each id came from: bos (`^`), one entry per kept character (its id
    and its pad) and eos (`$`), contiguous from sample 0.  An utterance whose ids all got 0 frames is still one frame
    long; that frame (after every id) goes to the last entry, so the entries always end at n_samples.  Audio resampled
    by up/down puts the boundary after F frames at ceil(F * hop * up / down).  `warped` (a pitch or tempo ratio changed
    the length): the boundary after F of the utterance's T frames is at floor(F * n_samples / T + 0.5), whatever the
    output rate; the time stretch moves a sample by at most D = rate // 160 input samples from that linear map, so a
    boundary is accurate to within D / tempo samples of the warped signal."""
    total = int(sum(int(f) for f in frames))
    hop = n_samples // max(total, 1) if (up, down) == (1, 1) else HOP
    at = lambda frames_before: -((-frames_before * hop * up) // down)
    if warped:
        at = lambda frames_before: (2 * frames_before * n_samples + max(total, 1)) // (2 * max(total, 1))
    out: List[PhonemeAlignment] = []
    start, i, fsum = 0, 0, 0
    while i < len(frames):
        src = int(src_char[i])
        j, f = i, 0
        while j < len(frames) and int(src_char[j]) == src and not (src < 0 and j > i):
            f += int(frames[j])
            j += 1
        ph = phonemes[src] if src >= 0 else ("^" if i == 0 else "$")
        fsum += f
        end = at(fsum)
        out.append(PhonemeAlignment(ph, start, end - start))
        start = end
        i = j
    if out and start != n_samples:
        out[-1].num_samples += n_samples - start
    return out


def _check(rc: int, err: N.sb200_error):
    if rc != 0:
        msg = ""
        if err.message:
            msg = C.string_at(err.message).decode("utf-8", "replace")
            N.lib().sb200_string_free(err.message)
        raise SonataError.from_code(err.code if err.code else rc, msg)


class _PinnedOwner:
    """Keeps one library-owned (pinned) result buffer alive for as long as a numpy view of it exists."""

    def __init__(self, a: N.sb200_audio):
        self.a = N.sb200_audio(a.data, a.len, a.inference_ms, a.sample_rate)

    def __del__(self):
        try:
            N.lib().sb200_audio_free(C.byref(self.a))
        except Exception:
            pass


def _take_chunks(lib, outs, lens, dtype) -> list:
    """Copies of the chunk buffers `outs` (malloc'ed, lens[k] samples of `dtype` each) as numpy arrays; frees them."""
    ptr = C.POINTER(np.ctypeslib.as_ctypes_type(dtype))
    res = []
    for k in range(len(lens)):
        m = int(lens[k])
        res.append(np.ctypeslib.as_array(C.cast(outs[k], ptr), (m,)).copy() if m else np.zeros(0, dtype))
        lib.sb200_i16_free(C.cast(outs[k], C.POINTER(C.c_int16)))
    return res


def _take_bytes(lib, outs, lens) -> List[bytes]:
    """Copies of the byte buffers `outs` (malloc'ed, lens[k] bytes each) as bytes; frees them."""
    res = []
    for k in range(len(lens)):
        res.append(C.string_at(outs[k], int(lens[k])) if int(lens[k]) else b"")
        lib.sb200_bytes_free(C.cast(outs[k], C.POINTER(C.c_uint8)))
    return res


def _take_audio(a: N.sb200_audio) -> Audio:
    """Zero-copy: the returned samples are a read-only view of the library's pinned host buffer (the
    reference copies `outputs[0]` into a Vec at piper/src/lib.rs:392)."""
    if not a.len:
        N.lib().sb200_audio_free(C.byref(a))
        return Audio(AudioSamples(np.zeros(0, np.float32)), int(a.sample_rate), float(a.inference_ms))
    owner = _PinnedOwner(a)
    buf = (C.c_float * a.len).from_address(C.addressof(a.data.contents))
    buf._owner = owner
    arr = np.frombuffer(buf, dtype=np.float32)
    arr.flags.writeable = False
    return Audio(AudioSamples._wrap(arr), int(a.sample_rate), float(a.inference_ms))


class AdaptiveMelChunker:
    """piper/src/lib.rs:860-913 — yields ((mel_start, mel_end|None), (audio_start, audio_end|None))."""

    def __init__(self, num_frames: int, chunk_size: int, chunk_padding: int):
        self.num_frames = num_frames
        self.chunk_size = chunk_size
        self.chunk_padding = chunk_padding
        self.last_end_index: Optional[int] = 0
        self.step = 1

    def consume(self):
        self.last_end_index = None

    def __iter__(self):
        return self

    def __next__(self):
        last_index = self.last_end_index
        if last_index is None:
            raise StopIteration
        chunk_size = min(self.chunk_size * self.step, MAX_CHUNK_SIZE)
        if last_index == 0:
            start_index, start_padding = 0, 0
        else:
            start_index = last_index - self.chunk_padding * 2
            start_padding = self.chunk_padding
        chunk_end = last_index + chunk_size + self.chunk_padding
        remaining = self.num_frames - chunk_end
        if remaining <= MIN_CHUNK_SIZE:
            end_index, end_padding = None, None
        else:
            end_index, end_padding = chunk_end, -self.chunk_padding
        self.step += 1
        self.last_end_index = end_index
        return ((start_index, end_index),
                (start_padding * HOP, None if end_padding is None else end_padding * HOP))


class _VitsCommons:
    def __init__(self, config_path: str, device: int = 0):
        lib = N.lib()
        self._lib = lib
        self._h = C.c_void_p()
        err = N.sb200_error()
        _check(lib.sb200_voice_load(str(config_path).encode("utf-8"), device, C.byref(self._h), C.byref(err)), err)
        self.config_path = str(config_path)
        self.device = device
        self._speakers = None

    def get_speakers(self) -> Optional[dict]:
        """SonataModel::get_speakers (piper/src/lib.rs:463-465): {speaker id: name} of a multi-speaker voice, read from
        the `speaker_id_map` of the voice config (None for single-speaker voices)."""
        if self._speakers is None:
            import json
            with open(self.config_path, encoding="utf-8") as f:
                m = json.load(f).get("speaker_id_map") or {}
            self._speakers = {int(v): k for k, v in m.items()}
        return self._speakers or None

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.sb200_voice_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- trait SonataModel (core/src/lib.rs:82-131) ----
    def audio_output_info(self) -> AudioInfo:
        ai, err = N.sb200_audio_info(), N.sb200_error()
        _check(self._lib.sb200_audio_output_info(self._h, C.byref(ai), C.byref(err)), err)
        return AudioInfo(int(ai.sample_rate), int(ai.num_channels), int(ai.sample_width))

    def phonemize_text(self, text: str) -> Phonemes:
        # espeak-ng front-end is outside the hot path (SURVEY §2 row 8); callers pass phonemes.
        raise PhonemizationError("Failed to phonemize given text using espeak-ng. Error: "
                                 "the espeak-ng front-end is not part of sonata_b200; pass phonemes")

    def phonemes_to_input_ids(self, phonemes: str) -> List[int]:
        ids = C.POINTER(C.c_int64)()
        n = C.c_size_t()
        err = N.sb200_error()
        _check(self._lib.sb200_phonemes_to_input_ids(self._h, phonemes.encode("utf-8"), C.byref(ids), C.byref(n),
                                                     C.byref(err)), err)
        out = [int(ids[i]) for i in range(n.value)]
        self._lib.sb200_ids_free(ids)
        return out

    def phonemes_to_input_ids_map(self, phonemes: str) -> Tuple[List[int], List[int]]:
        """phonemes_to_input_ids plus, per id, the index (in characters of `phonemes`) of the character it came from: a
        pad belongs to the character before it, bos and eos get -1, dropped characters own no id."""
        ids, src = C.POINTER(C.c_int64)(), C.POINTER(C.c_int64)()
        n = C.c_size_t()
        err = N.sb200_error()
        _check(self._lib.sb200_phonemes_to_input_ids_map(self._h, phonemes.encode("utf-8"), C.byref(ids), C.byref(src),
                                                         C.byref(n), C.byref(err)), err)
        out = ([int(ids[i]) for i in range(n.value)], [int(src[i]) for i in range(n.value)])
        self._lib.sb200_ids_free(ids)
        self._lib.sb200_ids_free(src)
        return out

    def speak_one_sentence(self, phonemes: str) -> Audio:
        a, err = N.sb200_audio(), N.sb200_error()
        _check(self._lib.sb200_speak_one_sentence(self._h, phonemes.encode("utf-8"), C.byref(a), C.byref(err)), err)
        return _take_audio(a)

    def speak_batch(self, phoneme_batches: Sequence[str],
                    configs: Optional[Sequence[PiperSynthesisConfig]] = None, seeds: Optional[Sequence] = None,
                    output_rates: Optional[Sequence] = None, loudness: Optional[Sequence] = None,
                    pitches: Optional[Sequence] = None, tempos: Optional[Sequence] = None) -> List[Audio]:
        """`configs`: one PiperSynthesisConfig per utterance (speaker and scales), still synthesised as one pass;
        None uses the fallback config for every utterance.  `seeds`: noise seeds as for infer_batch_with_values.
        `output_rates` / `loudness` / `pitches` / `tempos`: per-utterance output sample rates, loudness targets and
        pitch and tempo ratios as for infer_batch_with_values."""
        n = len(phoneme_batches)
        _config_array(configs, n)             # argument errors before any id mapping
        sv, _ = _seed_arrays(seeds, n)
        rates = _rate_array(output_rates, n)
        loud = _loudness_array(loudness, n)
        pros = any(a is not None for a in _prosody_arrays(pitches, tempos, n))
        if n == 0:
            return []
        if configs is not None or sv is not None or rates is not None or loud is not None or pros:
            extra = {} if sv is None else {"seeds": seeds}
            if pros:
                extra.update(_prosody_kwargs(pitches, tempos))
            if rates is not None:
                extra["output_rates"] = output_rates
            if loud is not None:
                extra["loudness"] = loudness
            return self.infer_batch_with_values([self.phonemes_to_input_ids(p) for p in phoneme_batches], configs,
                                                **extra)
        arr = (C.c_char_p * n)(*[p.encode("utf-8") for p in phoneme_batches])
        outs = (N.sb200_audio * n)()
        err = N.sb200_error()
        _check(self._lib.sb200_speak_batch(self._h, arr, n, outs, C.byref(err)), err)
        return [_take_audio(outs[i]) for i in range(n)]

    def infer_with_values(self, input_phonemes: Sequence[int]) -> Audio:
        """VitsModel::infer_with_values (piper/src/lib.rs:342-399)."""
        ids = np.ascontiguousarray(input_phonemes, dtype=np.int64)
        a, err = N.sb200_audio(), N.sb200_error()
        _check(self._lib.sb200_speak_ids(self._h, ids.ctypes.data_as(C.POINTER(C.c_int64)), ids.size, C.byref(a),
                                         C.byref(err)), err)
        return _take_audio(a)

    def infer_batch_with_values(self, batches: Sequence[Sequence[int]],
                                configs: Optional[Sequence[PiperSynthesisConfig]] = None,
                                seeds: Optional[Sequence] = None,
                                output_rates: Optional[Sequence] = None,
                                loudness: Optional[Sequence] = None, pitches: Optional[Sequence] = None,
                                tempos: Optional[Sequence] = None) -> List[Audio]:
        """Batched infer_with_values.  `configs`: one PiperSynthesisConfig per utterance (speaker and scales), or None
        for the fallback config; each utterance's result equals a single-utterance call with its config as the
        fallback, except for the on-device noise of an unseeded utterance, whose draws depend on the batch position.

        `seeds`: one noise seed per utterance, an int in [0, 2**64) or None.  A seeded utterance's noise depends on its
        seed alone, so its result is the same bits in any batch, on any call and on any handle of the voice; an
        unseeded one keeps the positional noise of a call without seeds.

        `output_rates`: one output sample rate per utterance, one of OUTPUT_RATES, or None / 0 for the voice's own.
        The waveform is resampled on the device with scipy.signal.resample_poly's default filter, and the Audio
        reports the rate it is at.

        `loudness`: one target integrated loudness per utterance in LUFS (finite, in [-70, 0]) or None.  The delivered
        signal (after any resampling) is measured on the device as ITU-R BS.1770-4 defines it and scaled to the target,
        never past a sample peak of 1.0; an utterance under 400 ms or silent keeps its samples, as does one whose target
        is None (see include/sonata_b200.h, sb200_speak_batch_ids_loudness).

        `pitches` / `tempos`: one ratio per utterance, or None.  A pitch p in PITCH_RANGE multiplies every frequency of
        the utterance and keeps its duration; a tempo t in TEMPO_RANGE plays it t times faster at the same pitch (about
        len / t samples), keeping the model's articulation where a small length_scale would ask the duration predictor
        for durations it never saw.  Both are signal processing on the decoder's waveform on the device (WSOLA, then a
        windowed-sinc resampler; sb200_speak_batch_ids_prosody), before any resampling and loudness; None, NaN or 1.0
        leaves the utterance's samples as they are, bit for bit."""
        n = len(batches)
        cfgs = _config_array(configs, n)
        sv, _ = _seed_arrays(seeds, n)
        rates = _rate_array(output_rates, n)
        loud = _loudness_array(loudness, n)
        pros = any(a is not None for a in _prosody_arrays(pitches, tempos, n))
        if sv is not None or rates is not None or loud is not None or pros:
            return [a for a, _ in self.infer_batch_with_durations(batches, configs, seeds=seeds,
                                                                  output_rates=output_rates, loudness=loudness,
                                                                  **(_prosody_kwargs(pitches, tempos) if pros else {}))]
        packed = np.ascontiguousarray(np.concatenate([np.asarray(b, dtype=np.int64) for b in batches]))
        offs = np.zeros(n + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(b) for b in batches])
        outs = (N.sb200_audio * n)()
        err = N.sb200_error()
        _check(self._lib.sb200_speak_batch_ids_configs(self._h, packed.ctypes.data_as(C.POINTER(C.c_int64)),
                                                       offs.ctypes.data_as(C.POINTER(C.c_size_t)), n, cfgs, outs,
                                                       C.byref(err)), err)
        return [_take_audio(outs[i]) for i in range(n)]

    def infer_batch_with_durations(self, batches: Sequence[Sequence[int]],
                                   configs: Optional[Sequence[PiperSynthesisConfig]] = None,
                                   duration_scales: Optional[Sequence] = None,
                                   durations: Optional[Sequence] = None,
                                   seeds: Optional[Sequence] = None,
                                   output_rates: Optional[Sequence] = None,
                                   loudness: Optional[Sequence] = None, pitches: Optional[Sequence] = None,
                                   tempos: Optional[Sequence] = None) -> List[Tuple[Audio, np.ndarray]]:
        """infer_batch_with_values with per-id duration control, returning (audio, frames per id) per utterance.

        duration_scales[b]: one scale (finite, >= 0) per id of utterance b, applied before the duration's ceil, so 1.0
        gives the plain result bit for bit; durations[b]: one frame count per id, -1 for "predicted" or >= 0 to fix it.
        Either list, or any of its entries, may be None.  The frame counts times 256 are each id's samples; an
        utterance whose ids all got 0 frames is still one frame long.  `seeds`: as for infer_batch_with_values; a
        seeded frame's noise depends on its index only, so controls that move frames never reshuffle it.
        `output_rates` / `loudness` / `pitches` / `tempos`: as for infer_batch_with_values (the frame counts stay frame
        counts of the utterance before any warp)."""
        n = len(batches)
        cfgs = _config_array(configs, n)
        lens = [len(b) for b in batches]
        scales, frames = _duration_arrays(lens, duration_scales, durations)
        sv, sf = _seed_arrays(seeds, n)
        rates = _rate_array(output_rates, n)
        loud = _loudness_array(loudness, n)
        pit, tem = _prosody_arrays(pitches, tempos, n)
        if n == 0:
            return []
        if any(x == 0 for x in lens):
            raise OperationError("Failed to run model inference. Error: empty input sequence")
        packed = np.ascontiguousarray(np.concatenate([np.asarray(b, dtype=np.int64) for b in batches]))
        offs = np.zeros(n + 1, dtype=np.uint64)
        offs[1:] = np.cumsum(lens)
        outs = (N.sb200_audio * n)()
        id_frames = np.zeros(int(offs[-1]), np.int32)
        err = N.sb200_error()
        _check(self._lib.sb200_speak_batch_ids_prosody(
            self._h, packed.ctypes.data_as(C.POINTER(C.c_int64)), offs.ctypes.data_as(C.POINTER(C.c_size_t)), n, cfgs,
            _ptr(scales, C.c_float), _ptr(frames, C.c_int32), _ptr(sv, C.c_uint64), _ptr(sf, C.c_int32),
            _ptr(rates, C.c_uint32), _ptr(loud, C.c_float), _ptr(pit, C.c_float), _ptr(tem, C.c_float), outs,
            _ptr(id_frames, C.c_int32), None, None, C.byref(err)), err)
        return [(_take_audio(outs[b]), id_frames[int(offs[b]):int(offs[b + 1])].copy()) for b in range(n)]

    def speak_batch_with_alignment(self, phoneme_batches: Sequence[str],
                                   configs: Optional[Sequence[PiperSynthesisConfig]] = None,
                                   duration_scales: Optional[Sequence] = None,
                                   seeds: Optional[Sequence] = None,
                                   output_rates: Optional[Sequence] = None,
                                   loudness: Optional[Sequence] = None, pitches: Optional[Sequence] = None,
                                   tempos: Optional[Sequence] = None) -> List[Tuple[Audio, List[PhonemeAlignment]]]:
        """speak_batch that also says when each phoneme is spoken: per utterance (audio, alignment), the alignment
        holding one entry for bos (`^`), one per kept phoneme character (its id and its trailing pad) and one for eos
        (`$`), contiguous from sample 0 to len(audio).

        duration_scales[b] (or None): one scale per character of phoneme_batches[b], applied to that character's id and
        pad; characters the voice drops have no entry and their scales are ignored.  `seeds`: as for
        infer_batch_with_values.  `output_rates`: as for infer_batch_with_values; the alignment is then in samples of
        the output rate, the boundary after F frames at ceil(F * 256 * up / down).  `loudness`: as for
        infer_batch_with_values; it scales samples and moves no boundary.  `pitches` / `tempos`: as for
        infer_batch_with_values; an utterance with a ratio has every boundary scaled by delivered / original length
        (floor(F * len(audio) / T + 0.5) after F of its T frames), accurate to within (rate // 160) / tempo samples of
        the warped signal because the time stretch takes each frame from within that many samples of the linear map."""
        n = len(phoneme_batches)
        _config_array(configs, n)
        _seed_arrays(seeds, n)
        _rate_array(output_rates, n)
        _loudness_array(loudness, n)
        pit, tem = _prosody_arrays(pitches, tempos, n)
        warped = [(pit is not None and not np.isnan(pit[b])) or (tem is not None and not np.isnan(tem[b]))
                  for b in range(n)]
        per_char = None if duration_scales is None else _per_utterance(duration_scales, n, "duration scales")
        maps = [self.phonemes_to_input_ids_map(p) for p in phoneme_batches]
        id_scales = None
        if per_char is not None:
            id_scales = []
            for b, (ph, (ids, src)) in enumerate(zip(phoneme_batches, maps)):
                v = per_char[b]
                if v is None:
                    id_scales.append(None)
                    continue
                v = list(v) if not isinstance(v, np.ndarray) else v.reshape(-1).tolist()
                if len(v) != len(ph):
                    raise OperationError(f"utterance {b}: {len(v)} duration scales for {len(ph)} characters")
                kept = {c: _scale_value(v[c], b, c, "character") for c in sorted(set(src)) if c >= 0}
                id_scales.append([1.0 if c < 0 else kept[c] for c in src])
        extra = {} if seeds is None else {"seeds": seeds}
        if output_rates is not None:
            extra["output_rates"] = output_rates
        if loudness is not None:
            extra["loudness"] = loudness
        if any(warped):
            extra.update(_prosody_kwargs(pitches, tempos))
        res = self.infer_batch_with_durations([m[0] for m in maps], configs, id_scales, **extra)
        voice_rate = self.audio_output_info().sample_rate if output_rates is not None else None
        ratio = lambda audio: (1, 1) if voice_rate is None else rate_ratio(voice_rate, audio.info.sample_rate)
        return [(audio, _alignment(ph, src, frames, len(audio), *ratio(audio), warped=w))
                for ph, (_, src), (audio, frames), w in zip(phoneme_batches, maps, res, warped)]

    def infer_batch_g711(self, batches: Sequence[Sequence[int]], law,
                         configs: Optional[Sequence[PiperSynthesisConfig]] = None, seeds: Optional[Sequence] = None,
                         output_rates: Optional[Sequence] = None, loudness: Optional[Sequence] = None,
                         gains: Optional[Sequence] = None, pitches: Optional[Sequence] = None,
                         tempos: Optional[Sequence] = None) -> List[bytes]:
        """infer_batch_with_values delivered as G.711 telephony audio: one `bytes` per utterance, one byte per sample.
        `law`: "mulaw" (PCMU) or "alaw" (PCMA), or one of those per utterance.  The bytes are G.711 of exactly the
        16-bit samples the i16 route gives (SynthesisJob.fetch_i16): to_i16_vec of the utterance after gains[b] (None:
        1), or the fixed scale for an utterance with a loudness target.  They are encoded on the device in the i16
        conversion's launches, so only one byte per sample leaves the card.  `configs`, `seeds`, `output_rates` and
        `loudness` as for infer_batch_with_values, and so are `pitches` and `tempos`; a batch mixing laws runs one
        conversion per law."""
        from .job import SynthesisJob
        n = len(batches)
        _config_array(configs, n)
        _seed_arrays(seeds, n)
        _rate_array(output_rates, n)
        _loudness_array(loudness, n)
        laws = _encoding_list(law, n)
        _gain_array(gains, n)
        _prosody_arrays(pitches, tempos, n)
        if n == 0:
            return []
        if any(len(b) == 0 for b in batches):
            raise OperationError("Failed to run model inference. Error: empty input sequence")
        job = SynthesisJob(self, batches, configs=configs, seeds=seeds, output_rates=output_rates, loudness=loudness,
                           pitches=pitches, tempos=tempos)
        try:
            job.run()
            out: List[Optional[bytes]] = [None] * n
            for e in dict.fromkeys(laws):
                res = job.fetch_g711(e, gains)
                for b in range(n):
                    if laws[b] == e:
                        out[b] = res[b]
            return out
        finally:
            job.close()

    def speak_batch_g711(self, phoneme_batches: Sequence[str], law,
                         configs: Optional[Sequence[PiperSynthesisConfig]] = None, seeds: Optional[Sequence] = None,
                         output_rates: Optional[Sequence] = None, loudness: Optional[Sequence] = None,
                         gains: Optional[Sequence] = None, pitches: Optional[Sequence] = None,
                         tempos: Optional[Sequence] = None) -> List[bytes]:
        """speak_batch delivered as G.711 bytes: infer_batch_g711 over the phonemes' ids."""
        n = len(phoneme_batches)
        _config_array(configs, n)
        _encoding_list(law, n)
        return self.infer_batch_g711([self.phonemes_to_input_ids(p) for p in phoneme_batches], law, configs, seeds,
                                     output_rates, loudness, gains, pitches, tempos)

    def infer_batch_flac(self, batches: Sequence[Sequence[int]],
                         configs: Optional[Sequence[PiperSynthesisConfig]] = None, seeds: Optional[Sequence] = None,
                         output_rates: Optional[Sequence] = None, loudness: Optional[Sequence] = None,
                         gains: Optional[Sequence] = None, pitches: Optional[Sequence] = None,
                         tempos: Optional[Sequence] = None) -> List[bytes]:
        """infer_batch_with_values delivered as lossless FLAC: one complete stream (`bytes`) per utterance.  Its samples
        are exactly the 16-bit samples the i16 route gives (SynthesisJob.fetch_i16): to_i16_vec of the utterance after
        gains[b] (None: 1), or the fixed scale for an utterance with a loudness target, at its delivered rate.  They are
        encoded on the device, and only the compressed bytes leave the card.  `configs`, `seeds`, `output_rates`,
        `loudness`, `pitches` and `tempos` as for infer_batch_with_values."""
        from .job import SynthesisJob
        n = len(batches)
        _config_array(configs, n)
        _seed_arrays(seeds, n)
        _rate_array(output_rates, n)
        _loudness_array(loudness, n)
        _gain_array(gains, n)
        _prosody_arrays(pitches, tempos, n)
        if n == 0:
            return []
        if any(len(b) == 0 for b in batches):
            raise OperationError("Failed to run model inference. Error: empty input sequence")
        job = SynthesisJob(self, batches, configs=configs, seeds=seeds, output_rates=output_rates, loudness=loudness,
                           pitches=pitches, tempos=tempos)
        try:
            job.run()
            return job.fetch_flac(gains)
        finally:
            job.close()

    def speak_batch_flac(self, phoneme_batches: Sequence[str],
                         configs: Optional[Sequence[PiperSynthesisConfig]] = None, seeds: Optional[Sequence] = None,
                         output_rates: Optional[Sequence] = None, loudness: Optional[Sequence] = None,
                         gains: Optional[Sequence] = None, pitches: Optional[Sequence] = None,
                         tempos: Optional[Sequence] = None) -> List[bytes]:
        """speak_batch delivered as FLAC streams: infer_batch_flac over the phonemes' ids."""
        _config_array(configs, len(phoneme_batches))
        return self.infer_batch_flac([self.phonemes_to_input_ids(p) for p in phoneme_batches], configs, seeds,
                                     output_rates, loudness, gains, pitches, tempos)

    def _cfg(self, fn) -> PiperSynthesisConfig:
        c, err = N.sb200_synth_config(), N.sb200_error()
        _check(fn(self._h, C.byref(c), C.byref(err)), err)
        return PiperSynthesisConfig(int(c.speaker) if c.has_speaker else None, float(c.noise_scale),
                                    float(c.length_scale), float(c.noise_w))

    def get_default_synthesis_config(self) -> PiperSynthesisConfig:
        return self._cfg(self._lib.sb200_get_default_synthesis_config)

    def get_fallback_synthesis_config(self) -> PiperSynthesisConfig:
        return self._cfg(self._lib.sb200_get_fallback_synthesis_config)

    def set_fallback_synthesis_config(self, synthesis_config) -> None:
        if not isinstance(synthesis_config, PiperSynthesisConfig):
            raise OperationError("Invalid configuration for Vits Model")
        c = N.sb200_synth_config(synthesis_config.speaker or 0, 0 if synthesis_config.speaker is None else 1,
                                 synthesis_config.noise_scale, synthesis_config.length_scale, synthesis_config.noise_w)
        err = N.sb200_error()
        _check(self._lib.sb200_set_fallback_synthesis_config(self._h, C.byref(c), C.byref(err)), err)

    def _str(self, fn) -> str:
        p, err = C.c_void_p(), N.sb200_error()
        _check(fn(self._h, C.byref(p), C.byref(err)), err)
        s = C.string_at(p).decode("utf-8")
        self._lib.sb200_string_free(p)
        return s

    def get_language(self) -> Optional[str]:
        return self._str(self._lib.sb200_get_language)

    def properties(self) -> dict:
        return {"quality": self._str(self._lib.sb200_get_quality)}

    def speaker_name_to_id(self, name: str) -> Optional[int]:
        r = int(self._lib.sb200_speaker_name_to_id(self._h, name.encode("utf-8")))
        return None if r < 0 else r

    def supports_streaming_output(self) -> bool:
        return False

    def stream_synthesis(self, phonemes: str, chunk_size: int, chunk_padding: int, seed: Optional[int] = None):
        raise OperationError("Streaming synthesis is not supported for this model")

    def set_backend(self, backend: int) -> int:
        return int(self._lib.sb200_set_backend(self._h, backend))


class VitsModel(_VitsCommons):
    """piper/src/lib.rs:291-478"""


class EncoderOutputs:
    """piper/src/lib.rs:671-763 — `z` stays on the device."""

    def __init__(self, model: "_VitsCommons", handle: C.c_void_p):
        self._m, self._h = model, handle
        self.num_frames = int(model._lib.sb200_latent_frames(handle))
        # frames per id of the encoder pass (the reference's optional `p_duration` output)
        n = int(model._lib.sb200_latent_id_frames(handle, None, 0))
        self.p_duration = np.zeros(n, np.int32)
        model._lib.sb200_latent_id_frames(handle, _ptr(self.p_duration, C.c_int32), n)

    def infer_decoder(self, lo: int = 0, hi: Optional[int] = None) -> AudioSamples:
        hi = self.num_frames if hi is None else hi
        a, err = N.sb200_audio(), N.sb200_error()
        _check(self._m._lib.sb200_decode_chunk(self._m._h, self._h, lo, hi, C.byref(a), C.byref(err)), err)
        return _take_audio(a).samples

    def __del__(self):
        try:
            if self._h:
                self._m._lib.sb200_latent_free(self._h)
                self._h = None
        except Exception:
            pass


class Resampler:
    """One stream's output-rate resampler on the device (sb200_resampler_*): it carries the stream's last inputs and
    counts between chunks, so the concatenation of what it emits is the whole stream resampled at once.  `out_rate`: one
    of OUTPUT_RATES other than the voice's own."""

    def __init__(self, model: "_VitsCommons", out_rate: int):
        _rate_array([out_rate], 1)
        self._m, self.rate, self._h = model, int(out_rate), C.c_void_p()
        err = N.sb200_error()
        _check(model._lib.sb200_resampler_create(model._h, int(out_rate), C.byref(self._h), C.byref(err)), err)

    def __del__(self):
        try:
            if self._h:
                self._m._lib.sb200_resampler_free(self._h)
                self._h = None
        except Exception:
            pass


def _stream_resampler(model, output_rate) -> Optional[Resampler]:
    """A Resampler for a stream at output_rate, or None when the stream stays at the voice's rate."""
    _rate_array([output_rate], 1)
    if not output_rate or int(output_rate) == model.audio_output_info().sample_rate:
        return None
    return Resampler(model, output_rate)


class ProsodyStream:
    """One stream's pitch and tempo state on the device (sb200_prosody_stream_*): it carries the tails of the stream's
    input and stretched signal, and its last frames' offsets, between chunks, so the concatenation of what it emits is
    the whole stream warped at once.  `pitch` / `tempo`: ratios as for infer_batch_with_values, not both neutral."""

    def __init__(self, model: "_VitsCommons", pitch=None, tempo=None):
        p, t = _prosody_arrays([pitch], [tempo], 1)
        if p is None and t is None:
            raise OperationError("a prosody stream needs a pitch or a tempo ratio other than 1 (None, NaN or 1: none)")
        self._m, self._h = model, C.c_void_p()
        self.pitch = None if p is None else float(p[0])
        self.tempo = None if t is None else float(t[0])
        err = N.sb200_error()
        _check(model._lib.sb200_prosody_stream_create(model._h, float("nan") if p is None else float(p[0]),
                                                      float("nan") if t is None else float(t[0]), C.byref(self._h),
                                                      C.byref(err)), err)

    def last_pass_ms(self) -> Tuple[float, float]:
        """The "stretch" and "pitch" device time (ms) of the last chunk pass this stream was in."""
        s, p = C.c_float(), C.c_float()
        self._m._lib.sb200_prosody_stream_profile(self._h, C.byref(s), C.byref(p))
        return float(s.value), float(p.value)

    def __del__(self):
        try:
            if self._h:
                self._m._lib.sb200_prosody_stream_free(self._h)
                self._h = None
        except Exception:
            pass


def _stream_prosody(model, pitch, tempo) -> Optional[ProsodyStream]:
    """A ProsodyStream for a stream with these ratios, or None when neither asks for anything."""
    p, t = _prosody_arrays([pitch], [tempo], 1)
    if p is None and t is None:
        return None
    return ProsodyStream(model, pitch, tempo)


def _trim_frames(trim: slice) -> Tuple[int, int]:
    """The overlap frames a SpeechStreamer audio slice drops at each end."""
    return (trim.start or 0) // HOP, (-trim.stop // HOP) if trim.stop is not None else 0


class SpeechStreamer:
    """piper/src/lib.rs:765-858: chunked decoder runs with overlap trimming + crossfade(42).  With a resampler, each
    chunk's trim and crossfade run on the device and the chunk leaves at the resampler's rate.  With an encoding, they
    run on the device too and each chunk leaves as G.711 bytes of its to_i16_vec after `gain`."""

    def __init__(self, enc: EncoderOutputs, chunk_size: int, chunk_padding: int,
                 resampler: Optional[Resampler] = None, encoding: Optional[str] = None, gain: float = 1.0,
                 warp: Optional[ProsodyStream] = None):
        self.enc = enc
        self.chunker = AdaptiveMelChunker(enc.num_frames, chunk_size, chunk_padding)
        self.one_shot = enc.num_frames <= (chunk_size * 2 + chunk_padding * 2)
        self.resampler = resampler
        self.encoding, self.gain = encoding, gain
        self.warp = warp

    def __iter__(self) -> Iterator[AudioSamples]:
        return self

    def __next__(self) -> AudioSamples:
        (m0, m1), (a0, a1) = next(self.chunker)
        # encoded, resampled or warped: the post-path runs on the device, then the stream's resampler / prosody stream
        if self.encoding is not None or self.resampler is not None or self.warp is not None:
            if self.one_shot:
                self.chunker.consume()
                chunk, fade = (self.enc, 0, self.enc.num_frames, 0, 0), 0
            else:
                hi = self.enc.num_frames if m1 is None else m1
                chunk, fade = (self.enc, m0, hi) + _trim_frames(slice(a0, a1)), 42
            kw = {}
            if self.resampler is not None or self.warp is not None:     # whether this chunk ends the stream: after
                kw.update(resamplers=[self.resampler],                  # the one-shot consume()
                          last=[self.chunker.last_end_index is None])
            if self.warp is not None:
                kw["warps"] = [self.warp]
            if self.encoding is not None:
                kw.update(gains=[self.gain], encoding=self.encoding)
            return self.enc._m.infer_decoder_batch([chunk], fade=fade, **kw)[0]
        if self.one_shot:
            self.chunker.consume()
            return self.enc.infer_decoder()
        hi = self.enc.num_frames if m1 is None else m1
        audio = self.enc.infer_decoder(m0, hi).as_slice()
        audio = audio[a0:a1] if a1 is not None else audio[a0:]
        out = AudioSamples(audio)
        out.crossfade(42)
        return out


class VitsStreamingModel(_VitsCommons):
    """piper/src/lib.rs:480-669"""

    def infer_encoder(self, input_phonemes: Sequence[int]) -> EncoderOutputs:
        ids = np.ascontiguousarray(input_phonemes, dtype=np.int64)
        h, err = C.c_void_p(), N.sb200_error()
        _check(self._lib.sb200_encode_ids(self._h, ids.ctypes.data_as(C.POINTER(C.c_int64)), ids.size, C.byref(h),
                                          C.byref(err)), err)
        return EncoderOutputs(self, h)

    def infer_encoder_batch(self, batches: Sequence[Sequence[int]],
                            configs: Optional[Sequence[PiperSynthesisConfig]] = None,
                            duration_scales: Optional[Sequence] = None,
                            durations: Optional[Sequence] = None,
                            seeds: Optional[Sequence] = None) -> List[EncoderOutputs]:
        """infer_encoder over many utterances in one encoder pass.  `configs`: one PiperSynthesisConfig per utterance,
        or None for the fallback config; each latent equals infer_encoder alone with its config as the fallback,
        except for the on-device noise of an unseeded utterance, whose draws depend on the batch position.
        `duration_scales` / `durations`: per-id duration controls as for infer_batch_with_durations; each output's
        `p_duration` holds its frames per id.  `seeds`: noise seeds as for infer_batch_with_values; a seeded latent
        equals the `z` of the same utterance synthesised with the same seed."""
        n = len(batches)
        cfgs = _config_array(configs, n)
        scales, frames = _duration_arrays([len(b) for b in batches], duration_scales, durations)
        sv, sf = _seed_arrays(seeds, n)
        if any(len(b) == 0 for b in batches):
            raise OperationError("Failed to run model inference. Error: empty input sequence")
        if n == 0:
            return []
        packed = np.ascontiguousarray(np.concatenate([np.asarray(b, dtype=np.int64) for b in batches]))
        offs = np.zeros(n + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(b) for b in batches])
        outs = (C.c_void_p * n)()
        err = N.sb200_error()
        _check(self._lib.sb200_encode_batch_ids_seeded(self._h, packed.ctypes.data_as(C.POINTER(C.c_int64)),
                                                       offs.ctypes.data_as(C.POINTER(C.c_size_t)), n, cfgs,
                                                       _ptr(scales, C.c_float), _ptr(frames, C.c_int32),
                                                       _ptr(sv, C.c_uint64), _ptr(sf, C.c_int32), outs,
                                                       C.byref(err)), err)
        return [EncoderOutputs(self, C.c_void_p(outs[i])) for i in range(n)]

    def infer_decoder_batch(self, chunks: Sequence[tuple], pcm16: bool = False, fade: int = 0,
                            gains: Optional[Sequence[float]] = None, resamplers: Optional[Sequence] = None,
                            last: Optional[Sequence[bool]] = None, encoding: Optional[str] = None,
                            warps: Optional[Sequence] = None) -> list:
        """Many `EncoderOutputs.infer_decoder(lo, hi)` calls as one decoder pass.  `chunks`: (encoder outputs, lo, hi)
        per chunk; each result equals that chunk decoded alone, bit for bit.

        With pcm16, a chunk may be (encoder outputs, lo, hi, trim_lo, trim_hi) and each result is what the realtime
        mode emits for it as int16: trim_lo / trim_hi overlap frames dropped, crossfade(fade), gains[k] (None: 1),
        peak-normalised to the chunk's own peak.

        With `resamplers` (one Resampler or None per chunk), chunks may carry trims in either format: after the same
        post-path each chunk is appended to its stream's resampler and the result is what that stream emits for it at
        its output rate (AudioSamples, or int16 normalised to the emitted samples' own peak with pcm16); last[k] flushes
        the stream.  A None resampler returns the chunk after the post-path at the voice's rate.

        With `encoding` ("mulaw" or "alaw"; None: none), chunks take pcm16's tuples and each result is `bytes`: G.711 of
        the int16 samples pcm16 returns for that chunk (with or without resamplers), encoded on the device in the same
        launches.

        With `warps` (one ProsodyStream or None per chunk; chunks may carry trims, as with resamplers), chunk k after
        the post-path is appended to its prosody stream first, and what that emits goes on to resamplers[k] (None
        entries, or resamplers None: the voice's rate) and the conversion; last[k] flushes both streams."""
        refuse_flac(encoding, "a decoder chunk pass")
        check_encoding(encoding)
        if encoding is not None and pcm16:
            raise OperationError("pcm16 and an encoding are two output formats: give one")
        n = len(chunks)
        lo, hi = np.zeros(n, np.int64), np.zeros(n, np.int64)
        tlo, thi = np.zeros(n, np.int64), np.zeros(n, np.int64)
        hs = (C.c_void_p * n)()
        for k, c in enumerate(chunks):
            if len(c) not in ((3, 5) if pcm16 or encoding or resamplers is not None or warps is not None else (3,)):
                raise OperationError(f"Invalid decoder chunk {k}: expected (encoder outputs, lo, hi"
                                     + (", trim_lo, trim_hi)" if pcm16 else ")"))
            enc = c[0]
            if not isinstance(enc, EncoderOutputs) or enc._m is not self or not enc._h:
                raise OperationError(f"Invalid decoder chunk {k}: encoder outputs of another model")
            lo[k], hi[k] = int(c[1]), int(c[2])
            if len(c) == 5:
                tlo[k], thi[k] = int(c[3]), int(c[4])
            hs[k] = enc._h.value
        if gains is not None and len(gains) != n:
            raise OperationError(f"Invalid decoder gains: {len(gains)} gains for {n} chunks")
        if n == 0:
            return []
        p64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))
        err = N.sb200_error()
        if resamplers is not None or warps is not None:
            resamplers = _per_utterance([None] * n if resamplers is None else resamplers, n, "resamplers")
            rs = (C.c_void_p * n)()
            for k, r in enumerate(resamplers):
                if r is not None and (not isinstance(r, Resampler) or not r._h):
                    raise OperationError(f"chunk {k}: not a Resampler")
                rs[k] = None if r is None else r._h.value
            ws = None
            if warps is not None:
                ws = (C.c_void_p * n)()
                for k, w in enumerate(_per_utterance(warps, n, "warps")):
                    if w is not None and (not isinstance(w, ProsodyStream) or not w._h):
                        raise OperationError(f"chunk {k}: not a ProsodyStream")
                    ws[k] = None if w is None else w._h.value
            fl = np.zeros(n, np.int32) if last is None else np.array([1 if x else 0 for x in
                                                                        _per_utterance(last, n, "last flags")], np.int32)
            g = None if gains is None else np.ascontiguousarray(gains, dtype=np.float32)
            outs = (C.c_void_p * n)()
            lens = (C.c_size_t * n)()
            fmt = G711_LAW[encoding] + 2 if encoding else 1 if pcm16 else 0
            gp = None if g is None else g.ctypes.data_as(C.POINTER(C.c_float))
            if ws is None:
                _check(self._lib.sb200_decode_chunks_resampled(
                    self._h, hs, p64(lo), p64(hi), p64(tlo), p64(thi), n, int(fade), gp, rs, _ptr(fl, C.c_int32), fmt,
                    outs, lens, C.byref(err)), err)
            else:
                _check(self._lib.sb200_decode_chunks_warped(
                    self._h, hs, p64(lo), p64(hi), p64(tlo), p64(thi), n, int(fade), gp, rs, ws, _ptr(fl, C.c_int32),
                    fmt, outs, lens, C.byref(err)), err)
            if encoding:
                return _take_bytes(self._lib, outs, lens)
            if pcm16:
                return _take_chunks(self._lib, outs, lens, np.int16)
            return [AudioSamples(a) for a in _take_chunks(self._lib, outs, lens, np.float32)]
        if encoding:
            g = None if gains is None else np.ascontiguousarray(gains, dtype=np.float32)
            outs = (C.POINTER(C.c_uint8) * n)()
            lens = (C.c_size_t * n)()
            _check(self._lib.sb200_decode_chunks_g711(self._h, hs, p64(lo), p64(hi), p64(tlo), p64(thi), n, int(fade),
                                                      None if g is None else g.ctypes.data_as(C.POINTER(C.c_float)),
                                                      G711_LAW[encoding], outs, lens, C.byref(err)), err)
            return _take_bytes(self._lib, outs, lens)
        if not pcm16:
            outs = (N.sb200_audio * n)()
            _check(self._lib.sb200_decode_chunks(self._h, hs, p64(lo), p64(hi), n, outs, C.byref(err)), err)
            return [_take_audio(outs[k]).samples for k in range(n)]
        g = None if gains is None else np.ascontiguousarray(gains, dtype=np.float32)
        outs = (C.POINTER(C.c_int16) * n)()
        lens = (C.c_size_t * n)()
        _check(self._lib.sb200_decode_chunks_i16(self._h, hs, p64(lo), p64(hi), p64(tlo), p64(thi), n, int(fade),
                                                 None if g is None else g.ctypes.data_as(C.POINTER(C.c_float)), outs,
                                                 lens, C.byref(err)), err)
        return _take_chunks(self._lib, outs, lens, np.int16)

    def supports_streaming_output(self) -> bool:
        return True

    def stream_synthesis(self, phonemes: str, chunk_size: int, chunk_padding: int,
                         seed: Optional[int] = None, output_rate: Optional[int] = None,
                         encoding: Optional[str] = None, gain: Optional[float] = None,
                         pitch: Optional[float] = None, tempo: Optional[float] = None) -> SpeechStreamer:
        """`seed`: the sentence's noise seed (see infer_batch_with_values), or None for positional noise.
        `output_rate`: the chunks' sample rate (see infer_batch_with_values), the sentence resampled as one stream.
        `encoding`: "mulaw" / "alaw" for chunks of G.711 `bytes`: each is G.711 of to_i16_vec of the chunk the stream
        yields without an encoding, after the linear `gain` (None: 1; encoded streams only), encoded on the device.
        `pitch` / `tempo`: ratios as for infer_batch_with_values, the sentence warped as one stream on the device
        (ProsodyStream): the concatenation of the chunks is the sentence the stream yields without ratios, warped at
        once, then resampled and encoded as without ratios."""
        if not isinstance(self, VitsStreamingModel):
            refuse_prosody(pitch, tempo, "stream_synthesis")
        _prosody_arrays([pitch], [tempo], 1)
        _seed_arrays([seed], 1)
        _rate_array([output_rate], 1)
        refuse_flac(encoding, "stream_synthesis")
        g = _stream_gain(encoding, gain)
        ids = self.phonemes_to_input_ids(phonemes)
        enc = self.infer_encoder(ids) if seed is None else self.infer_encoder_batch([ids], seeds=[seed])[0]
        return SpeechStreamer(enc, chunk_size, chunk_padding, _stream_resampler(self, output_rate), encoding, g,
                              _stream_prosody(self, pitch, tempo))


def _stream_gain(encoding, gain) -> float:
    """Checks a stream's encoding and gain; the gain as a float (1 when None)."""
    check_encoding(encoding)
    if gain is None:
        return 1.0
    if encoding is None:
        raise OperationError("a stream's gain applies before its G.711 encoding: give an encoding with it")
    return float(_gain_array([gain], 1)[0])


class _Stream:
    """One sentence of a StreamBatch: its latent and its own chunk schedule, with SpeechStreamer's one-shot rule."""

    def __init__(self, key, enc, chunk_size: int, chunk_padding: int, resampler: Optional[Resampler] = None,
                 encoding: Optional[str] = None, gain: float = 1.0, warp: Optional[ProsodyStream] = None):
        self.key, self.enc, self.resampler = key, enc, resampler
        self.encoding, self.gain = encoding, gain
        self.warp = warp
        self.chunker = AdaptiveMelChunker(enc.num_frames, chunk_size, chunk_padding)
        self.one_shot = enc.num_frames <= (chunk_size * 2 + chunk_padding * 2)

    def next_chunk(self):
        """(lo, hi, audio slice or None): the frames to decode next, and how SpeechStreamer.__next__ trims them (None:
        the one-shot chunk, returned as decoded)."""
        (m0, m1), (a0, a1) = next(self.chunker)
        if self.one_shot:
            self.chunker.consume()
            return 0, self.enc.num_frames, None
        return m0, self.enc.num_frames if m1 is None else m1, slice(a0, a1)

    @property
    def done(self) -> bool:
        return self.chunker.last_end_index is None


def _check_chunking(chunk_size, chunk_padding):
    if not isinstance(chunk_size, int) or chunk_size < 1:
        raise OperationError(f"Invalid chunk size {chunk_size!r}: expected a positive integer")
    if not isinstance(chunk_padding, int) or chunk_padding < 0:
        raise OperationError(f"Invalid chunk padding {chunk_padding!r}: expected a non-negative integer")


class StreamBatch:
    """Many realtime streams served together (a server holding K `stream_synthesis` clients).

    `add` admits a sentence (phonemes or ids) with an optional PiperSynthesisConfig (None: the fallback config); a
    config whose speaker the voice does not have is refused there.  Each `step` encodes every stream added since the
    last step in ONE encoder pass, then decodes the next chunk of every active stream in ONE decoder pass, and returns
    [(key, AudioSamples)] in admission order.  Each stream keeps its own AdaptiveMelChunker, trim, one-shot rule and
    crossfade(42), so its chunks are exactly what `stream_synthesis` yields for that sentence with its config as the
    fallback.  A stream added with an output rate has its own resampler: its chunks are trimmed, crossfaded and
    resampled on the device.  Those chunks go through a second decoder pass of the step (a third for one-shot ones,
    which are not crossfaded), so the streams at the voice's rate keep their pass and their bits.  A stream added with
    an encoding yields G.711 `bytes` (see stream_synthesis); its chunks go through a pass per encoding, output rate or
    not, and one-shot or not, with its trim, crossfade and gain on the device.

    One stream's failure stays that stream's, as with one `stream_synthesis` per client: when a batched pass raises,
    its streams are run one at a time, and a stream whose own encoder or decoder work fails gets its SonataError as
    its item, (key, error), once, and ends.  The other streams carry on."""

    def __init__(self, model, chunk_size: int, chunk_padding: int):
        _check_chunking(chunk_size, chunk_padding)
        self.model = model
        self.chunk_size, self.chunk_padding = chunk_size, chunk_padding
        self._pending: list = []      # (key, ids, config, chunk_size, seed, output rate, encoding, gain) not encoded yet
        self._active: List[_Stream] = []
        self._next_key = 0

    def add(self, ids_or_phonemes, config: Optional[PiperSynthesisConfig] = None, seed: Optional[int] = None,
            output_rate: Optional[int] = None, encoding: Optional[str] = None, gain: Optional[float] = None,
            pitch: Optional[float] = None, tempo: Optional[float] = None) -> int:
        """`seed`: the stream's noise seed (see infer_batch_with_values); a seeded stream yields what
        `stream_synthesis(..., seed=seed)` yields, whatever other streams share its encoder pass.  `output_rate`,
        `encoding` and `gain`: the stream's sample rate and G.711 encoding, as for stream_synthesis; `pitch` / `tempo`:
        its ratios, as there.  A warped stream's chunks go through passes of their own, so the other streams keep their
        passes and their bits."""
        if not isinstance(self.model, VitsStreamingModel):
            refuse_prosody(pitch, tempo, "StreamBatch")
        return self._add(ids_or_phonemes, config, self.chunk_size, seed, output_rate, encoding, gain, pitch, tempo)

    def _add(self, ids_or_phonemes, config, chunk_size: int, seed: Optional[int] = None,
             output_rate: Optional[int] = None, encoding: Optional[str] = None, gain: Optional[float] = None,
             pitch: Optional[float] = None, tempo: Optional[float] = None) -> int:
        if config is not None and not isinstance(config, PiperSynthesisConfig):
            raise OperationError("Invalid configuration for Vits Model")
        _prosody_arrays([pitch], [tempo], 1)
        _seed_arrays([seed], 1)
        _rate_array([output_rate], 1)
        refuse_flac(encoding, "StreamBatch")
        gain = _stream_gain(encoding, gain)
        if config is not None and config.speaker is not None and config.speaker not in (self.model.get_speakers() or {}):
            raise OperationError(f"No speaker was found with the given id `{config.speaker}`")     # as check_config
        _check_chunking(chunk_size, self.chunk_padding)
        if isinstance(ids_or_phonemes, str):
            ids = self.model.phonemes_to_input_ids(ids_or_phonemes)
        else:
            ids = [int(i) for i in ids_or_phonemes]
        if not ids:
            raise OperationError("Failed to run model inference. Error: empty input sequence")
        key = self._next_key
        self._next_key += 1
        self._pending.append((key, ids, config, chunk_size, seed, output_rate, encoding, gain, pitch, tempo))
        return key

    def __len__(self) -> int:
        """Streams added and not yet finished."""
        return len(self._pending) + len(self._active)

    def __contains__(self, key) -> bool:
        """Whether stream `key` has chunks still to come."""
        return any(p[0] == key for p in self._pending) or any(s.key == key for s in self._active)

    def step(self) -> List[tuple]:
        out = []
        active = self._active
        if self._pending:
            pend, self._pending = self._pending, []
            fallback = None
            if any(p[2] is not None for p in pend):
                fallback = self.model.get_fallback_synthesis_config()

            def encode(ps):
                configs = None if fallback is None else [fallback if p[2] is None else p[2] for p in ps]
                if all(p[4] is None for p in ps):
                    return self.model.infer_encoder_batch([p[1] for p in ps], configs)
                return self.model.infer_encoder_batch([p[1] for p in ps], configs, seeds=[p[4] for p in ps])
            for p, (enc, err) in zip(pend, _each_or_alone(encode, pend)):
                if err is None:
                    try:
                        active.append(_Stream(p[0], enc, p[3], self.chunk_padding,
                                              _stream_resampler(self.model, p[5]), p[6], p[7],
                                              _stream_prosody(self.model, p[8], p[9])))
                        continue
                    except SonataError as e:
                        err = e
                out.append((p[0], err))
        plan = [(s,) + s.next_chunk() for s in active]
        failed = set()
        # one pass per (encoding, resampled, one-shot, warped): the streams without an encoding first, in their usual
        # passes; warped streams in passes of their own
        plain_key = (None, False, False, False)
        groups = {plain_key: [], (None, True, False, False): [], (None, True, True, False): []}
        for p in plan:
            s = p[0]
            plain = s.encoding is None and s.resampler is None and s.warp is None
            k = plain_key if plain else (s.encoding, s.resampler is not None, p[3] is None, s.warp is not None)
            groups.setdefault(k, []).append(p)

        def device_post(pl, key):
            encoding, resampled, whole, warped = key
            chunks = [(s.enc, lo, hi) + ((0, 0) if trim is None else _trim_frames(trim)) for s, lo, hi, trim in pl]
            extra = {} if not (resampled or warped) else {"resamplers": [p[0].resampler for p in pl],
                                                          "last": [p[0].done for p in pl]}
            if warped:
                extra["warps"] = [p[0].warp for p in pl]
            if encoding is not None:
                extra.update(encoding=encoding, gains=[p[0].gain for p in pl])
            return self.model.infer_decoder_batch(chunks, fade=0 if whole else 42, **extra)
        decoded = {}
        for key, group in groups.items():
            if key == plain_key:
                call = lambda pl: self.model.infer_decoder_batch([(s.enc, lo, hi) for s, lo, hi, _ in pl])
            else:
                call = lambda pl, key=key: device_post(pl, key)
            if group:
                decoded.update({id(p): r for p, r in zip(group, _each_or_alone(call, group))})
        for p in plan:
            s, _, _, trim = p
            a, err = decoded[id(p)]
            if err is not None:
                out.append((s.key, err))
                failed.add(s.key)
                continue
            if trim is not None and s.resampler is None and s.encoding is None and s.warp is None:
                a = AudioSamples(a.as_slice()[trim])
                a.crossfade(42)
            out.append((s.key, a))
        self._active = [s for s in active if not s.done and s.key not in failed]
        return out


def _each_or_alone(call, items):
    """call(items) as one pass -> [(result, None)]; when that pass raises a SonataError, each item alone, so an item's
    failure is reported as its own (None, error) and the others still get their results."""
    try:
        return [(r, None) for r in call(items)]
    except SonataError as e:
        if len(items) == 1:
            return [(None, e)]
    out = []
    for it in items:
        try:
            out.append((call([it])[0], None))
        except SonataError as e:
            out.append((None, e))
    return out


def from_config_path(config_path, device: int = 0):
    """sonata_piper::from_config_path (piper/src/lib.rs:88-110): `streaming: true` selects the
    two-stage model."""
    import json
    try:
        with open(config_path, "r", encoding="utf-8") as f:
            streaming = bool(json.load(f).get("streaming") or False)
    except OSError:
        streaming = False   # let the library produce the reference's FailedToLoadResource error
    except ValueError:
        streaming = False
    return (VitsStreamingModel if streaming else VitsModel)(config_path, device)
