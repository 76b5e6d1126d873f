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
                   PhonemizationError, SonataError, check_encoding, check_watermark, refuse_flac)

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


def _loudness_array(targets, n: int, who: Optional[Sequence[str]] = None):
    """The C image of per-utterance loudness targets (f32, NaN for none), or None when `targets` is None or holds no
    target.  targets[b] is a LUFS value, finite and in [-70, 0], or None / NaN (utterance b is measured only).  Errors
    name who[b] (default "utterance b")."""
    if targets is None:
        return None
    out = np.full(n, np.nan, np.float32)
    for b, t in enumerate(_per_utterance(targets, n, "loudness targets")):
        name = f"utterance {b}" if who is None else who[b]
        if t is None:
            continue
        if isinstance(t, bool) or not isinstance(t, numbers.Real):
            raise OperationError(f"{name}: loudness target {t!r} is not a number")
        if math.isnan(float(t)):
            continue
        if not (math.isfinite(float(t)) and -70.0 <= float(t) <= 0.0):
            raise OperationError(f"{name}: loudness target {float(t)} LUFS is not a finite value in [-70, 0]")
        out[b] = float(t)
    return None if np.isnan(out).all() else out


MAX_GAIN_RANGE = (0.0, 40.0)     # the maximum gains (dB) a live loudness meter may apply


def _check_max_gain(max_gain_db, who: str) -> float:
    """A live loudness meter's maximum gain in dB as a float: finite and in [0, 40], or the call fails naming `who`."""
    if isinstance(max_gain_db, bool) or not isinstance(max_gain_db, numbers.Real):
        raise OperationError(f"{who}: maximum gain {max_gain_db!r} is not a number")
    g = float(max_gain_db)
    if not (math.isfinite(g) and MAX_GAIN_RANGE[0] <= g <= MAX_GAIN_RANGE[1]):
        raise OperationError(f"{who}: maximum gain {g} dB is not a finite value in [0, 40]")
    return g


PITCH_RANGE = (0.5, 2.0)     # pitch ratios a result can be shifted by
TEMPO_RANGE = (0.25, 4.0)    # tempo ratios a result can be played at
FORMANT_RANGE = (0.5, 2.0)   # formant ratios a result's spectral envelope can be moved by


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


def _formant_array(values, n: int):
    """The C image of per-utterance formant ratios (f32, NaN for none), or None when not given or when every entry is
    None / NaN.  Unlike a pitch or tempo ratio, 1.0 asks for something: the voice's own formants under a pitch ratio or
    contour."""
    if values is None:
        return None
    out = np.full(n, np.nan, np.float32)
    for b, v in enumerate(_per_utterance(values, n, "formant ratios")):
        if v is None:
            continue
        if isinstance(v, bool) or not isinstance(v, numbers.Real):
            raise OperationError(f"utterance {b}: formant ratio {v!r} is not a number")
        if math.isnan(float(v)):
            continue
        if not (math.isfinite(float(v)) and FORMANT_RANGE[0] <= float(v) <= FORMANT_RANGE[1]):
            raise OperationError(f"utterance {b}: formant ratio {float(v)} is not a finite value in "
                                 f"[{FORMANT_RANGE[0]}, {FORMANT_RANGE[1]}] (None or NaN: none)")
        out[b] = float(v)
    return None if np.isnan(out).all() else out


def _stream_formant(formant_ratio, who: str) -> Optional[float]:
    """A stream's formant ratio as a float, or None for None / NaN; an OperationError names the stream `who`."""
    if formant_ratio is None:
        return None
    if isinstance(formant_ratio, bool) or not isinstance(formant_ratio, numbers.Real):
        raise OperationError(f"{who}: formant ratio {formant_ratio!r} is not a number")
    v = float(formant_ratio)
    if math.isnan(v):
        return None
    if not (math.isfinite(v) and FORMANT_RANGE[0] <= v <= FORMANT_RANGE[1]):
        raise OperationError(f"{who}: formant ratio {v} is not a finite value in "
                             f"[{FORMANT_RANGE[0]}, {FORMANT_RANGE[1]}] (None or NaN: none)")
    return v


def refuse_formants(formant_ratio, where: str) -> None:
    """OperationError when `where`, a mode that hands out a sentence chunk by chunk, is asked for a formant ratio."""
    if formant_ratio is not None and not (isinstance(formant_ratio, numbers.Real) and math.isnan(float(formant_ratio))):
        raise OperationError(f"{where} cannot apply a formant ratio: the formant stage is not carried from chunk to "
                             "chunk (use speak_batch, a SynthesisJob or the lazy, parallel or file modes)")


def _blend_terms(model, blend, who: str) -> List[Tuple[int, float]]:
    """The (speaker id, f32 weight) pairs of one blend, a mapping {speaker: weight} whose keys are ids or names of the
    voice's speaker_id_map, checked as the library checks a blend (include/sonata_b200.h, sb200_speak_batch_ids_blends);
    errors name `who` and the speaker or weight."""
    p = f"{who}: speaker blend: "
    speakers = model.get_speakers()
    if not speakers:
        raise OperationError(p + "the voice has a single speaker")
    if not isinstance(blend, dict) and not hasattr(blend, "items"):
        raise OperationError(p + f"{blend!r} is not a mapping of speakers to weights")
    sids, seen = [], set()
    for key, u in blend.items():
        if isinstance(key, str):
            sid = model.speaker_name_to_id(key)
            if sid is None:
                raise OperationError(p + f"No speaker was found with the name `{key}`")
        elif type(key) is int or isinstance(key, numbers.Integral) and not isinstance(key, bool):
            sid = int(key)
            if sid not in speakers:
                raise OperationError(p + f"No speaker was found with the given id `{sid}`")
        else:
            raise OperationError(p + f"speaker {key!r} is neither an id nor a name")
        if sid in seen:
            raise OperationError(p + f"speaker {sid} appears more than once")
        if type(u) is not float and (isinstance(u, bool) or not isinstance(u, numbers.Real)):
            raise OperationError(p + f"the weight {u!r} of speaker {sid} is not a number")
        seen.add(sid)
        sids.append(sid)
    if not sids:
        raise OperationError(p + "the blend is empty")
    u = list(blend.values())
    with np.errstate(over="ignore"):
        w = np.array(u, np.float64).astype(np.float32)
    bad = np.flatnonzero(~(np.isfinite(w) & (w >= 0)))
    if bad.size:
        i = int(bad[0])
        raise OperationError(p + f"the weight {float(u[i])} of speaker {sids[i]} is not a finite number >= 0")
    if not w.any():
        raise OperationError(p + "every weight is zero")
    return list(zip(sids, w.tolist()))


def _blend_arrays(model, blends, n: int, who: Optional[Sequence[str]] = None):
    """The C image of per-utterance speaker blends: (speakers i64, weights f32, offsets size_t [n + 1]), or
    (None, None, None) when `blends` is None or every entry is None.  blends[b] is a mapping {speaker: weight} (see
    _blend_terms) or None for the utterance's config speaker.  Errors name utterance b, or who[b]."""
    if blends is None:
        return None, None, None
    terms = []
    for b, v in enumerate(_per_utterance(blends, n, "speaker blends")):
        terms.append([] if v is None else _blend_terms(model, v, f"utterance {b}" if who is None else who[b]))
    if not any(terms):
        return None, None, None
    offs = np.zeros(n + 1, np.uint64)
    offs[1:] = np.cumsum([len(t) for t in terms])
    flat = [x for t in terms for x in t]
    return (np.array([s for s, _ in flat], np.int64), np.array([w for _, w in flat], np.float32), offs)


def _who(b) -> str:
    """What an error names: utterance b of a batch, or a label such as "stream 3" given instead of the index."""
    return b if isinstance(b, str) else f"utterance {b}"


def _contour_value(x, b, i: int, unit: str = "id") -> float:
    if x is None:
        return math.nan
    if isinstance(x, bool) or not isinstance(x, numbers.Real):
        raise OperationError(f"{_who(b)}, {unit} {i}: pitch ratio {x!r} is not a number")
    x = float(x)
    if not (math.isnan(x) or x == 1.0 or (math.isfinite(x) and PITCH_RANGE[0] <= x <= PITCH_RANGE[1])):
        raise OperationError(f"{_who(b)}, {unit} {i}: pitch ratio {x} is not a finite value in "
                             f"[{PITCH_RANGE[0]}, {PITCH_RANGE[1]}] (NaN or 1: none)")
    return x


def _contour_arrays(lens: Sequence[int], pitch_contours=None, pitches=None, who: Optional[Sequence[str]] = None):
    """The packed C image of per-id pitch ratios (f32, NaN for none), checked as the library checks them, or None when
    not given or when no utterance has a contour.  pitch_contours[b] holds one ratio per id of utterance b (in
    PITCH_RANGE, or None / NaN / 1.0 for none), or is None.  An utterance with a contour may not also have a pitch ratio
    in `pitches` (the C image of _prosody_arrays, or None).  Numeric arrays are checked in one vectorised pass; anything
    else element by element, which also names the first bad element.  `who`: what the errors name instead of
    "utterance b" (one label per entry), for callers that are not batches."""
    if pitch_contours is None:
        return None
    n = len(lens)
    out = np.full(int(sum(lens)), np.nan, np.float32)
    pos = 0
    for b, v in enumerate(_per_utterance(pitch_contours, n, "pitch contours")):
        if v is not None:
            label = b if who is None else who[b]
            a = _numeric(v, "fiu")
            if a is None:
                v = list(v)
                a = np.array([_contour_value(x, label, i) for i, x in enumerate(v)] if len(v) == lens[b] else v)
            if a.size != lens[b]:
                raise OperationError(f"{_who(label)}: {a.size} pitch ratios for {lens[b]} ids")
            f = a.astype(np.float32)
            asked = ~np.isnan(f) & (f != 1)
            bad = np.nonzero(asked & ~(np.isfinite(f) & (f >= PITCH_RANGE[0]) & (f <= PITCH_RANGE[1])))[0]
            if bad.size:
                _contour_value(float(f[bad[0]]), label, int(bad[0]))
            if asked.any() and pitches is not None and not np.isnan(pitches[b]):
                raise OperationError(f"{_who(label)}: a pitch contour and a pitch ratio together (give one or the other)")
            out[pos:pos + lens[b]] = f
        pos += lens[b]
    return None if (np.isnan(out) | (out == 1)).all() else out


def _char_values_to_ids(v, phonemes: str, src: Sequence[int], b, what: str, check, none: float = 1.0) -> list:
    """Per-character values v (one per character of `phonemes`) as per-id values: each id takes its source character's
    value, checked by check(x, b, character, "character"); bos, eos and pads of no character take `none`.  Characters
    the voice drops have no id and their values are ignored.  b: the utterance's index, or a label naming the stream."""
    v = list(v) if not isinstance(v, np.ndarray) else v.reshape(-1).tolist()
    if len(v) != len(phonemes):
        raise OperationError(f"{_who(b)}: {len(v)} {what} for {len(phonemes)} characters")
    kept = {c: check(v[c], b, c, "character") for c in sorted(set(src)) if c >= 0}
    return [none if c < 0 else kept[c] for c in src]


VOLUME_RANGE = (-60.0, 20.0)   # volume levels (dB) an id can be given, besides -inf (silence)


def _volume_value(x, b, i: int, unit: str = "id") -> float:
    if x is None:
        return math.nan
    if isinstance(x, bool) or not isinstance(x, numbers.Real):
        raise OperationError(f"{_who(b)}, {unit} {i}: volume level {x!r} is not a number")
    x = float(x)
    if not (math.isnan(x) or x == 0.0 or x == -math.inf or
            (math.isfinite(x) and VOLUME_RANGE[0] <= x <= VOLUME_RANGE[1])):
        raise OperationError(f"{_who(b)}, {unit} {i}: volume level {x} dB is not a finite value in "
                             f"[{VOLUME_RANGE[0]}, {VOLUME_RANGE[1]}] or -inf (None, NaN or 0: none)")
    return x


def _volume_arrays(lens: Sequence[int], volume_contours=None, who: Optional[Sequence[str]] = None):
    """The packed C image of per-id volume levels in dB (f32, NaN for none), checked as the library checks them, or None
    when not given or when every level is None / NaN / 0.  volume_contours[b] holds one level per id of utterance b (in
    VOLUME_RANGE, -inf for silence, or None / NaN / 0 for none), or is None.  `who`: as for _contour_arrays."""
    if volume_contours is None:
        return None
    n = len(lens)
    out = np.full(int(sum(lens)), np.nan, np.float32)
    pos = 0
    for b, v in enumerate(_per_utterance(volume_contours, n, "volume contours")):
        if v is not None:
            label = b if who is None else who[b]
            a = _numeric(v, "fiu")
            if a is None:
                v = list(v)
                a = np.array([_volume_value(x, label, i) for i, x in enumerate(v)] if len(v) == lens[b] else v)
            if a.size != lens[b]:
                raise OperationError(f"{_who(label)}: {a.size} volume levels for {lens[b]} ids")
            f = a.astype(np.float32).reshape(-1)
            asked = ~np.isnan(f) & (f != 0)
            ok = (f == -np.inf) | (np.isfinite(f) & (f >= VOLUME_RANGE[0]) & (f <= VOLUME_RANGE[1]))
            bad = np.nonzero(asked & ~ok)[0]
            if bad.size:
                _volume_value(float(f[bad[0]]), label, int(bad[0]))
            out[pos:pos + lens[b]] = f
        pos += lens[b]
    return None if (np.isnan(out) | (out == 0)).all() else out


BREAK_RANGE_MS = (0.0, 10000.0)   # a break (ms) is in (low, high]; None, NaN or 0 ask for none


def _break_value(x, b, i: int, unit: str = "id") -> float:
    if x is None:
        return math.nan
    if isinstance(x, bool) or not isinstance(x, numbers.Real):
        raise OperationError(f"{_who(b)}, {unit} {i}: break {x!r} is not a number")
    x = float(x)
    if not (math.isnan(x) or x == 0.0 or (math.isfinite(x) and BREAK_RANGE_MS[0] < x <= BREAK_RANGE_MS[1])):
        raise OperationError(f"{_who(b)}, {unit} {i}: break {x} ms is not a finite value in "
                             f"({BREAK_RANGE_MS[0]}, {BREAK_RANGE_MS[1]}] (None, NaN or 0: none)")
    return x


def _break_arrays(lens: Sequence[int], breaks=None, who: Optional[Sequence[str]] = None):
    """The packed C image of per-id breaks in ms (f32, NaN for none), checked as the library checks them, or None when
    not given or when every break is None / NaN / 0.  breaks[b] holds one break per id of utterance b, the pause after
    that id (in BREAK_RANGE_MS, or None / NaN / 0 for none), or is None.  `who`: as for _contour_arrays."""
    if breaks is None:
        return None
    n = len(lens)
    out = np.full(int(sum(lens)), np.nan, np.float32)
    pos = 0
    for b, v in enumerate(_per_utterance(breaks, n, "breaks")):
        if v is not None:
            label = b if who is None else who[b]
            a = _numeric(v, "fiu")
            if a is None:
                v = list(v)
                a = np.array([_break_value(x, label, i) for i, x in enumerate(v)] if len(v) == lens[b] else v)
            if a.size != lens[b]:
                raise OperationError(f"{_who(label)}: {a.size} breaks for {lens[b]} ids")
            f = a.astype(np.float32).reshape(-1)
            asked = ~np.isnan(f) & (f != 0)
            bad = np.nonzero(asked & ~(np.isfinite(f) & (f > BREAK_RANGE_MS[0]) & (f <= BREAK_RANGE_MS[1])))[0]
            if bad.size:
                _break_value(float(f[bad[0]]), label, int(bad[0]))
            out[pos:pos + lens[b]] = f
        pos += lens[b]
    return None if (np.isnan(out) | (out == 0)).all() else out


def _char_breaks_to_ids(v, phonemes: str, src: Sequence[int], b) -> list:
    """Per-character breaks v (one per character of `phonemes`) as per-id breaks: a character's break goes after the
    last id it maps to (its pad); a character the voice drops puts its break after the last id before it (bos when no
    kept character precedes it), so no requested pause is lost.  Breaks that land on one id add up.  Each break is
    checked by _break_value, naming its character."""
    v = list(v) if not isinstance(v, np.ndarray) else v.reshape(-1).tolist()
    if len(v) != len(phonemes):
        raise OperationError(f"{_who(b)}: {len(v)} breaks for {len(phonemes)} characters")
    ms = [_break_value(x, b, c, "character") for c, x in enumerate(v)]
    # the ids a break can follow: bos (before every character) and each id of a kept character, in order
    keys = [(-1 if i == 0 else int(c), i) for i, c in enumerate(src) if i == 0 or int(c) >= 0]
    out = [math.nan] * len(src)
    for c, x in enumerate(ms):
        if math.isnan(x) or x == 0.0:
            continue
        i = [i for k, i in keys if k <= c][-1]
        out[i] = x if math.isnan(out[i]) else out[i] + x
    return out


def _breaks_ask(image, rate: int) -> bool:
    """Whether a per-id breaks image (of _break_arrays, or None) asks for a pause of one sample or more at `rate`: some
    floor(ms * rate / 1000 + 0.5) > 0, in double as the library computes it."""
    if image is None:
        return False
    ms = image.astype(np.float64)
    ms = ms[~np.isnan(ms)]
    return bool(np.any(np.floor(ms * rate / 1000.0 + 0.5) > 0))


TARGET_RANGE_MS = (0.0, 600000.0)   # a target duration (ms) is in (low, high]; None or NaN ask for none


def _target_ms(x, label, k: Optional[int]) -> float:
    """A target duration checked as the library checks it (NaN for None); k: its span, or None for a whole utterance."""
    where = _who(label) if k is None else f"{_who(label)}, span {k}"
    if x is None:
        return math.nan
    if isinstance(x, bool) or not isinstance(x, numbers.Real):
        raise OperationError(f"{where}: target duration {x!r} is not a number")
    x = float(x)
    if not (math.isnan(x) or (math.isfinite(x) and TARGET_RANGE_MS[0] < x <= TARGET_RANGE_MS[1])):
        raise OperationError(f"{where}: target duration {x} ms is not a finite value in "
                             f"({TARGET_RANGE_MS[0]}, {TARGET_RANGE_MS[1]}] (None or NaN: none)")
    return x


def _target_entry(v, label, tempo=None, count: Optional[int] = None, unit: str = "id"):
    """One utterance's target durations, checked for form: None, a duration in ms for the whole utterance (a float, NaN
    for none), or a list of (first, last, ms) spans, inclusive, ascending and disjoint (a list of (int, int, float)).
    `count`: the ids (or characters) the spans index, None when not known yet.  An entry that asks for something with a
    tempo ratio (tempo not None / NaN) is refused."""
    if v is None:
        return None
    if isinstance(v, numbers.Real) and not isinstance(v, bool):
        out = _target_ms(v, label, None)
        asks = not math.isnan(out)
    else:
        if isinstance(v, (str, bytes)) or not hasattr(v, "__iter__"):
            raise OperationError(f"{_who(label)}: target durations {v!r} are neither a duration in ms nor a list of "
                                 "(first, last, ms) spans")
        out, prev, asks = [], -1, False
        for k, sp in enumerate(v):
            if isinstance(sp, (str, bytes)) or not hasattr(sp, "__len__") or len(sp) != 3:
                raise OperationError(f"{_who(label)}, span {k}: {sp!r} is not a (first, last, ms) span")
            a, b, ms = sp
            if any(isinstance(x, bool) or not isinstance(x, numbers.Integral) for x in (a, b)):
                raise OperationError(f"{_who(label)}, span {k}: {unit}s {a!r} .. {b!r} are not integers")
            a, b = int(a), int(b)
            if not (0 <= a <= b and (count is None or b < count)):
                raise OperationError(f"{_who(label)}, span {k}: {unit}s {a} .. {b} are not a range of the "
                                     + (f"{count} {unit}s" if count is not None else f"{unit}s"))
            if a <= prev:
                raise OperationError(f"{_who(label)}, span {k}: {unit}s {a} .. {b} overlap or precede the span before "
                                     f"it, which ends at {unit} {prev}")
            prev = b
            ms = _target_ms(ms, label, k)
            asks |= not math.isnan(ms)
            out.append((a, b, ms))
    if asks and tempo is not None and not math.isnan(float(tempo)):
        raise OperationError(f"{_who(label)}: a target duration and a tempo ratio together (give one or the other)")
    return out


def _char_targets_to_ids(entry, phonemes: str, src: Sequence[int], label):
    """A checked phoneme-surface target entry (of _target_entry) as id spans: a span of characters [a, b] covers the
    ids whose source character lies in it (its ids and pads, as pitch contours map characters); one that covers no id
    is refused.  A whole-utterance duration stays one."""
    if entry is None or isinstance(entry, float):
        return entry
    out = []
    for k, (a, b, ms) in enumerate(entry):
        if b >= len(phonemes):
            raise OperationError(f"{_who(label)}, span {k}: characters {a} .. {b} are not a range of the "
                                 f"{len(phonemes)} characters")
        ids = [i for i, c in enumerate(src) if a <= int(c) <= b]
        if not ids:
            raise OperationError(f"{_who(label)}, span {k}: characters {a} .. {b} map to no id (the voice drops them)")
        out.append((ids[0], ids[-1], ms))
    return out


def _target_arrays(lens: Sequence[int], entries):
    """The C target table (first i64, end i64, ms f32, offsets size_t [n + 1]) of checked per-utterance entries (of
    _target_entry, in ids; a whole-utterance duration is the span of every id), or None when no span asks."""
    if entries is None:
        return None
    first, end, ms, offs = [], [], [], [0]
    for n_ids, e in zip(lens, entries):
        spans = [] if e is None else [(0, n_ids - 1, e)] if isinstance(e, float) else e
        for a, b, m in spans:
            first.append(a); end.append(b + 1); ms.append(m)
        offs.append(len(first))
    if all(math.isnan(m) for m in ms):
        return None
    return (np.array(first, np.int64), np.array(end, np.int64), np.array(ms, np.float32),
            np.array(offs, np.uint64))


def _target_images(t):
    """The four C pointers of a target table of _target_arrays (all None for none)."""
    if t is None:
        return None, None, None, None
    return _ptr(t[0], C.c_int64), _ptr(t[1], C.c_int64), _ptr(t[2], C.c_float), _ptr(t[3], C.c_size_t)


def _check_target_list(targets, n: int, tempo, lens: Optional[Sequence[int]]):
    """Each utterance's entry of `targets` (one per utterance, or None) checked by _target_entry; None when not given."""
    if targets is None:
        return None
    return [_target_entry(v, b, None if tempo is None else tempo[b], None if lens is None else lens[b],
                          "id" if lens is not None else "character")
            for b, v in enumerate(_per_utterance(targets, n, "target durations"))]


def refuse_prosody(pitch, tempo, where: str) -> None:
    """OperationError when `where`, a mode that hands out a sentence chunk by chunk, is asked for a pitch or tempo
    ratio."""
    if any(a is not None for a in _prosody_arrays([pitch], [tempo], 1)):
        raise OperationError(f"{where} cannot shift pitch or tempo: the time stretch walks a whole sentence frame by "
                             "frame, and this mode hands out a sentence's first chunk before its last one is decoded "
                             "(use the lazy, parallel or file modes, speak_batch or a SynthesisJob)")


def refuse_volume(volume_contour, where: str) -> None:
    """OperationError when `where`, a mode without this library's streaming voices, is asked for a volume contour."""
    if volume_contour is not None:
        raise OperationError(f"{where} cannot apply a volume contour: only this library's streaming voices carry a "
                             "contour from chunk to chunk (use speak_batch or a SynthesisJob)")


def refuse_breaks(breaks, where: str) -> None:
    """OperationError when `where`, a mode without this library's streaming voices, is asked for breaks."""
    if breaks is not None:
        raise OperationError(f"{where} cannot insert breaks: only this library's streaming voices carry them from chunk "
                             "to chunk (use speak_batch or a SynthesisJob)")


def refuse_targets(target_duration, where: str) -> None:
    """OperationError when `where`, a mode without this library's streaming voices, is asked for a target duration."""
    if target_duration is not None:
        raise OperationError(f"{where} cannot fit a target duration: only this library's streaming voices fit a "
                             "sentence's latent (use speak_batch or a SynthesisJob)")


def refuse_contour(pitch_contour, where: str) -> None:
    """OperationError when `where`, a mode without this library's streaming voices, is asked for a pitch contour."""
    if pitch_contour is not None:
        raise OperationError(f"{where} cannot apply a pitch contour: only this library's streaming voices carry a "
                             "contour from chunk to chunk (use speak_batch_with_alignment or a SynthesisJob)")


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


@dataclass
class _BatchOptions:
    """A batch's options, checked once by _batch_options, as the C images the library takes: each None when not given
    or when no utterance asks for it.  A phoneme surface's per-character controls (char_scales, char_contours,
    char_volumes, char_breaks: one entry or None per utterance) become the per-id images `scales`, `contour`, `volume`
    and `breaks` once its phonemes are mapped (map_characters)."""
    n: int
    cfgs: object = None                       # sb200_synth_config [n]
    scales: Optional[np.ndarray] = None       # per id, packed
    frames: Optional[np.ndarray] = None       # per id, packed
    seeds: Optional[np.ndarray] = None
    seeded: Optional[np.ndarray] = None
    rates: Optional[np.ndarray] = None
    loudness: Optional[np.ndarray] = None
    laws: Optional[list] = None               # G.711 surfaces only
    gains: Optional[np.ndarray] = None
    pitch: Optional[np.ndarray] = None
    tempo: Optional[np.ndarray] = None
    contour: Optional[np.ndarray] = None      # per id, packed
    formants: Optional[np.ndarray] = None
    blend_speakers: Optional[np.ndarray] = None
    blend_weights: Optional[np.ndarray] = None
    blend_offsets: Optional[np.ndarray] = None
    volume: Optional[np.ndarray] = None       # per id, packed
    breaks: Optional[np.ndarray] = None       # per id, packed
    targets: Optional[tuple] = None           # target table (_target_arrays)
    char_scales: Optional[list] = None
    char_contours: Optional[list] = None
    char_volumes: Optional[list] = None
    char_breaks: Optional[list] = None
    char_targets: Optional[list] = None       # checked entries in characters (_target_entry)

    def map_characters(self, phonemes: Sequence[str], maps) -> None:
        """Makes the per-id images of the per-character controls once the phonemes are mapped: maps[b] is (ids, source
        character of each id) of phonemes[b], as phonemes_to_input_ids_map gives it."""
        def per_id(values, what, check, none=1.0):
            return None if values is None else [
                None if v is None else _char_values_to_ids(v, ph, src, b, what, check, none)
                for b, (v, ph, (_, src)) in enumerate(zip(values, phonemes, maps))]
        lens = [len(ids) for ids, _ in maps]
        self.scales, _ = _duration_arrays(lens, per_id(self.char_scales, "duration scales", _scale_value))
        self.contour = _contour_arrays(lens, per_id(self.char_contours, "pitch ratios", _contour_value), self.pitch)
        self.volume = _volume_arrays(lens, per_id(self.char_volumes, "volume levels", _volume_value, 0.0))
        self.breaks = None if self.char_breaks is None else _break_arrays(lens, [
            None if v is None else _char_breaks_to_ids(v, ph, src, b)
            for b, (v, ph, (_, src)) in enumerate(zip(self.char_breaks, phonemes, maps))])
        if self.char_targets is not None:
            self.targets = _target_arrays(lens, [_char_targets_to_ids(e, ph, src, b) for b, (e, ph, (_, src)) in
                                                 enumerate(zip(self.char_targets, phonemes, maps))])

    @property
    def per_character(self) -> bool:
        """Whether a per-character control needs the phonemes' character map."""
        return any(x is not None for x in (self.char_scales, self.char_contours, self.char_volumes, self.char_breaks,
                                           self.char_targets))


def _batch_options(model, n: int, lens: Optional[Sequence[int]] = None, configs=None, duration_scales=None,
                   durations=None, seeds=None, output_rates=None, loudness=None, law=None, gains=None, pitches=None,
                   tempos=None, pitch_contours=None, formants=None, speaker_blends=None, volume_contours=None,
                   breaks=None, g711: bool = False, target_durations=None) -> _BatchOptions:
    """The options of a batch of n utterances, each checked as its C image is made, in one order at every surface:
    configs, duration scales, durations, seeds, output rates, loudness, law (with `g711`), gains, pitch and tempo, pitch
    contours, formants, speaker blends, volume contours, breaks, target durations.  `lens`: the utterances' id counts, for per-id controls; None for a phoneme
    surface, whose per-character controls are only counted here, before any phoneme is mapped (see map_characters)."""
    o = _BatchOptions(n, _config_array(configs, n))
    if lens is None:
        o.char_scales = None if duration_scales is None else _per_utterance(duration_scales, n, "duration scales")
    else:
        o.scales, o.frames = _duration_arrays(lens, duration_scales, durations)
    o.seeds, o.seeded = _seed_arrays(seeds, n)
    o.rates = _rate_array(output_rates, n)
    o.loudness = _loudness_array(loudness, n)
    if g711:
        o.laws = _encoding_list(law, n)
    o.gains = _gain_array(gains, n)
    o.pitch, o.tempo = _prosody_arrays(pitches, tempos, n)
    if lens is None:
        o.char_contours = None if pitch_contours is None else _per_utterance(pitch_contours, n, "pitch contours")
    else:
        o.contour = _contour_arrays(lens, pitch_contours, o.pitch)
    o.formants = _formant_array(formants, n)
    o.blend_speakers, o.blend_weights, o.blend_offsets = _blend_arrays(model, speaker_blends, n)
    if lens is None:
        o.char_volumes = None if volume_contours is None else _per_utterance(volume_contours, n, "volume contours")
    else:
        o.volume = _volume_arrays(lens, volume_contours)
    if lens is None:
        o.char_breaks = None if breaks is None else _per_utterance(breaks, n, "breaks")
    else:
        o.breaks = _break_arrays(lens, breaks)
    checked = _check_target_list(target_durations, n, o.tempo, lens)
    if lens is None:
        o.char_targets = checked
    else:
        o.targets = _target_arrays(lens, checked)
    return o


def _pack_ids(batches):
    """The ids of a batch back to back (int64) and each utterance's offset into them (size_t [n + 1])."""
    packed = np.ascontiguousarray(np.concatenate([np.asarray(b, dtype=np.int64) for b in batches]))
    offs = np.zeros(len(batches) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(b) for b in batches])
    return packed, offs


def _check_not_empty(batches) -> None:
    if any(len(b) == 0 for b in batches):
        raise OperationError("Failed to run model inference. Error: empty input sequence")


def rate_ratio(in_rate: int, out_rate: Optional[int]) -> Tuple[int, int]:
    """(up, down): out_rate / in_rate reduced, (1, 1) for no resampling (None, 0 or the same rate)."""
    if not out_rate or int(out_rate) == int(in_rate):
        return 1, 1
    g = math.gcd(int(in_rate), int(out_rate))
    return int(out_rate) // g, int(in_rate) // g


def _ptr(a, ctype):
    return None if a is None else a.ctypes.data_as(C.POINTER(ctype))


def _alignment(phonemes: str, src_char: Sequence[int], frames: Sequence[int], n_samples: int,
               up: int = 1, down: int = 1, warped: bool = False,
               bounds: Optional[Sequence[int]] = None) -> List[PhonemeAlignment]:
    """Groups per-id frame counts by the character each id came from: bos (`^`), one entry per kept character (its id
    and its pad) and eos (`$`), contiguous from sample 0.  An utterance whose ids all got 0 frames is still one frame
    long; that frame (after every id) goes to the last entry, so the entries always end at n_samples.  Audio resampled
    by up/down puts the boundary after F frames at ceil(F * hop * up / down).  `warped` (a pitch or tempo ratio changed
    the length): the boundary after F of the utterance's T frames is at floor(F * n_samples / T + 0.5), whatever the
    output rate; the time stretch moves a sample by at most D = rate // 160 input samples from that linear map, so a
    boundary is accurate to within D / tempo samples of the warped signal.  `bounds` (a pitch contour): each id's
    delivered end at the voice's rate (sb200_speak_batch_ids_contour); an entry ends where its last id does, at
    ceil(end * up / down)."""
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
        end = at(fsum) if bounds is None else -((-int(bounds[j - 1]) * up) // down)
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

    def set_watermark(self, key, payload: int = 0, strength_db: float = -26.0):
        """Mark everything this voice delivers from now on with key's watermark carrying `payload` (include/sonata_b200.h,
        sb200_voice_set_watermark): every job and batch route, at each utterance's delivered rate.  key None turns it
        off.  A realtime stream reads the setting when it is made and keeps it to its end.  Bad values raise
        OperationError and leave the voice as it was."""
        err = N.sb200_error()
        if key is None:
            _check(self._lib.sb200_voice_set_watermark(self._h, None, C.byref(err)), err)
            return
        k, p, s = check_watermark(key, payload, strength_db)
        wm = N.sb200_watermark(k, p, s)
        _check(self._lib.sb200_voice_set_watermark(self._h, C.byref(wm), C.byref(err)), err)

    def watermark(self) -> Optional[Tuple[int, int, float]]:
        """(key, payload, strength_db) of the voice's watermark, or None when it marks nothing."""
        wm, on, err = N.sb200_watermark(), C.c_int32(), N.sb200_error()
        _check(self._lib.sb200_voice_watermark(self._h, C.byref(wm), C.byref(on), C.byref(err)), err)
        return (int(wm.key), int(wm.payload), float(wm.strength_db)) if on.value else None

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
                    pitches: Optional[Sequence] = None, tempos: Optional[Sequence] = None,
                    pitch_contours: Optional[Sequence] = None, formants: Optional[Sequence] = None,
                    speaker_blends: Optional[Sequence] = None,
                    volume_contours: Optional[Sequence] = None, breaks: Optional[Sequence] = None,
                    target_durations: Optional[Sequence] = None) -> List[Audio]:
        """`configs`: one PiperSynthesisConfig per utterance (speaker and scales), still synthesised as one pass;
        None uses the fallback config for every utterance.  `seeds`: noise seeds as for infer_batch_with_values.
        `speaker_blends`: as for infer_batch_with_values.
        `output_rates` / `loudness` / `pitches` / `tempos` / `formants`: per-utterance output sample rates, loudness
        targets, pitch and tempo ratios and formant ratios as for infer_batch_with_values.  `pitch_contours` /
        `volume_contours` / `breaks`: as for speak_batch_with_alignment, one ratio, level or break per phoneme
        character.  `target_durations`: as for speak_batch_with_alignment, spans in phoneme characters."""
        n = len(phoneme_batches)
        o = _batch_options(self, n, None, configs, seeds=seeds, output_rates=output_rates, loudness=loudness,
                           pitches=pitches, tempos=tempos, pitch_contours=pitch_contours, formants=formants,
                           speaker_blends=speaker_blends, volume_contours=volume_contours, breaks=breaks,
                           target_durations=target_durations)
        if n == 0:
            return []
        if o.per_character:
            maps = [self.phonemes_to_input_ids_map(p) for p in phoneme_batches]
            o.map_characters(phoneme_batches, maps)
            return [a for a, _, _ in self._speak_ids([ids for ids, _ in maps], o)]
        if any(x is not None for x in (o.cfgs, o.seeds, o.rates, o.loudness, o.pitch, o.tempo, o.formants,
                                       o.blend_offsets)):
            return [a for a, _, _ in self._speak_ids([self.phonemes_to_input_ids(p) for p in phoneme_batches], o)]
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
                                tempos: Optional[Sequence] = None,
                                pitch_contours: Optional[Sequence] = None,
                                formants: Optional[Sequence] = None,
                                speaker_blends: Optional[Sequence] = None,
                                volume_contours: Optional[Sequence] = None,
                                breaks: Optional[Sequence] = None,
                                target_durations: Optional[Sequence] = None) -> List[Audio]:
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
        leaves the utterance's samples as they are, bit for bit.

        `pitch_contours`: one pitch ratio per id for each utterance (in PITCH_RANGE, or None / NaN / 1.0 for none), or
        None.  Each id's samples are shifted by its own ratio and the id keeps its duration (divided by the utterance's
        tempo, which a contour combines with; an utterance's pitch ratio does not).  A contour whose ratio is the same
        on every id gives the bits of that pitch ratio (sb200_speak_batch_ids_contour).

        `formants`: one formant ratio per utterance (in FORMANT_RANGE, or None / NaN for none), or None.  The delivered
        audio gets the voice's own spectral envelope with every frequency multiplied by the ratio, on the device after
        the pitch stage (sb200_speak_batch_ids_formants): 1.0 with a pitch ratio or contour keeps the formants where
        they were, so the voice sounds like the same speaker at another pitch (unlike the other ratios, an explicit 1.0
        asks for something there), and a ratio without a pitch moves them at the same pitch and duration.  Lengths and
        alignments do not change.

        `speaker_blends`: one blend or None per utterance, or None.  A blend is a mapping {speaker: weight} of a
        multi-speaker voice: keys are speaker ids or names of its speaker_id_map, weights finite and >= 0, not all zero.
        The utterance speaks with the weighted mean of those speakers' embeddings, which replaces its config's speaker
        (the config's scales still apply; include/sonata_b200.h, sb200_speak_batch_ids_blends).  A blend of one speaker
        (any positive weight) gives that speaker's bits, and blends equal up to order, zero weights or a common
        power-of-two scale give the same bits.

        `volume_contours`: one volume level in dB per id for each utterance (in VOLUME_RANGE, -inf to mute, or None /
        NaN / 0 for none), or None: SSML's <prosody volume> on a span.  Each id's delivered samples are scaled by its
        level, with a 10 ms smoothstep between levels, on the device after the formant stage and before any resampling
        and loudness (sb200_speak_batch_ids_volume); a loudness target then normalises the utterance as a whole, so the
        relative levels survive.  Lengths and alignments do not change, and there is no clamp.

        `breaks`: one pause in ms per id for each utterance, inserted after that id (in BREAK_RANGE_MS, or None / NaN
        / 0 for none), or None: SSML's <break time>.  Each pause is round(ms * rate / 1000) samples of silence at the
        voice's rate, with a 5 ms smoothstep fade of the speech on either side, inserted on the device after the
        volume stage and before any resampling and loudness (sb200_speak_batch_ids_breaks); a loudness target then
        normalises the paused utterance as a whole.  The utterance gets longer by its pauses.

        `target_durations`: one entry per utterance, or None: None, a duration in ms for the whole utterance (bos and
        eos included), or a list of (first, last, ms) spans of ids, inclusive, ascending and disjoint; ms in
        TARGET_RANGE_MS, or None / NaN for none.  Each span's predicted durations are multiplied by one factor u in
        [0.5, 2] before their ceil, the largest whose frames (times 256, plus the span's breaks) do not pass the target
        (u = 0.5 when even that overruns), found on the device in the same pass (include/sonata_b200.h,
        sb200_speak_batch_ids_fit).  Ids outside the spans and fixed durations keep their counts, and the rest of the
        pass runs as with those counts fixed.  A target may not go with a tempo ratio.  SynthesisJob.targets()
        reports each span's u and delivered length."""
        o = _batch_options(self, len(batches), [len(b) for b in batches], configs, seeds=seeds,
                           output_rates=output_rates, loudness=loudness, pitches=pitches, tempos=tempos,
                           pitch_contours=pitch_contours, formants=formants, speaker_blends=speaker_blends,
                           volume_contours=volume_contours, breaks=breaks, target_durations=target_durations)
        return [a for a, _, _ in self._speak_ids(batches, o)]

    def infer_batch_with_durations(self, batches: Sequence[Sequence[int]],
                                   configs: Optional[Sequence[PiperSynthesisConfig]] = None,
                                   duration_scales: Optional[Sequence] = None,
                                   durations: Optional[Sequence] = None,
                                   seeds: Optional[Sequence] = None,
                                   output_rates: Optional[Sequence] = None,
                                   loudness: Optional[Sequence] = None, pitches: Optional[Sequence] = None,
                                   tempos: Optional[Sequence] = None,
                                   pitch_contours: Optional[Sequence] = None,
                                   formants: Optional[Sequence] = None,
                                   speaker_blends: Optional[Sequence] = None,
                                   volume_contours: Optional[Sequence] = None,
                                   breaks: Optional[Sequence] = None,
                                   target_durations: Optional[Sequence] = None) -> List[Tuple[Audio, np.ndarray]]:
        """infer_batch_with_values with per-id duration control, returning (audio, frames per id) per utterance.

        duration_scales[b]: one scale (finite, >= 0) per id of utterance b, applied before the duration's ceil, so 1.0
        gives the plain result bit for bit; durations[b]: one frame count per id, -1 for "predicted" or >= 0 to fix it.
        Either list, or any of its entries, may be None.  The frame counts times 256 are each id's samples; an
        utterance whose ids all got 0 frames is still one frame long.  `seeds`: as for infer_batch_with_values; a
        seeded frame's noise depends on its index only, so controls that move frames never reshuffle it.
        `output_rates` / `loudness` / `pitches` / `tempos` / `pitch_contours` / `formants` / `speaker_blends` /
        `volume_contours` / `breaks` / `target_durations`: as for infer_batch_with_values (the frame counts stay
        frame counts of the utterance before any warp or pause, and are the fitted ones with a target)."""
        o = _batch_options(self, len(batches), [len(b) for b in batches], configs, duration_scales, durations, seeds,
                           output_rates, loudness, pitches=pitches, tempos=tempos, pitch_contours=pitch_contours,
                           formants=formants, speaker_blends=speaker_blends, volume_contours=volume_contours,
                           breaks=breaks, target_durations=target_durations)
        return [(a, f) for a, f, _ in self._speak_ids(batches, o, frames=True)]

    def _speak_ids(self, batches, o: _BatchOptions, frames: bool = False) -> List[tuple]:
        """The f32 batch route: `batches` with options `o` in one sb200_speak_batch_ids_fit call.  Per utterance
        (audio, frames per id, each id's delivered end): the frames only when asked for, since fetching them costs a
        device->host copy and a synchronise, and the ends only when o has a pitch contour or breaks (None
        otherwise)."""
        n = len(batches)
        if n == 0:
            return []
        _check_not_empty(batches)
        packed, offs = _pack_ids(batches)
        outs = (N.sb200_audio * n)()
        id_frames = np.zeros(int(offs[-1]), np.int32) if frames else None
        bounds = None if o.contour is None and o.breaks is None else np.zeros(int(offs[-1]), np.int64)
        err = N.sb200_error()
        _check(self._lib.sb200_speak_batch_ids_fit(
            self._h, _ptr(packed, C.c_int64), _ptr(offs, C.c_size_t), n, o.cfgs, _ptr(o.scales, C.c_float),
            _ptr(o.frames, C.c_int32), _ptr(o.seeds, C.c_uint64), _ptr(o.seeded, C.c_int32), _ptr(o.rates, C.c_uint32),
            _ptr(o.loudness, C.c_float), _ptr(o.pitch, C.c_float), _ptr(o.tempo, C.c_float), _ptr(o.contour, C.c_float),
            _ptr(o.formants, C.c_float), _ptr(o.blend_speakers, C.c_int64), _ptr(o.blend_weights, C.c_float),
            _ptr(o.blend_offsets, C.c_size_t), _ptr(o.volume, C.c_float), _ptr(o.breaks, C.c_float),
            *_target_images(o.targets), outs, _ptr(id_frames, C.c_int32), _ptr(bounds, C.c_int64), None, None, None,
            None, C.byref(err)), err)
        cut = lambda a, b: None if a is None else a[int(offs[b]):int(offs[b + 1])].copy()
        return [(_take_audio(outs[b]), cut(id_frames, b), cut(bounds, b)) for b in range(n)]

    def speak_batch_with_alignment(self, phoneme_batches: Sequence[str],
                                   configs: Optional[Sequence[PiperSynthesisConfig]] = None,
                                   duration_scales: Optional[Sequence] = None,
                                   seeds: Optional[Sequence] = None,
                                   output_rates: Optional[Sequence] = None,
                                   loudness: Optional[Sequence] = None, pitches: Optional[Sequence] = None,
                                   tempos: Optional[Sequence] = None, pitch_contours: Optional[Sequence] = None,
                                   formants: Optional[Sequence] = None,
                                   speaker_blends: Optional[Sequence] = None,
                                   volume_contours: Optional[Sequence] = None,
                                   breaks: Optional[Sequence] = None,
                                   target_durations: Optional[Sequence] = None
                                   ) -> List[Tuple[Audio, List[PhonemeAlignment]]]:
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
        the warped signal because the time stretch takes each frame from within that many samples of the linear map.

        pitch_contours[b] (or None): one pitch ratio per character of phoneme_batches[b] (in PITCH_RANGE, or None / NaN
        / 1.0 for none), applied to that character's id and pad, bos and eos keeping their pitch; see
        infer_batch_with_values.  An utterance with a contour is aligned from each id's delivered end
        (sb200_speak_batch_ids_contour), exact rather than scaled: with no tempo a boundary stays where it was.
        `formants`: as for infer_batch_with_values; it moves no boundary.  `speaker_blends`: as for
        infer_batch_with_values.  volume_contours[b] (or None): one volume level per character of phoneme_batches[b]
        (see infer_batch_with_values), applied to that character's id and pad, bos and eos keeping their level; it
        moves no boundary.  breaks[b] (or None): one pause in ms per character of phoneme_batches[b] (see
        infer_batch_with_values), after that character's pad; a character the voice drops puts its pause after the
        last id before it.  An utterance with breaks is aligned from each id's delivered end after the pauses before
        it, so a pause belongs to the entry it follows and the entries still end at len(audio).
        target_durations[b] (or None): as for infer_batch_with_values, with spans (first, last, ms) of phoneme
        characters, inclusive: a span covers the ids (and pads) of the characters in it, and one whose characters the
        voice all drops is refused.  The alignment then holds the fitted durations."""
        n = len(phoneme_batches)
        o = _batch_options(self, n, None, configs, duration_scales, seeds=seeds, output_rates=output_rates,
                           loudness=loudness, pitches=pitches, tempos=tempos, pitch_contours=pitch_contours,
                           formants=formants, speaker_blends=speaker_blends, volume_contours=volume_contours,
                           breaks=breaks, target_durations=target_durations)
        maps = [self.phonemes_to_input_ids_map(p) for p in phoneme_batches]
        o.map_characters(phoneme_batches, maps)
        res = self._speak_ids([ids for ids, _ in maps], o, frames=True)
        voice_rate = self.audio_output_info().sample_rate if o.rates is not None else None
        ratio = lambda audio: (1, 1) if voice_rate is None else rate_ratio(voice_rate, audio.info.sample_rate)
        warped = lambda b: any(r is not None and not np.isnan(r[b]) for r in (o.pitch, o.tempo))
        offs = np.cumsum([0] + [len(ids) for ids, _ in maps])

        def shaped(b):          # utterance b has a contour or breaks that ask: aligned from its delivered ends
            c = None if o.contour is None else o.contour[offs[b]:offs[b + 1]]
            k = None if o.breaks is None else o.breaks[offs[b]:offs[b + 1]]
            return ((c is not None and bool(np.any(~np.isnan(c) & (c != 1)))) or
                    (k is not None and bool(np.any(~np.isnan(k) & (k != 0)))))
        return [(audio, _alignment(ph, src, frames, len(audio), *ratio(audio), warped=warped(b),
                                   bounds=bounds if shaped(b) else None))
                for b, (ph, (_, src), (audio, frames, bounds)) in enumerate(zip(phoneme_batches, maps, res))]

    def infer_batch_g711(self, batches: Sequence[Sequence[int]], law,
                         configs: Optional[Sequence[PiperSynthesisConfig]] = None, seeds: Optional[Sequence] = None,
                         output_rates: Optional[Sequence] = None, loudness: Optional[Sequence] = None,
                         gains: Optional[Sequence] = None, pitches: Optional[Sequence] = None,
                         tempos: Optional[Sequence] = None, formants: Optional[Sequence] = None,
                         speaker_blends: Optional[Sequence] = None, breaks: Optional[Sequence] = None,
                         target_durations: Optional[Sequence] = None) -> List[bytes]:
        """infer_batch_with_values delivered as G.711 telephony audio: one `bytes` per utterance, one byte per sample.
        `law`: "mulaw" (PCMU) or "alaw" (PCMA), or one of those per utterance.  The bytes are G.711 of exactly the
        16-bit samples the i16 route gives (SynthesisJob.fetch_i16): to_i16_vec of the utterance after gains[b] (None:
        1), or the fixed scale for an utterance with a loudness target.  They are encoded on the device in the i16
        conversion's launches, so only one byte per sample leaves the card.  `configs`, `seeds`, `output_rates` and
        `loudness` as for infer_batch_with_values, and so are `pitches`, `tempos`, `formants`, `speaker_blends`,
        `breaks` and `target_durations`; a batch mixing laws runs one conversion per law."""
        o = _batch_options(self, len(batches), [len(b) for b in batches], configs, seeds=seeds,
                           output_rates=output_rates, loudness=loudness, law=law, gains=gains, pitches=pitches,
                           tempos=tempos, formants=formants, speaker_blends=speaker_blends, breaks=breaks, g711=True,
                           target_durations=target_durations)
        return self._encode_batch(batches, o)

    def speak_batch_g711(self, phoneme_batches: Sequence[str], law,
                         configs: Optional[Sequence[PiperSynthesisConfig]] = None, seeds: Optional[Sequence] = None,
                         output_rates: Optional[Sequence] = None, loudness: Optional[Sequence] = None,
                         gains: Optional[Sequence] = None, pitches: Optional[Sequence] = None,
                         tempos: Optional[Sequence] = None, formants: Optional[Sequence] = None,
                         speaker_blends: Optional[Sequence] = None, breaks: Optional[Sequence] = None,
                         target_durations: Optional[Sequence] = None) -> List[bytes]:
        """speak_batch delivered as G.711 bytes: infer_batch_g711 over the phonemes' ids (`breaks`: one per phoneme
        character, and `target_durations` in characters, as for speak_batch_with_alignment)."""
        o = _batch_options(self, len(phoneme_batches), None, configs, seeds=seeds, output_rates=output_rates,
                           loudness=loudness, law=law, gains=gains, pitches=pitches, tempos=tempos, formants=formants,
                           speaker_blends=speaker_blends, breaks=breaks, g711=True,
                           target_durations=target_durations)
        return self._encode_batch(self._phoneme_ids(phoneme_batches, o), o)

    def infer_batch_flac(self, batches: Sequence[Sequence[int]],
                         configs: Optional[Sequence[PiperSynthesisConfig]] = None, seeds: Optional[Sequence] = None,
                         output_rates: Optional[Sequence] = None, loudness: Optional[Sequence] = None,
                         gains: Optional[Sequence] = None, pitches: Optional[Sequence] = None,
                         tempos: Optional[Sequence] = None, formants: Optional[Sequence] = None,
                         speaker_blends: Optional[Sequence] = None, breaks: Optional[Sequence] = None,
                         target_durations: Optional[Sequence] = None) -> List[bytes]:
        """infer_batch_with_values delivered as lossless FLAC: one complete stream (`bytes`) per utterance.  Its samples
        are exactly the 16-bit samples the i16 route gives (SynthesisJob.fetch_i16): to_i16_vec of the utterance after
        gains[b] (None: 1), or the fixed scale for an utterance with a loudness target, at its delivered rate.  They are
        encoded on the device, and only the compressed bytes leave the card.  `configs`, `seeds`, `output_rates`,
        `loudness`, `pitches`, `tempos`, `formants`, `speaker_blends`, `breaks` and `target_durations` as for
        infer_batch_with_values."""
        o = _batch_options(self, len(batches), [len(b) for b in batches], configs, seeds=seeds,
                           output_rates=output_rates, loudness=loudness, gains=gains, pitches=pitches, tempos=tempos,
                           formants=formants, speaker_blends=speaker_blends, breaks=breaks,
                           target_durations=target_durations)
        return self._encode_batch(batches, o)

    def speak_batch_flac(self, phoneme_batches: Sequence[str],
                         configs: Optional[Sequence[PiperSynthesisConfig]] = None, seeds: Optional[Sequence] = None,
                         output_rates: Optional[Sequence] = None, loudness: Optional[Sequence] = None,
                         gains: Optional[Sequence] = None, pitches: Optional[Sequence] = None,
                         tempos: Optional[Sequence] = None, formants: Optional[Sequence] = None,
                         speaker_blends: Optional[Sequence] = None, breaks: Optional[Sequence] = None,
                         target_durations: Optional[Sequence] = None) -> List[bytes]:
        """speak_batch delivered as FLAC streams: infer_batch_flac over the phonemes' ids (`breaks`: one per phoneme
        character, and `target_durations` in characters, as for speak_batch_with_alignment)."""
        o = _batch_options(self, len(phoneme_batches), None, configs, seeds=seeds, output_rates=output_rates,
                           loudness=loudness, gains=gains, pitches=pitches, tempos=tempos, formants=formants,
                           speaker_blends=speaker_blends, breaks=breaks,
                           target_durations=target_durations)
        return self._encode_batch(self._phoneme_ids(phoneme_batches, o), o)

    def _phoneme_ids(self, phoneme_batches: Sequence[str], o: _BatchOptions) -> list:
        """The ids of each phoneme string; with per-character controls in `o`, mapped so o gets their per-id images."""
        if not o.per_character:
            return [self.phonemes_to_input_ids(p) for p in phoneme_batches]
        maps = [self.phonemes_to_input_ids_map(p) for p in phoneme_batches]
        o.map_characters(phoneme_batches, maps)
        return [ids for ids, _ in maps]

    def _encode_batch(self, batches, o: _BatchOptions) -> List[bytes]:
        """The G.711 bytes (when o has laws) or FLAC streams of `batches` with options `o`: one SynthesisJob run, then
        one fetch per law."""
        from .job import SynthesisJob
        if o.n == 0:
            return []
        _check_not_empty(batches)
        job = SynthesisJob._of(self, batches, o)
        try:
            job.run()
            g = _ptr(o.gains, C.c_float)
            if o.laws is None:
                return job._fetch_bytes(self._lib.sb200_job_fetch_flac, g)
            out: List[Optional[bytes]] = [None] * o.n
            for e in dict.fromkeys(o.laws):
                res = job._fetch_bytes(self._lib.sb200_job_fetch_g711, G711_LAW[e], g)
                for b in range(o.n):
                    if o.laws[b] == e:
                        out[b] = res[b]
            return out
        finally:
            job.close()

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
        self.fit: Optional[List[Tuple[float, int]]] = None     # per target span: (u, delivered length) of the fit

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


def _handles(objs, n: int, kind, what: str):
    """The C handles of one `kind` (Resampler, ProsodyStream or LoudnessStream) or None per chunk of a decoder pass."""
    out = (C.c_void_p * n)()
    for k, x in enumerate(_per_utterance(objs, n, what)):
        if x is not None and (not isinstance(x, kind) or not x._h):
            raise OperationError(f"chunk {k}: not a {kind.__name__}")
        out[k] = None if x is None else x._h.value
    return out


def _stream_resampler(model, output_rate) -> Optional[Resampler]:
    """A Resampler for a stream at output_rate, or None when the stream stays at the voice's rate."""
    _rate_array([output_rate], 1)
    if not output_rate or int(output_rate) == model.audio_output_info().sample_rate:
        return None
    return Resampler(model, output_rate)


class ProsodyStream:
    """One stream's pitch and tempo state on the device (sb200_prosody_stream_*): it carries the tails of the stream's
    input and stretched signal, and its last frames' offsets, between chunks, so the concatenation of what it emits is
    the whole stream warped at once.  `pitch` / `tempo`: ratios as for infer_batch_with_values, not both neutral.

    `pitch_contour`: one pitch ratio per id of `enc` (the EncoderOutputs of the sentence the stream carries; values as
    for infer_batch_with_values' pitch_contours), instead of `pitch` (sb200_prosody_stream_create_contour).  Its plan is
    fixed by enc's frames, so the stream must be fed exactly enc's chunks; `bounds` then holds each id's delivered end
    at the voice's rate (None without a contour).

    `formant`: a formant ratio as for infer_batch_with_values' formants (None / NaN: none), applied on top of the
    ratios or contour, or alone when they ask for nothing (sb200_prosody_stream_create_formant): the concatenation of
    what the stream emits is the formant stage of the sentence it warps, applied at once.  Its stage holds back 768 -
    1023 samples more than the warp alone.

    `volume`: one volume level in dB per id of `enc` (values as for infer_batch_with_values' volume_contours), applied
    on top of the rest, or alone when it asks for nothing (sb200_prosody_stream_create_volume): each sample the stream
    emits is scaled at its delivered position, holding nothing back.

    `breaks`: one pause in ms per id of `enc` (values as for infer_batch_with_values' breaks), inserted after that id,
    on top of the rest or alone (sb200_prosody_stream_create_breaks): each chunk emits the pauses its input reaches,
    holding nothing back, and `bounds` then holds each id's delivered end after the pauses before it.  The stream must
    be fed exactly enc's chunks."""

    def __init__(self, model: "_VitsCommons", pitch=None, tempo=None, pitch_contour=None,
                 enc: Optional["EncoderOutputs"] = None, formant=None, volume=None, breaks=None):
        p, t = _prosody_arrays([pitch], [tempo], 1)
        phi = _stream_formant(formant, "stream")
        vol = None                      # the volume contour's per-id image
        if volume is not None:
            if not isinstance(enc, EncoderOutputs) or enc._m is not model or not enc._h:
                raise OperationError("a volume contour needs the EncoderOutputs of its sentence, from this model")
            vol = _volume_arrays([len(enc.p_duration)], [volume], ["stream"])
        bk = None                       # the breaks' per-id image
        if breaks is not None:
            if not isinstance(enc, EncoderOutputs) or enc._m is not model or not enc._h:
                raise OperationError("breaks need the EncoderOutputs of their sentence, from this model")
            bk = _break_arrays([len(enc.p_duration)], [breaks], ["stream"])
        self._m, self._h = model, C.c_void_p()
        self.pitch = None if p is None else float(p[0])
        self.tempo = None if t is None else float(t[0])
        self.formant = phi
        self.bounds = None
        c = None                        # the contour's per-id image
        if pitch_contour is not None:
            if phi is None and p is not None:
                raise OperationError("stream: a pitch contour and a pitch ratio together (give one or the other)")
            if not isinstance(enc, EncoderOutputs) or enc._m is not model or not enc._h:
                raise OperationError("a pitch contour needs the EncoderOutputs of its sentence, from this model")
            c = _contour_arrays([len(enc.p_duration)], [pitch_contour], None, ["stream"])
            if c is None:
                c = np.full(len(enc.p_duration), np.nan, np.float32)
        nan = float("nan")
        pv, tv = nan if p is None else float(p[0]), nan if t is None else float(t[0])
        err = N.sb200_error()
        if bk is not None:
            # any of the above with the breaks on top, or the breaks alone
            _check(model._lib.sb200_prosody_stream_create_breaks(
                model._h, enc._h, pv, _ptr(c, C.c_float), bk.size, tv, nan if phi is None else phi,
                _ptr(vol, C.c_float), _ptr(bk, C.c_float), C.byref(self._h), C.byref(err)), err)
        elif vol is not None:
            # any of the above with the volume contour on top, or the contour alone
            _check(model._lib.sb200_prosody_stream_create_volume(
                model._h, enc._h, pv, _ptr(c, C.c_float), vol.size, tv, nan if phi is None else phi,
                _ptr(vol, C.c_float), C.byref(self._h), C.byref(err)), err)
        elif phi is not None:
            # the ratio or contour stream with phi on top, or phi alone
            _check(model._lib.sb200_prosody_stream_create_formant(
                model._h, None if c is None else enc._h, pv, _ptr(c, C.c_float), 0 if c is None else c.size, tv, phi,
                C.byref(self._h), C.byref(err)), err)
        elif c is not None:
            _check(model._lib.sb200_prosody_stream_create_contour(model._h, enc._h, _ptr(c, C.c_float), c.size, tv,
                                                                  C.byref(self._h), C.byref(err)), err)
        elif p is None and t is None:
            raise OperationError("a prosody stream needs a pitch or a tempo ratio other than 1 (None, NaN or 1: none)")
        else:
            _check(model._lib.sb200_prosody_stream_create(model._h, pv, tv, C.byref(self._h), C.byref(err)), err)
        if c is not None or _breaks_ask(bk, model.audio_output_info().sample_rate):
            n_ids = len(enc.p_duration)
            self.bounds = np.zeros(n_ids, np.int64)
            _check(model._lib.sb200_prosody_stream_bounds(self._h, _ptr(self.bounds, C.c_int64), n_ids,
                                                          C.byref(err)), err)

    def last_pass_ms(self) -> Tuple[float, float]:
        """The "stretch" and "pitch" device time (ms) of the last chunk pass this stream was in."""
        s, p = C.c_float(), C.c_float()
        self._m._lib.sb200_prosody_stream_profile(self._h, C.byref(s), C.byref(p))
        return float(s.value), float(p.value)

    def last_formant_ms(self) -> float:
        """The "formant" device time (ms) of the last chunk pass this stream was in (0: its stage did not run)."""
        f = C.c_float()
        self._m._lib.sb200_prosody_stream_profile_formant(self._h, C.byref(f))
        return float(f.value)

    def last_volume_ms(self) -> float:
        """The "volume" device time (ms) of the last chunk pass this stream was in (0: its stage did not run)."""
        f = C.c_float()
        self._m._lib.sb200_prosody_stream_profile_volume(self._h, C.byref(f))
        return float(f.value)

    def last_break_ms(self) -> float:
        """The "break" device time (ms) of the last chunk pass this stream was in (0: its stage did not run)."""
        f = C.c_float()
        self._m._lib.sb200_prosody_stream_profile_breaks(self._h, C.byref(f))
        return float(f.value)

    def __del__(self):
        try:
            if self._h:
                self._m._lib.sb200_prosody_stream_free(self._h)
                self._h = None
        except Exception:
            pass


def _stream_prosody(model, pitch, tempo, pitch_contour=None, enc=None, formant=None,
                    volume=None, breaks=None) -> Optional[ProsodyStream]:
    """A ProsodyStream for a stream with these ratios, or with this per-id contour of enc's sentence and the tempo, and
    the formant ratio, or None when nothing asks for anything.  A given contour makes a contoured stream (which has
    bounds) whenever the contour or the tempo asks for something; a contour of None / NaN / 1 only is no contour beside a
    pitch ratio, as in the batch calls, and with neither a pitch nor a tempo it leaves the plain stream, which has no
    bounds.  A formant ratio asks for something unless it equals the pitch ratio (1 without one): it then makes a
    formant-only stream of a plain one.  A volume contour that asks for something (see _volume_arrays) is carried on
    top of the rest, or alone, and so are breaks of one sample or more (see _breaks_ask)."""
    p, t = _prosody_arrays([pitch], [tempo], 1)
    if breaks is not None and _breaks_ask(_break_arrays([len(enc.p_duration)], [breaks], ["stream"]),
                                          model.audio_output_info().sample_rate):
        if pitch_contour is not None and _contour_arrays([len(enc.p_duration)], [pitch_contour], p, ["stream"]) is None \
                and (p is not None or t is None):
            pitch_contour = None
        return ProsodyStream(model, pitch, tempo, pitch_contour, enc, formant, volume, breaks)
    if volume is not None and _volume_arrays([len(enc.p_duration)], [volume], ["stream"]) is not None:
        if pitch_contour is not None and _contour_arrays([len(enc.p_duration)], [pitch_contour], p, ["stream"]) is None \
                and (p is not None or t is None):
            pitch_contour = None
        return ProsodyStream(model, pitch, tempo, pitch_contour, enc, formant, volume)
    phi = _stream_formant(formant, "stream")
    if pitch_contour is not None:
        asks = _contour_arrays([len(enc.p_duration)], [pitch_contour], p, ["stream"]) is not None
        if asks or (p is None and t is not None):
            return ProsodyStream(model, pitch, tempo, pitch_contour, enc, phi)
    if phi is not None and np.float32(phi) == (np.float32(1.0) if p is None else p[0]):
        phi = None                      # r_m = 1 on every frame: the stage would not run
    if p is None and t is None and phi is None:
        return None
    return ProsodyStream(model, pitch, tempo, formant=phi)


class LoudnessStream:
    """One stream's live loudness meter on the device (sb200_loudness_stream_*): a causal ITU-R BS.1770 meter of
    everything the stream has delivered so far drives a gain ramped across each 100 ms step, so the stream holds
    `target` LUFS (finite, in [-70, 0]) without holding anything back.  `max_gain_db` (finite, in [0, 40]) caps the
    gain; `output_rate` is the rate it meters (None: the voice's).  The first 100 ms play at gain 1, readings before
    400 ms are provisional, and peaks are held by clamping to [-1, 1], not by a look-ahead limiter.  A meter may be
    passed with the chunks of several sentences in turn: their signal just continues.  See include/sonata_b200.h."""

    def __init__(self, model: "_VitsCommons", target, max_gain_db=20.0, output_rate: Optional[int] = None,
                 who: str = "stream"):
        t = _loudness_array([target], 1, [who])
        if t is None:
            raise OperationError(f"{who}: a live loudness stream needs a target in LUFS")
        g = _check_max_gain(max_gain_db, who)
        _rate_array([output_rate], 1)
        self._m, self._h = model, C.c_void_p()
        self.target, self.max_gain_db = float(t[0]), g
        self.rate = int(output_rate) if output_rate else model.audio_output_info().sample_rate
        err = N.sb200_error()
        _check(model._lib.sb200_loudness_stream_create(model._h, int(output_rate or 0), self.target, g,
                                                       C.byref(self._h), C.byref(err)), err)

    def state(self) -> dict:
        """{"lufs": the last reading (-inf before any), "gain": the last gain, "samples": samples metered, "clipped":
        samples clamped}."""
        lufs, gain, n, clipped = C.c_double(), C.c_float(), C.c_int64(), C.c_int64()
        err = N.sb200_error()
        _check(self._m._lib.sb200_loudness_stream_state(self._h, C.byref(lufs), C.byref(gain), C.byref(n),
                                                        C.byref(clipped), None, C.byref(err)), err)
        return {"lufs": float(lufs.value), "gain": float(gain.value), "samples": int(n.value),
                "clipped": int(clipped.value)}

    @property
    def last_pass_ms(self) -> float:
        """The "loudness" device time (ms) of the last chunk pass this meter was in."""
        ms, err = C.c_float(), N.sb200_error()
        _check(self._m._lib.sb200_loudness_stream_state(self._h, None, None, None, None, C.byref(ms), C.byref(err)),
               err)
        return float(ms.value)

    def __del__(self):
        try:
            if self._h:
                self._m._lib.sb200_loudness_stream_free(self._h)
                self._h = None
        except Exception:
            pass


class WatermarkStream:
    """One realtime stream's watermark on the device (sb200_watermark_stream_*): the voice's watermark as it was when
    the stream was made, kept to the stream's end, at the stream's delivered rate `output_rate` (None: the voice's).
    The stage holds back fewer than 10 ms (the samples past the last whole block) until the stream's last chunk.
    Made by `open`, which gives None for a voice that marks nothing."""

    def __init__(self, model: "_VitsCommons", handle: C.c_void_p, rate: int):
        self._m, self._h, self.rate = model, handle, rate

    @classmethod
    def open(cls, model: "_VitsCommons", output_rate: Optional[int] = None) -> Optional["WatermarkStream"]:
        h, err = C.c_void_p(), N.sb200_error()
        _check(model._lib.sb200_watermark_stream_create(model._h, int(output_rate or 0), C.byref(h), C.byref(err)),
               err)
        if not h.value:
            return None
        return cls(model, h, int(output_rate) if output_rate else model.audio_output_info().sample_rate)

    @property
    def last_pass_ms(self) -> float:
        """The "watermark" device time (ms) of the last chunk pass this stream was in."""
        ms = C.c_float()
        self._m._lib.sb200_watermark_stream_profile(self._h, C.byref(ms))
        return float(ms.value)

    def __del__(self):
        try:
            if self._h:
                self._m._lib.sb200_watermark_stream_free(self._h)
                self._h = None
        except Exception:
            pass


def _stream_mark(model, output_rate) -> Optional[WatermarkStream]:
    """The watermark of a new stream of `model` (None when the voice marks nothing, or is not a loaded streaming voice
    of this library, which holds no setting)."""
    if not isinstance(model, VitsStreamingModel) or not getattr(model, "_h", None):
        return None
    return WatermarkStream.open(model, output_rate)


def _stream_meter(model, live_loudness, max_gain_db, output_rate, who: str) -> Optional[LoudnessStream]:
    """The meter of a stream with `live_loudness` (None: none; a target in LUFS: a fresh meter; a LoudnessStream: that
    meter, continued), checked against the stream's output rate.  Errors name `who`."""
    if live_loudness is None:
        return None
    if isinstance(live_loudness, LoudnessStream):
        rate = int(output_rate) if output_rate else model.audio_output_info().sample_rate
        if live_loudness._m is not model or not live_loudness._h:
            raise OperationError(f"{who}: the loudness stream was made for another voice")
        if live_loudness.rate != rate:
            raise OperationError(f"{who}: the loudness stream meters {live_loudness.rate} Hz and the stream is "
                                 f"delivered at {rate} Hz")
        return live_loudness
    return LoudnessStream(model, live_loudness, 20.0 if max_gain_db is None else max_gain_db, output_rate, who)


def _check_live_loudness(live_loudness, max_gain_db, encoding, who: str) -> None:
    """The checks of a stream's live loudness that need no device: its target, its maximum gain, and an encoding that
    can be metered (FLAC cannot stream)."""
    if live_loudness is None:
        if max_gain_db is not None:
            raise OperationError(f"{who}: a maximum gain is the cap of a live loudness meter: give live_loudness")
        return
    if encoding == "flac":
        raise OperationError(f"{who}: live loudness cannot meter FLAC, which does not stream")
    if not isinstance(live_loudness, LoudnessStream):
        if _loudness_array([live_loudness], 1, [who]) is None:
            raise OperationError(f"{who}: live loudness target {live_loudness!r} is not a target in LUFS")
    elif max_gain_db is not None:
        raise OperationError(f"{who}: a LoudnessStream keeps its own maximum gain")
    if max_gain_db is not None:
        _check_max_gain(max_gain_db, who)


def refuse_live_loudness(live_loudness, where: str) -> None:
    """Models without device streaming cannot meter a stream."""
    if live_loudness is not None:
        raise OperationError(f"{where}: live loudness needs a streaming voice of this library")


def _delivered_bounds(warp: Optional[ProsodyStream], resampler: Optional["Resampler"]):
    """A contoured stream's (or one with breaks) per-id delivered ends at its delivered rate: ceil(end * up / down) with an output rate, as
    the batch alignments place them; None for a stream without a contour."""
    if warp is None or warp.bounds is None:
        return None
    up, down = rate_ratio(warp._m.audio_output_info().sample_rate, None if resampler is None else resampler.rate)
    return -((-warp.bounds * up) // down)


def _trim_frames(trim: slice) -> Tuple[int, int]:
    """The overlap frames a SpeechStreamer audio slice drops at each end."""
    return (trim.start or 0) // HOP, (-trim.stop // HOP) if trim.stop is not None else 0


class _Stream:
    """One sentence streamed from its latent `enc`: its own chunk schedule with the one-shot rule of piper/src/lib.rs
    (a sentence of at most 2 chunks and 2 paddings is decoded whole), and the stream objects its chunks pass through
    on the device.  `key`: what a StreamBatch calls it."""

    def __init__(self, key, enc, chunk_size: int, chunk_padding: int, resampler: Optional[Resampler] = None,
                 encoding: Optional[str] = None, gain: float = 1.0, warp: Optional[ProsodyStream] = None,
                 meter: Optional[LoudnessStream] = None, mark: Optional[WatermarkStream] = None):
        self.key, self.enc, self.resampler = key, enc, resampler
        self.meter, self.mark = meter, mark
        self.encoding, self.gain = encoding, gain
        self.warp = warp
        self.chunker = AdaptiveMelChunker(enc.num_frames, chunk_size, chunk_padding)
        self.one_shot = enc.num_frames <= (chunk_size * 2 + chunk_padding * 2)

    @property
    def bounds(self) -> Optional[np.ndarray]:
        """Each id's delivered end (int64, one per id) at the stream's delivered rate when the stream has a pitch
        contour (see ProsodyStream; with an output rate at ceil(end * up / down)), else None."""
        return _delivered_bounds(self.warp, self.resampler)

    @property
    def on_device(self) -> bool:
        """Whether the chunks' trim and crossfade run on the device, with the stream's encoding, resampler, prosody
        stream or meter."""
        return not (self.encoding is None and self.resampler is None and self.warp is None and self.meter is None
                    and self.mark is None)

    def next_chunk(self):
        """(lo, hi, audio slice or None): the frames to decode next, and how the plain path trims them (None: the
        one-shot chunk, returned as decoded)."""
        (m0, m1), (a0, a1) = next(self.chunker)
        if self.one_shot:
            self.chunker.consume()
            return 0, self.enc.num_frames, None
        return m0, self.enc.num_frames if m1 is None else m1, slice(a0, a1)

    @property
    def done(self) -> bool:
        return self.chunker.last_end_index is None


def _device_post(model, plan) -> list:
    """One infer_decoder_batch call for planned chunks [(stream, lo, hi, trim)] of streams with the same encoding,
    trim kind (one-shot or not) and kinds of resampler, prosody stream and meter: each chunk trimmed and crossfaded on
    the device, then passed through its stream's objects, whose last chunk flushes them."""
    s0 = plan[0][0]
    streams = [s for s, _, _, _ in plan]
    kw = {}
    if s0.resampler is not None or s0.warp is not None or s0.meter is not None or s0.mark is not None:
        kw.update(resamplers=[s.resampler for s in streams], last=[s.done for s in streams])
    if s0.mark is not None:
        kw["marks"] = [s.mark for s in streams]
    if s0.warp is not None:
        kw["warps"] = [s.warp for s in streams]
    if s0.meter is not None:
        kw["meters"] = [s.meter for s in streams]
    if s0.encoding is not None:
        kw.update(gains=[s.gain for s in streams], encoding=s0.encoding)
    chunks = [(s.enc, lo, hi) + ((0, 0) if trim is None else _trim_frames(trim)) for s, lo, hi, trim in plan]
    return model.infer_decoder_batch(chunks, fade=0 if plan[0][3] is None else 42, **kw)


class SpeechStreamer(_Stream):
    """piper/src/lib.rs:765-858: chunked decoder runs with overlap trimming + crossfade(42).  With a resampler, each
    chunk's trim and crossfade run on the device and the chunk leaves at the resampler's rate.  With an encoding, they
    run on the device too and each chunk leaves as G.711 bytes of its to_i16_vec after `gain`."""

    def __init__(self, enc: EncoderOutputs, chunk_size: int, chunk_padding: int,
                 resampler: Optional[Resampler] = None, encoding: Optional[str] = None, gain: float = 1.0,
                 warp: Optional[ProsodyStream] = None, meter: Optional[LoudnessStream] = None,
                 mark: Optional[WatermarkStream] = None):
        super().__init__(None, enc, chunk_size, chunk_padding, resampler, encoding, gain, warp, meter, mark)

    def __iter__(self) -> Iterator[AudioSamples]:
        return self

    def __next__(self) -> AudioSamples:
        lo, hi, trim = self.next_chunk()
        if self.on_device:
            return _device_post(self.enc._m, [(self, lo, hi, trim)])[0]
        if trim is None:
            return self.enc.infer_decoder()
        out = AudioSamples(self.enc.infer_decoder(lo, hi).as_slice()[trim])
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
                            seeds: Optional[Sequence] = None,
                            speaker_blends: Optional[Sequence] = None,
                            target_durations: Optional[Sequence] = None,
                            breaks: Optional[Sequence] = None) -> List[EncoderOutputs]:
        """infer_encoder over many utterances in one encoder pass.  `configs`: one PiperSynthesisConfig per utterance,
        or None for the fallback config; each latent equals infer_encoder alone with its config as the fallback,
        except for the on-device noise of an unseeded utterance, whose draws depend on the batch position.
        `duration_scales` / `durations`: per-id duration controls as for infer_batch_with_durations; each output's
        `p_duration` holds its frames per id.  `seeds`: noise seeds as for infer_batch_with_values; a seeded latent
        equals the `z` of the same utterance synthesised with the same seed.  `speaker_blends`: as for
        infer_batch_with_values; each latent keeps its blend, and every decoder chunk of it speaks with that blend.
        `target_durations`: as for infer_batch_with_values: each latent's frames are fitted in this encoder pass, and
        its chunks then decode unchanged; each output's `fit` holds (u, delivered length) per span (None without).
        `breaks`: the pauses (per id, as for infer_batch_with_values) the latent's stream will insert, counted in its
        targets; this pass inserts none, and without targets they are only checked."""
        n = len(batches)
        o = _batch_options(self, n, [len(b) for b in batches], configs, duration_scales, durations, seeds,
                           speaker_blends=speaker_blends, breaks=breaks, target_durations=target_durations)
        _check_not_empty(batches)
        if n == 0:
            return []
        packed, offs = _pack_ids(batches)
        outs = (C.c_void_p * n)()
        err = N.sb200_error()
        t = o.targets
        u = None if t is None else np.zeros(len(t[2]), np.float32)
        ln = None if t is None else np.zeros(len(t[2]), np.int64)
        _check(self._lib.sb200_encode_batch_ids_targets(
            self._h, _ptr(packed, C.c_int64), _ptr(offs, C.c_size_t), n, o.cfgs, _ptr(o.scales, C.c_float),
            _ptr(o.frames, C.c_int32), _ptr(o.seeds, C.c_uint64), _ptr(o.seeded, C.c_int32),
            _ptr(o.blend_speakers, C.c_int64), _ptr(o.blend_weights, C.c_float), _ptr(o.blend_offsets, C.c_size_t),
            _ptr(o.breaks if t is not None else None, C.c_float), *_target_images(t), _ptr(u, C.c_float),
            _ptr(ln, C.c_int64), outs, C.byref(err)), err)
        res = [EncoderOutputs(self, C.c_void_p(outs[i])) for i in range(n)]
        if t is not None:
            for b, e in enumerate(res):
                k0, k1 = int(t[3][b]), int(t[3][b + 1])
                e.fit = [(float(u[k]), int(ln[k])) for k in range(k0, k1)]
        return res

    def infer_decoder_batch(self, chunks: Sequence[tuple], pcm16: bool = False, fade: int = 0,
                            gains: Optional[Sequence[float]] = None, resamplers: Optional[Sequence] = None,
                            last: Optional[Sequence[bool]] = None, encoding: Optional[str] = None,
                            warps: Optional[Sequence] = None, meters: Optional[Sequence] = None,
                            marks: Optional[Sequence] = None) -> list:
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
        entries, or resamplers None: the voice's rate) and the conversion; last[k] flushes both streams.

        With `meters` (one LoudnessStream or None per chunk; chunks may carry trims, as with resamplers), what chunk k
        delivers is metered by its live loudness stream after all that, gains[k] applies after the meter, and pcm16 /
        G.711 convert it at the fixed scale (sb200_decode_chunks_metered).

        With `marks` (one WatermarkStream or None per chunk; chunks may carry trims, as with resamplers), what chunk k
        delivers after resampling is marked by its stream before any meter and conversion: the stream emits its
        whole 10 ms blocks and holds back the rest until its last chunk (sb200_decode_chunks_marked)."""
        refuse_flac(encoding, "a decoder chunk pass")
        check_encoding(encoding)
        if encoding is not None and pcm16:
            raise OperationError("pcm16 and an encoding are two output formats: give one")
        n = len(chunks)
        lo, hi = np.zeros(n, np.int64), np.zeros(n, np.int64)
        tlo, thi = np.zeros(n, np.int64), np.zeros(n, np.int64)
        hs = (C.c_void_p * n)()
        for k, c in enumerate(chunks):
            if len(c) not in ((3, 5) if pcm16 or encoding or resamplers is not None or warps is not None
                              or meters is not None or marks is not None else (3,)):
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
        if resamplers is not None or warps is not None or meters is not None or marks is not None:
            rs = _handles([None] * n if resamplers is None else resamplers, n, Resampler, "resamplers")
            mk = None if marks is None else _handles(marks, n, WatermarkStream, "marks")
            ws = None if warps is None else _handles(warps, n, ProsodyStream, "warps")
            ms = None if meters is None else _handles(meters, n, LoudnessStream, "meters")
            fl = np.zeros(n, np.int32) if last is None else np.array([1 if x else 0 for x in
                                                                        _per_utterance(last, n, "last flags")], np.int32)
            g = None if gains is None else np.ascontiguousarray(gains, dtype=np.float32)
            outs = (C.c_void_p * n)()
            lens = (C.c_size_t * n)()
            fmt = G711_LAW[encoding] + 2 if encoding else 1 if pcm16 else 0
            gp = None if g is None else g.ctypes.data_as(C.POINTER(C.c_float))
            _check(self._lib.sb200_decode_chunks_marked(
                self._h, hs, p64(lo), p64(hi), p64(tlo), p64(thi), n, int(fade), gp, rs, ws, ms, mk,
                _ptr(fl, C.c_int32), fmt, outs, lens, C.byref(err)), err)
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
                         pitch: Optional[float] = None, tempo: Optional[float] = None,
                         pitch_contour: Optional[Sequence] = None,
                         formant_ratio: Optional[float] = None, speaker_blend=None,
                         live_loudness=None, max_gain_db: Optional[float] = None,
                         volume_contour: Optional[Sequence] = None,
                         breaks: Optional[Sequence] = None, target_duration=None) -> SpeechStreamer:
        """`formant_ratio`: as for infer_batch_with_values' formants, on top of `pitch` / `tempo` / `pitch_contour` or
        alone, the sentence's formant stage carried as one stream on the device (ProsodyStream): the concatenation of
        the chunks is the formant stage applied at once to the sentence the stream yields without it, then resampled and
        encoded as without it.  The stage holds back 768 - 1023 samples (35 - 46 ms at 22.05 kHz) more.
        `speaker_blend`: the sentence's speaker blend (a mapping {speaker: weight}, see infer_batch_with_values), or
        None for the fallback config's speaker; the latent keeps it, so every chunk speaks with it.
        `seed`: the sentence's noise seed (see infer_batch_with_values), or None for positional noise.
        `output_rate`: the chunks' sample rate (see infer_batch_with_values), the sentence resampled as one stream.
        `encoding`: "mulaw" / "alaw" for chunks of G.711 `bytes`: each is G.711 of to_i16_vec of the chunk the stream
        yields without an encoding, after the linear `gain` (None: 1; encoded streams only), encoded on the device.
        `pitch` / `tempo`: ratios as for infer_batch_with_values, the sentence warped as one stream on the device
        (ProsodyStream): the concatenation of the chunks is the sentence the stream yields without ratios, warped at
        once, then resampled and encoded as without ratios.
        `pitch_contour`: one pitch ratio per character of `phonemes` (as for speak_batch_with_alignment), applied to
        that character's id and pad; it combines with `tempo` but not with `pitch`.  The concatenation of the chunks is
        the sentence the stream yields without it, with that contour applied at once (sb200_debug_prosody_contour), and
        the streamer's `bounds` give each id's delivered end.
        `live_loudness`: a target in LUFS, for a fresh live loudness meter (LoudnessStream, capped at `max_gain_db`,
        default 20), or a LoudnessStream to continue (a request's meter across its sentences).  What the stream
        delivers is metered and scaled on the device as it leaves, holding nothing back; `gain` applies after the
        meter, and G.711 is taken at the fixed scale.
        `volume_contour`: one volume level per character of `phonemes` (as for speak_batch_with_alignment's
        volume_contours), applied to that character's id and pad, on top of the rest or alone (ProsodyStream): the
        concatenation of the chunks is the sentence the stream yields without it with that contour applied at once,
        before resampling, metering and encoding.  It holds nothing back.
        `breaks`: one pause in ms per character of `phonemes` (as for speak_batch_with_alignment's breaks), on top of
        the rest or alone (ProsodyStream): the concatenation of the chunks is the sentence the stream yields without
        them with those pauses inserted at once, before resampling, metering and encoding.  A chunk emits the pauses its
        input reaches, holding nothing back, and the streamer's `bounds` give each id's delivered end.
        `target_duration`: the sentence's target durations (as for speak_batch_with_alignment's target_durations: a
        duration in ms, or (first, last, ms) spans of phoneme characters); the latent's frames are fitted in its
        encoder pass, with its breaks counted, and its chunks then run unchanged.  The encoder outputs' `fit` holds
        each span's (u, delivered length)."""
        if not isinstance(self, VitsStreamingModel):
            refuse_targets(target_duration, "stream_synthesis")
            refuse_breaks(breaks, "stream_synthesis")
            refuse_volume(volume_contour, "stream_synthesis")
            refuse_live_loudness(live_loudness, "stream_synthesis")
            refuse_formants(formant_ratio, "stream_synthesis")
            refuse_prosody(pitch, tempo, "stream_synthesis")
            refuse_contour(pitch_contour, "stream_synthesis")
        o = _stream_options(self, "stream_synthesis", None, phonemes, seed=seed, output_rate=output_rate,
                            encoding=encoding, gain=gain, pitch=pitch, tempo=tempo, pitch_contour=pitch_contour,
                            formant_ratio=formant_ratio, speaker_blend=speaker_blend, live_loudness=live_loudness,
                            max_gain_db=max_gain_db, volume_contour=volume_contour, breaks=breaks,
                            target_duration=target_duration)
        if o.target is not None:
            enc = self.infer_encoder_batch([o.ids], seeds=[o.seed], speaker_blends=[o.blend], target_durations=[o.target],
                                           breaks=[o.breaks])[0]
        elif o.seed is None and o.blend is None:
            enc = self.infer_encoder(o.ids)
        else:
            enc = self.infer_encoder_batch([o.ids], seeds=[o.seed], speaker_blends=[o.blend])[0]
        resampler, warp, meter = _open_stream(self, o, enc)
        return SpeechStreamer(enc, chunk_size, chunk_padding, resampler, o.encoding, o.gain, warp, meter,
                              _stream_mark(self, o.output_rate))


def _stream_gain(encoding, gain) -> float:
    """Checks a stream's encoding and gain; the gain as a float (1 when None)."""
    check_encoding(encoding)
    if gain is None:
        return 1.0
    if encoding is None:
        raise OperationError("a stream's gain applies before its G.711 encoding: give an encoding with it")
    return float(_gain_array([gain], 1)[0])


def _check_chunking(chunk_size, chunk_padding):
    if not isinstance(chunk_size, int) or chunk_size < 1:
        raise OperationError(f"Invalid chunk size {chunk_size!r}: expected a positive integer")
    if not isinstance(chunk_padding, int) or chunk_padding < 0:
        raise OperationError(f"Invalid chunk padding {chunk_padding!r}: expected a non-negative integer")


@dataclass
class _StreamOptions:
    """One stream's options, checked once by _stream_options."""
    key: Optional[int]                  # its StreamBatch key (None: a stream_synthesis stream)
    who: str                            # what its errors name
    ids: List[int]
    config: Optional[PiperSynthesisConfig]
    chunk_size: Optional[int]
    seed: Optional[int]
    output_rate: Optional[int]
    encoding: Optional[str]
    gain: float
    pitch: Optional[float]
    tempo: Optional[float]
    contour: Optional[Sequence]         # per id
    formant: Optional[float]
    blend: Optional[dict]
    live_loudness: object               # None, a target in LUFS or a LoudnessStream to continue
    max_gain_db: Optional[float]
    volume: Optional[Sequence] = None   # per id
    breaks: Optional[Sequence] = None   # per id
    target: object = None               # checked target entry in ids (_target_entry), or None
    mark: object = None                 # StreamBatch: the WatermarkStream read when the stream was added, or None


def _stream_options(model, where: str, key: Optional[int], ids_or_phonemes, config=None, chunk_size=None,
                    chunk_padding=None, seed=None, output_rate=None, encoding=None, gain=None, pitch=None, tempo=None,
                    pitch_contour=None, formant_ratio=None, speaker_blend=None, live_loudness=None, max_gain_db=None,
                    carried=(), volume_contour=None, breaks=None, target_duration=None) -> _StreamOptions:
    """The options of one stream of `model`, checked in one order: config, live loudness, speaker blend, formant ratio,
    pitch and tempo, seed, output rate, FLAC (refused by the name `where`), encoding and gain, the config's speaker,
    chunking, then the ids (phonemes are mapped), the contour, the volume contour, the breaks and the target duration.
    Errors name "stream" (key None) or "stream {key}".
    `chunk_size`: checked with `chunk_padding` when given.  `carried`: the LoudnessStreams the caller's unfinished
    streams carry, which live_loudness may not be."""
    if config is not None and not isinstance(config, PiperSynthesisConfig):
        raise OperationError("Invalid configuration for Vits Model")
    who = "stream" if key is None else f"stream {key}"
    _check_live_loudness(live_loudness, max_gain_db, encoding, who)
    if isinstance(live_loudness, LoudnessStream):
        if any(m is live_loudness for m in carried):
            raise OperationError(f"{who}: the LoudnessStream is already carried by an unfinished stream of this batch")
        _stream_meter(model, live_loudness, None, output_rate, who)
    _blend_arrays(model, [speaker_blend], 1, [who])
    phi = _stream_formant(formant_ratio, who)
    pit, tmp = _prosody_arrays([pitch], [tempo], 1)
    _seed_arrays([seed], 1)
    _rate_array([output_rate], 1)
    refuse_flac(encoding, where)
    g = _stream_gain(encoding, gain)
    if config is not None and config.speaker is not None and config.speaker not in (model.get_speakers() or {}):
        raise OperationError(f"No speaker was found with the given id `{config.speaker}`")     # as check_config
    if chunk_size is not None:
        _check_chunking(chunk_size, chunk_padding)
    contour, volume, brk, target = pitch_contour, volume_contour, breaks, None
    chars = isinstance(ids_or_phonemes, str)
    if target_duration is not None:
        target = _target_entry(target_duration, who, None if tmp is None else tmp[0], len(ids_or_phonemes),
                               "character" if chars else "id")
    if chars and (pitch_contour is not None or volume_contour is not None or breaks is not None or
                  target_duration is not None):
        ids, src = model.phonemes_to_input_ids_map(ids_or_phonemes)
        target = _char_targets_to_ids(target, ids_or_phonemes, src, who)
        if pitch_contour is not None:
            contour = _char_values_to_ids(pitch_contour, ids_or_phonemes, src, who, "pitch ratios", _contour_value)
        if volume_contour is not None:
            volume = _char_values_to_ids(volume_contour, ids_or_phonemes, src, who, "volume levels", _volume_value,
                                         0.0)
        if breaks is not None:
            brk = _char_breaks_to_ids(breaks, ids_or_phonemes, src, who)
    elif isinstance(ids_or_phonemes, str):
        ids = model.phonemes_to_input_ids(ids_or_phonemes)
    else:
        ids = [int(i) for i in ids_or_phonemes]
    if contour is not None:
        _contour_arrays([len(ids)], [contour], pit, [who])
    if volume is not None:
        _volume_arrays([len(ids)], [volume], [who])
    if brk is not None:
        _break_arrays([len(ids)], [brk], [who])
    if not ids:
        raise OperationError("Failed to run model inference. Error: empty input sequence")
    return _StreamOptions(key, who, ids, config, chunk_size, seed, output_rate, encoding, g, pitch, tempo, contour, phi,
                          speaker_blend, live_loudness, max_gain_db, volume, brk, target)


def _open_stream(model, o: _StreamOptions, enc):
    """(resampler, ProsodyStream, meter) of a stream with options `o` and latent `enc`, each None when not asked for."""
    return (_stream_resampler(model, o.output_rate),
            _stream_prosody(model, o.pitch, o.tempo, o.contour, enc, o.formant, o.volume, o.breaks),
            _stream_meter(model, o.live_loudness, o.max_gain_db, o.output_rate, o.who))


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
        self._pending: List[_StreamOptions] = []      # the streams not encoded yet
        self._active: List[_Stream] = []
        self._retired: dict = {}      # key -> delivered ends (None: no contour) of the streams the last step ended
        self._next_key = 0

    def add(self, ids_or_phonemes, config: Optional[PiperSynthesisConfig] = None, seed: Optional[int] = None,
            output_rate: Optional[int] = None, encoding: Optional[str] = None, gain: Optional[float] = None,
            pitch: Optional[float] = None, tempo: Optional[float] = None,
            pitch_contour: Optional[Sequence] = None, formant_ratio: Optional[float] = None,
            speaker_blend=None, live_loudness=None, max_gain_db: Optional[float] = None,
            volume_contour: Optional[Sequence] = None, breaks: Optional[Sequence] = None,
            target_duration=None) -> int:
        """`seed`: the stream's noise seed (see infer_batch_with_values); a seeded stream yields what
        `stream_synthesis(..., seed=seed)` yields, whatever other streams share its encoder pass.  `output_rate`,
        `encoding` and `gain`: the stream's sample rate and G.711 encoding, as for stream_synthesis; `pitch` / `tempo`:
        its ratios, as there.  `pitch_contour`: one pitch ratio per phoneme character (phonemes) or per id (ids), as
        for stream_synthesis; its length and values are checked here, and what needs the sentence's frames fails as the
        stream's error item.  `bounds(key)` gives a contoured stream's per-id delivered ends once it is encoded.  A
        warped stream's chunks go through passes of their own, so the other streams keep their passes and their
        bits.  `formant_ratio`: the stream's formant ratio, as for stream_synthesis; it is checked here, naming the
        stream, and a stream with one is warped (in those passes) even without pitch or tempo.  `speaker_blend`: the
        stream's speaker blend, as for stream_synthesis; it replaces its config's speaker and is checked here.
        `live_loudness` / `max_gain_db`: the stream's live loudness, as for stream_synthesis; a LoudnessStream that an
        unfinished stream of this batch already carries is refused.  Metered streams go through passes of their own,
        so the other streams keep their passes and their bits.  `volume_contour`: one volume level per phoneme
        character (phonemes) or per id (ids), as for stream_synthesis; checked here, naming the stream.  A stream with
        one goes through the warped passes.  `breaks`: one pause in ms per phoneme character (phonemes) or per id
        (ids), as for stream_synthesis; checked here, naming the stream.  A stream with pauses goes through the warped
        passes, and `bounds(key)` gives its per-id delivered ends once it is encoded.  `target_duration`: the
        stream's target durations, as for stream_synthesis (spans of phoneme characters or of ids); checked here,
        naming the stream, and fitted in the step's encoder pass, which the other streams share unchanged."""
        if not isinstance(self.model, VitsStreamingModel):
            refuse_targets(target_duration, "StreamBatch")
            refuse_breaks(breaks, "StreamBatch")
            refuse_volume(volume_contour, "StreamBatch")
            refuse_live_loudness(live_loudness, "StreamBatch")
            refuse_formants(formant_ratio, "StreamBatch")
            refuse_prosody(pitch, tempo, "StreamBatch")
            refuse_contour(pitch_contour, "StreamBatch")
        return self._add(ids_or_phonemes, config, self.chunk_size, seed, output_rate, encoding, gain, pitch, tempo,
                         pitch_contour, speaker_blend, formant_ratio, live_loudness, max_gain_db, volume_contour, breaks,
                         target_duration)

    def _add(self, ids_or_phonemes, config, chunk_size: int, seed: Optional[int] = None,
             output_rate: Optional[int] = None, encoding: Optional[str] = None, gain: Optional[float] = None,
             pitch: Optional[float] = None, tempo: Optional[float] = None, pitch_contour=None,
             speaker_blend=None, formant_ratio=None, live_loudness=None, max_gain_db=None, volume_contour=None,
             breaks=None, target_duration=None) -> int:
        carried = [o.live_loudness for o in self._pending] + [s.meter for s in self._active]
        o = _stream_options(self.model, "StreamBatch", self._next_key, ids_or_phonemes, config, chunk_size,
                            self.chunk_padding, seed=seed, output_rate=output_rate, encoding=encoding, gain=gain,
                            pitch=pitch, tempo=tempo, pitch_contour=pitch_contour, formant_ratio=formant_ratio,
                            speaker_blend=speaker_blend, live_loudness=live_loudness, max_gain_db=max_gain_db,
                            carried=carried, volume_contour=volume_contour, breaks=breaks,
                            target_duration=target_duration)
        o.mark = _stream_mark(self.model, o.output_rate)      # the voice's watermark as it is when the stream is added
        self._next_key += 1
        self._pending.append(o)
        return o.key

    def bounds(self, key) -> Optional[np.ndarray]:
        """Stream `key`'s per-id delivered ends at its delivered rate (see SpeechStreamer.bounds), or None when it has
        no pitch contour.  Available from the step that encodes the stream until the next step after the one that
        returns its last chunk (or its error): the batch keeps no state for a stream once that next step has run.
        KeyError outside that window or for an unknown key."""
        for s in self._active:
            if s.key == key:
                return s.bounds
        if key in self._retired:
            return self._retired[key]
        raise KeyError(f"stream {key!r} is not encoded, or ended before the last step")

    def __len__(self) -> int:
        """Streams added and not yet finished."""
        return len(self._pending) + len(self._active)

    def __contains__(self, key) -> bool:
        """Whether stream `key` has chunks still to come."""
        return any(o.key == key for o in self._pending) or any(s.key == key for s in self._active)

    def step(self) -> List[tuple]:
        out = []
        active = self._active
        if self._pending:
            pend, self._pending = self._pending, []
            fallback = None
            if any(o.config is not None for o in pend):
                fallback = self.model.get_fallback_synthesis_config()

            def encode(ps):
                ids = [o.ids for o in ps]
                configs = None if fallback is None else [fallback if o.config is None else o.config for o in ps]
                if any(o.target is not None for o in ps):
                    return self.model.infer_encoder_batch(ids, configs, seeds=[o.seed for o in ps],
                                                          speaker_blends=[o.blend for o in ps],
                                                          target_durations=[o.target for o in ps],
                                                          breaks=[o.breaks for o in ps])
                if all(o.seed is None and o.blend is None for o in ps):
                    return self.model.infer_encoder_batch(ids, configs)
                return self.model.infer_encoder_batch(ids, configs, seeds=[o.seed for o in ps],
                                                      speaker_blends=[o.blend for o in ps])
            for o, (enc, err) in zip(pend, _each_or_alone(encode, pend)):
                if err is None:
                    try:
                        resampler, warp, meter = _open_stream(self.model, o, enc)
                        active.append(_Stream(o.key, enc, o.chunk_size, self.chunk_padding, resampler, o.encoding,
                                              o.gain, warp, meter, o.mark))
                        continue
                    except SonataError as e:
                        err = e
                out.append((o.key, err))
        plan = [(s,) + s.next_chunk() for s in active]
        failed = set()
        # one pass per (encoding, resampled, one-shot, warped, metered): the streams without an encoding first, in
        # their usual passes; warped and metered streams in passes of their own
        plain_key = (None, False, False, False, False, False)
        groups = {plain_key: [], (None, True, False, False, False, False): [],
                  (None, True, True, False, False, False): []}
        for p in plan:
            s = p[0]
            k = plain_key if not s.on_device else (s.encoding, s.resampler is not None, p[3] is None,
                                                   s.warp is not None, s.meter is not None, s.mark is not None)
            groups.setdefault(k, []).append(p)
        decoded = {}
        for key, group in groups.items():
            if key == plain_key:
                call = lambda pl: self.model.infer_decoder_batch([(s.enc, lo, hi) for s, lo, hi, _ in pl])
            else:
                call = lambda pl: _device_post(self.model, pl)
            if group:
                decoded.update({id(p): r for p, r in zip(group, _each_or_alone(call, group))})
        for p in plan:
            s, _, _, trim = p
            a, err = decoded[id(p)]
            if err is not None:
                out.append((s.key, err))
                failed.add(s.key)
                continue
            if trim is not None and not s.on_device:
                a = AudioSamples(a.as_slice()[trim])
                a.crossfade(42)
            out.append((s.key, a))
        self._active = [s for s in active if not s.done and s.key not in failed]
        self._retired = {s.key: s.bounds for s in active if s.done or s.key in failed}
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
