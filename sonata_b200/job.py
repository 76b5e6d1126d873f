"""Low-level view of one batched synthesis pass (the `sb200_job_*` entry points): used by
bench.py (device-resident timing, NCCL send buffers) and by the parity tests (noise injection,
per-stage intermediates).  Ordinary callers use `VitsModel.speak_*`."""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _native as N
from .core import G711_LAW, Audio, OperationError, check_encoding
from .piper import (_check, _config_array, _duration_arrays, _gain_array, _loudness_array, _prosody_arrays, _ptr,
                    _rate_array, _seed_arrays, _take_audio, _take_bytes)


class SynthesisJob:
    def __init__(self, model, batches: Sequence[Sequence[int]], eps_w: Optional[Sequence] = None,
                 eps_z: Optional[Sequence] = None, debug: bool = False, configs: Optional[Sequence] = None,
                 seeds: Optional[Sequence] = None, output_rates: Optional[Sequence] = None,
                 loudness: Optional[Sequence] = None, pitches: Optional[Sequence] = None,
                 tempos: Optional[Sequence] = None):
        """`configs`: one PiperSynthesisConfig per utterance (see set_configs); None keeps the voice's fallback config.
        `seeds`: noise seeds (see set_seeds).  `output_rates`: output sample rates (see set_output_rates).
        `loudness`: loudness targets (see set_loudness).  `pitches` / `tempos`: pitch and tempo ratios (see
        set_prosody)."""
        self._m = model
        self._lib = model._lib
        n = len(batches)
        self.batch = n
        self._lens = [len(b) for b in batches]
        _config_array(configs, n)             # argument errors before the job exists
        _seed_arrays(seeds, n)
        _rate_array(output_rates, n)
        _loudness_array(loudness, n)
        _prosody_arrays(pitches, tempos, n)
        packed = np.ascontiguousarray(np.concatenate([np.asarray(b, dtype=np.int64) for b in batches]))
        offs = np.zeros(n + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(b) for b in batches])
        keep = []

        def ptrs(arrs):
            if arrs is None:
                return None
            out = (C.POINTER(C.c_float) * n)()
            for i, a in enumerate(arrs):
                if a is None:
                    out[i] = None
                else:
                    a = np.ascontiguousarray(a, dtype=np.float32)
                    keep.append(a)
                    out[i] = a.ctypes.data_as(C.POINTER(C.c_float))
            return out

        pw, pz = ptrs(eps_w), ptrs(eps_z)
        zf = None
        if eps_z is not None:
            zf = np.array([0 if a is None else np.asarray(a).shape[0] for a in eps_z], dtype=np.uint64)
        self._h = C.c_void_p()
        err = N.sb200_error()
        _check(self._lib.sb200_job_create(
            model._h, packed.ctypes.data_as(C.POINTER(C.c_int64)), offs.ctypes.data_as(C.POINTER(C.c_size_t)), n,
            pw, pz, None if zf is None else zf.ctypes.data_as(C.POINTER(C.c_size_t)), C.byref(self._h),
            C.byref(err)), err)
        if debug:
            self._lib.sb200_job_set_debug(self._h, 1)
        if configs is not None:
            self.set_configs(configs)
        if seeds is not None:
            self.set_seeds(seeds)
        if output_rates is not None:
            self.set_output_rates(output_rates)
        if loudness is not None:
            self.set_loudness(loudness)
        if pitches is not None or tempos is not None:
            self.set_prosody(pitches, tempos)

    def set_configs(self, configs: Optional[Sequence]) -> None:
        """Per-utterance PiperSynthesisConfigs for the next run, or None for the voice's fallback config.  A wrong
        length or an unknown speaker raises OperationError and leaves the job's configs as they were."""
        err = N.sb200_error()
        _check(self._lib.sb200_job_set_configs(self._h, _config_array(configs, self.batch), C.byref(err)), err)

    def set_durations(self, scales: Optional[Sequence] = None, frames: Optional[Sequence] = None) -> None:
        """Per-id duration controls for the next run (see VitsModel.infer_batch_with_durations): scales[b] / frames[b]
        hold one value per id of utterance b, or None.  None and None restores the default.  A bad entry raises
        OperationError naming the utterance and the id, and leaves the job's controls as they were."""
        sc, fr = _duration_arrays(self._lens, scales, frames)
        err = N.sb200_error()
        _check(self._lib.sb200_job_set_durations(self._h, _ptr(sc, C.c_float), _ptr(fr, C.c_int32), C.byref(err)), err)

    def set_seeds(self, seeds: Optional[Sequence]) -> None:
        """Per-utterance noise seeds for the next run (see VitsModel.infer_batch_with_values): an int in [0, 2**64) or
        None per utterance; None for the whole list restores positional noise.  With debug on, the run's draws are
        fetchable as "eps_w" and "eps_z".  A bad entry, or seeds on a job with injected noise, raises OperationError
        and leaves the job's seeds as they were."""
        sv, sf = _seed_arrays(seeds, self.batch)
        err = N.sb200_error()
        _check(self._lib.sb200_job_set_seeds(self._h, _ptr(sv, C.c_uint64), _ptr(sf, C.c_int32), C.byref(err)), err)

    def set_output_rates(self, rates: Optional[Sequence]) -> None:
        """Per-utterance output sample rates for the next run (see VitsModel.infer_batch_with_values), or None for the
        voice's rate throughout.  After such a run, fetch, fetch_i16, copy_out and the samples and offsets of lengths
        all report the resampled signal.  An unsupported rate raises OperationError naming the utterance and leaves the
        job's rates as they were."""
        r = _rate_array(rates, self.batch)
        err = N.sb200_error()
        _check(self._lib.sb200_job_set_output_rates(self._h, _ptr(r, C.c_uint32), C.byref(err)), err)

    def set_loudness(self, targets: Optional[Sequence]) -> None:
        """Per-utterance loudness targets for the next run (see VitsModel.infer_batch_with_values): LUFS in [-70, 0] or
        None per utterance; None for the whole list (or all None) turns loudness off.  A run with targets measures every
        utterance, scales those with a target in place on the device (d_out included), and fetch_i16 / copy_out(fmt=1)
        convert those at the fixed scale 32767 instead of their peak.  A bad entry raises OperationError naming the
        utterance and leaves the job's targets as they were."""
        t = _loudness_array(targets, self.batch)
        err = N.sb200_error()
        _check(self._lib.sb200_job_set_loudness(self._h, _ptr(t, C.c_float), C.byref(err)), err)

    def loudness(self) -> Tuple[np.ndarray, np.ndarray]:
        """(integrated loudness in LUFS as float64, -inf when no block passes the gates; gain applied as float32) per
        utterance of the last run, which must have had targets."""
        lufs = np.zeros(self.batch, np.float64)
        gain = np.zeros(self.batch, np.float32)
        err = N.sb200_error()
        _check(self._lib.sb200_job_loudness(self._h, _ptr(lufs, C.c_double), _ptr(gain, C.c_float), C.byref(err)), err)
        return lufs, gain

    def set_prosody(self, pitches: Optional[Sequence] = None, tempos: Optional[Sequence] = None) -> None:
        """Per-utterance pitch and tempo ratios for the next run (see VitsModel.infer_batch_with_values): a ratio or
        None per utterance in each list; None for a whole list, or lists of None / NaN / 1.0, turn that control off.
        After a run with ratios, fetch, fetch_i16, fetch_g711, fetch_flac, copy_out and the samples and offsets of
        lengths all report the warped signal.  A bad entry raises OperationError naming the utterance and leaves the
        job's ratios as they were."""
        p, t = _prosody_arrays(pitches, tempos, self.batch)
        err = N.sb200_error()
        _check(self._lib.sb200_job_set_prosody(self._h, _ptr(p, C.c_float), _ptr(t, C.c_float), C.byref(err)), err)

    def prosody(self) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """(stretched length n1, delivered length before any output-rate resampling n2, WSOLA frames F) per utterance of
        the last run, which must have had ratios."""
        n1, n2 = np.zeros(self.batch, np.int64), np.zeros(self.batch, np.int64)
        frames = np.zeros(self.batch, np.int32)
        err = N.sb200_error()
        _check(self._lib.sb200_job_prosody(self._h, _ptr(n1, C.c_int64), _ptr(n2, C.c_int64), _ptr(frames, C.c_int32),
                                           C.byref(err)), err)
        return n1, n2, frames

    def id_frames(self) -> List[np.ndarray]:
        """Frames per id of the last run, one int32 array per utterance (one device->host copy for the batch)."""
        total = int(sum(self._lens))
        out = np.zeros(total, np.int32)
        err = N.sb200_error()
        _check(self._lib.sb200_job_id_frames(self._h, _ptr(out, C.c_int32), total, C.byref(err)), err)
        offs = np.concatenate([[0], np.cumsum(self._lens)]).astype(int)
        return [out[offs[b]:offs[b + 1]].copy() for b in range(self.batch)]

    def run(self, d_out_ptr: int = 0, capacity: int = 0) -> float:
        ms, err = C.c_float(), N.sb200_error()
        _check(self._lib.sb200_job_run(self._h, C.c_void_p(d_out_ptr) if d_out_ptr else None, capacity,
                                       C.byref(ms), C.byref(err)), err)
        return float(ms.value)

    def fetch(self) -> List[Audio]:
        outs = (N.sb200_audio * self.batch)()
        err = N.sb200_error()
        _check(self._lib.sb200_job_fetch(self._h, outs, C.byref(err)), err)
        return [_take_audio(outs[i]) for i in range(self.batch)]

    def fetch_i16(self) -> List[np.ndarray]:
        """Per-utterance peak-normalised 16-bit PCM, converted on the device: bit-identical to
        `Audio.samples.to_i16_vec()` (audio/ops/src/samples.rs:51-75) at half the device->host bytes."""
        outs = (C.POINTER(C.c_int16) * self.batch)()
        lens = (C.c_size_t * self.batch)()
        err = N.sb200_error()
        _check(self._lib.sb200_job_fetch_i16(self._h, outs, lens, C.byref(err)), err)
        res = []
        for i in range(self.batch):
            n = int(lens[i])
            res.append(np.ctypeslib.as_array(outs[i], shape=(n,)).copy() if n else np.zeros(0, dtype=np.int16))
            self._lib.sb200_i16_free(outs[i])
        return res

    def fetch_g711(self, law: str, gains: Optional[Sequence] = None) -> List[bytes]:
        """Per-utterance G.711 bytes ("mulaw" or "alaw"), one per sample: the encoding of exactly what fetch_i16
        returns, after gains[b] (None: 1), computed on the device in the i16 conversion's launches."""
        if law is None or check_encoding(law) is None:
            raise OperationError(f"law {law!r} is neither 'mulaw' nor 'alaw'")
        g = _gain_array(gains, self.batch)
        outs = (C.POINTER(C.c_uint8) * self.batch)()
        lens = (C.c_size_t * self.batch)()
        err = N.sb200_error()
        _check(self._lib.sb200_job_fetch_g711(self._h, G711_LAW[law], _ptr(g, C.c_float), outs, lens, C.byref(err)), err)
        return _take_bytes(self._lib, outs, lens)

    def fetch_flac(self, gains: Optional[Sequence] = None) -> List[bytes]:
        """One complete FLAC stream per utterance (see sb200_job_fetch_flac): lossless, of exactly the 16-bit samples
        fetch_i16 returns after gains[b] (None: 1), at the utterance's delivered rate.  Analysed, laid out and packed on
        the device; only the compressed bytes leave the card."""
        g = _gain_array(gains, self.batch)
        outs = (C.POINTER(C.c_uint8) * self.batch)()
        lens = (C.c_size_t * self.batch)()
        err = N.sb200_error()
        _check(self._lib.sb200_job_fetch_flac(self._h, _ptr(g, C.c_float), outs, lens, C.byref(err)), err)
        return _take_bytes(self._lib, outs, lens)

    def copy_out(self, dst_address: int, capacity_bytes: int, fmt: int = 0) -> int:
        """Device -> host copy of the whole result (utterances back to back) into caller memory, e.g. a slice of the
        host segment shared by the ranks of one frontend; fmt 0 = f32, 1 = peak-normalised i16 PCM, 2 / 3 = G.711
        mu-law / A-law of those i16 samples (one byte each).  Returns bytes."""
        wr, err = C.c_size_t(), N.sb200_error()
        _check(self._lib.sb200_job_copy_out(self._h, C.c_void_p(dst_address), capacity_bytes, fmt, C.byref(wr),
                                            C.byref(err)), err)
        return int(wr.value)

    def lengths(self):
        f = (C.c_int64 * self.batch)()
        s = (C.c_int64 * self.batch)()
        o = (C.c_int64 * self.batch)()
        if self._lib.sb200_job_lengths(self._h, f, s, o) != 0:
            raise RuntimeError("job has not run")
        return list(f), list(s), list(o)

    def debug_fetch(self, name: str, b: int = 0) -> np.ndarray:
        data = C.POINTER(C.c_float)()
        rows, cols = C.c_size_t(), C.c_size_t()
        err = N.sb200_error()
        _check(self._lib.sb200_job_debug_fetch(self._h, name.encode(), b, C.byref(data), C.byref(rows),
                                               C.byref(cols), C.byref(err)), err)
        out = np.ctypeslib.as_array(data, shape=(rows.value, cols.value)).copy()
        self._lib.sb200_buffer_free(data)
        return out

    def durations(self, b: int = 0) -> np.ndarray:
        cum = C.POINTER(C.c_int32)()
        n = C.c_size_t()
        err = N.sb200_error()
        _check(self._lib.sb200_job_debug_durations(self._h, b, C.byref(cum), C.byref(n), C.byref(err)), err)
        out = np.ctypeslib.as_array(cum, shape=(n.value,)).copy()
        self._lib.sb200_buffer_free(C.cast(cum, C.POINTER(C.c_float)))
        return out

    def profile(self) -> List[dict]:
        st = (N.sb200_region_stat * 64)()
        k = self._lib.sb200_job_profile(self._h, st, 64)
        return [dict(name=st[i].name.decode(), ms=st[i].ms, flops=st[i].flops, bytes=st[i].bytes,
                     launches=st[i].launches) for i in range(k)]

    def close(self):
        if self._h:
            self._lib.sb200_job_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
