"""Low-level view of one batched synthesis pass (the `sb200_job_*` entry points): used by
bench.py (device-resident timing, NCCL send buffers) and by the parity tests (noise injection,
per-stage intermediates).  Ordinary callers use `VitsModel.speak_*`."""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _native as N
from .core import G711_LAW, Audio, OperationError, check_encoding
from .piper import (_batch_options, _blend_arrays, _break_arrays, _check, _config_array, _contour_arrays, _duration_arrays,
                    _formant_array, _gain_array, _loudness_array, _pack_ids, _prosody_arrays, _ptr, _rate_array,
                    _seed_arrays, _take_audio, _take_bytes, _volume_arrays, _target_arrays, _target_images,
                    _check_target_list)


class SynthesisJob:
    def __init__(self, model, batches: Sequence[Sequence[int]], eps_w: Optional[Sequence] = None,
                 eps_z: Optional[Sequence] = None, debug: bool = False, configs: Optional[Sequence] = None,
                 seeds: Optional[Sequence] = None, output_rates: Optional[Sequence] = None,
                 loudness: Optional[Sequence] = None, pitches: Optional[Sequence] = None,
                 tempos: Optional[Sequence] = None, pitch_contours: Optional[Sequence] = None,
                 formants: Optional[Sequence] = None, speaker_blends: Optional[Sequence] = None,
                 volume_contours: Optional[Sequence] = None, breaks: Optional[Sequence] = None,
                 target_durations: Optional[Sequence] = None):
        """`configs`: one PiperSynthesisConfig per utterance (see set_configs); None keeps the voice's fallback config.
        `seeds`: noise seeds (see set_seeds).  `output_rates`: output sample rates (see set_output_rates).
        `loudness`: loudness targets (see set_loudness).  `pitches` / `tempos`: pitch and tempo ratios (see
        set_prosody).  `pitch_contours`: per-id pitch ratios (see set_pitch_contours).  `formants`: formant ratios (see
        set_formants).  `speaker_blends`: speaker blends (see set_speaker_blends).  `volume_contours`: per-id volume
        levels (see set_volume_contours).  `breaks`: per-id pauses (see set_breaks).  `target_durations`: target
        durations (see set_target_durations)."""
        # argument errors before the job exists
        options = _batch_options(model, len(batches), [len(b) for b in batches], configs, seeds=seeds,
                                 output_rates=output_rates, loudness=loudness, pitches=pitches, tempos=tempos,
                                 pitch_contours=pitch_contours, formants=formants, speaker_blends=speaker_blends,
                                 volume_contours=volume_contours, breaks=breaks, target_durations=target_durations)
        self._open(model, batches, options, eps_w, eps_z, debug)

    @classmethod
    def _of(cls, model, batches: Sequence[Sequence[int]], options) -> "SynthesisJob":
        """A job of `batches` with options already checked by piper._batch_options."""
        job = cls.__new__(cls)
        job._open(model, batches, options)
        return job

    def _open(self, model, batches, o, eps_w=None, eps_z=None, debug: bool = False) -> None:
        """Creates the job and sets the checked images of options `o`, in the order the library's batch entry points
        set them; what o does not ask for keeps the new job's default."""
        self._m = model
        self._lib = model._lib
        n = len(batches)
        self.batch = n
        self._lens = [len(b) for b in batches]
        packed, offs = _pack_ids(batches)
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
        lib = self._lib
        if o.cfgs is not None:
            self._set(lib.sb200_job_set_configs, o.cfgs)
        if o.scales is not None or o.frames is not None:
            self._set(lib.sb200_job_set_durations, _ptr(o.scales, C.c_float), _ptr(o.frames, C.c_int32))
        if o.seeds is not None:
            self._set(lib.sb200_job_set_seeds, _ptr(o.seeds, C.c_uint64), _ptr(o.seeded, C.c_int32))
        if o.rates is not None:
            self._set(lib.sb200_job_set_output_rates, _ptr(o.rates, C.c_uint32))
        if o.loudness is not None:
            self._set(lib.sb200_job_set_loudness, _ptr(o.loudness, C.c_float))
        if o.pitch is not None or o.tempo is not None:
            self._set(lib.sb200_job_set_prosody, _ptr(o.pitch, C.c_float), _ptr(o.tempo, C.c_float))
        if o.contour is not None:
            self._set(lib.sb200_job_set_pitch_contour, _ptr(o.contour, C.c_float))
        if o.formants is not None:
            self._set(lib.sb200_job_set_formants, _ptr(o.formants, C.c_float))
        if o.blend_offsets is not None:
            self._set(lib.sb200_job_set_speaker_blends, _ptr(o.blend_speakers, C.c_int64),
                      _ptr(o.blend_weights, C.c_float), _ptr(o.blend_offsets, C.c_size_t))
        if o.volume is not None:
            self._set(lib.sb200_job_set_volume_contour, _ptr(o.volume, C.c_float))
        if o.breaks is not None:
            self._set(lib.sb200_job_set_breaks, _ptr(o.breaks, C.c_float))
        if o.targets is not None:
            self._set(lib.sb200_job_set_targets, *_target_images(o.targets))
        self._spans = None if o.targets is None else [int(x) for x in o.targets[3]]

    def _set(self, fn, *images) -> None:
        """One sb200_job_set_* call with its C images."""
        err = N.sb200_error()
        _check(fn(self._h, *images, C.byref(err)), err)

    def set_configs(self, configs: Optional[Sequence]) -> None:
        """Per-utterance PiperSynthesisConfigs for the next run, or None for the voice's fallback config.  A wrong
        length or an unknown speaker raises OperationError and leaves the job's configs as they were."""
        self._set(self._lib.sb200_job_set_configs, _config_array(configs, self.batch))

    def set_durations(self, scales: Optional[Sequence] = None, frames: Optional[Sequence] = None) -> None:
        """Per-id duration controls for the next run (see VitsModel.infer_batch_with_durations): scales[b] / frames[b]
        hold one value per id of utterance b, or None.  None and None restores the default.  A bad entry raises
        OperationError naming the utterance and the id, and leaves the job's controls as they were."""
        sc, fr = _duration_arrays(self._lens, scales, frames)
        self._set(self._lib.sb200_job_set_durations, _ptr(sc, C.c_float), _ptr(fr, C.c_int32))

    def set_seeds(self, seeds: Optional[Sequence]) -> None:
        """Per-utterance noise seeds for the next run (see VitsModel.infer_batch_with_values): an int in [0, 2**64) or
        None per utterance; None for the whole list restores positional noise.  With debug on, the run's draws are
        fetchable as "eps_w" and "eps_z".  A bad entry, or seeds on a job with injected noise, raises OperationError
        and leaves the job's seeds as they were."""
        sv, sf = _seed_arrays(seeds, self.batch)
        self._set(self._lib.sb200_job_set_seeds, _ptr(sv, C.c_uint64), _ptr(sf, C.c_int32))

    def set_output_rates(self, rates: Optional[Sequence]) -> None:
        """Per-utterance output sample rates for the next run (see VitsModel.infer_batch_with_values), or None for the
        voice's rate throughout.  After such a run, fetch, fetch_i16, copy_out and the samples and offsets of lengths
        all report the resampled signal.  An unsupported rate raises OperationError naming the utterance and leaves the
        job's rates as they were."""
        self._set(self._lib.sb200_job_set_output_rates, _ptr(_rate_array(rates, self.batch), C.c_uint32))

    def set_loudness(self, targets: Optional[Sequence]) -> None:
        """Per-utterance loudness targets for the next run (see VitsModel.infer_batch_with_values): LUFS in [-70, 0] or
        None per utterance; None for the whole list (or all None) turns loudness off.  A run with targets measures every
        utterance, scales those with a target in place on the device (d_out included), and fetch_i16 / copy_out(fmt=1)
        convert those at the fixed scale 32767 instead of their peak.  A bad entry raises OperationError naming the
        utterance and leaves the job's targets as they were."""
        self._set(self._lib.sb200_job_set_loudness, _ptr(_loudness_array(targets, self.batch), C.c_float))

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
        self._set(self._lib.sb200_job_set_prosody, _ptr(p, C.c_float), _ptr(t, C.c_float))

    def prosody(self) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """(stretched length n1, delivered length before any output-rate resampling n2, WSOLA frames F) per utterance of
        the last run, which must have had ratios."""
        n1, n2 = np.zeros(self.batch, np.int64), np.zeros(self.batch, np.int64)
        frames = np.zeros(self.batch, np.int32)
        err = N.sb200_error()
        _check(self._lib.sb200_job_prosody(self._h, _ptr(n1, C.c_int64), _ptr(n2, C.c_int64), _ptr(frames, C.c_int32),
                                           C.byref(err)), err)
        return n1, n2, frames

    def set_pitch_contours(self, contours: Optional[Sequence]) -> None:
        """Per-id pitch ratios for the next run (see VitsModel.infer_batch_with_values): contours[b] holds one ratio per
        id of utterance b, or is None; None for the whole list, or ratios that are all None / NaN / 1.0, turn contours
        off.  A contour combines with the job's tempos and not with its pitch ratios.  After a run with a contour the
        results report the warped signal, as after set_prosody, and prosody_bounds gives each id's delivered end.  A bad
        entry raises OperationError naming the utterance and the id, and leaves the job's contours as they were."""
        self._set(self._lib.sb200_job_set_pitch_contour, _ptr(_contour_arrays(self._lens, contours), C.c_float))

    def set_formants(self, formants: Optional[Sequence]) -> None:
        """Per-utterance formant ratios for the next run (see VitsModel.infer_batch_with_values), or None for none.  A
        ratio of 1.0 asks for something on an utterance with a pitch ratio or contour: its own formants.  A bad entry
        raises OperationError naming the utterance and leaves the job's ratios as they were."""
        self._set(self._lib.sb200_job_set_formants, _ptr(_formant_array(formants, self.batch), C.c_float))

    def set_volume_contours(self, contours: Optional[Sequence]) -> None:
        """Per-id volume levels in dB for the next run (see VitsModel.infer_batch_with_values): contours[b] holds one
        level per id of utterance b, or is None; None for the whole list, or levels that are all None / NaN / 0, turn
        contours off.  The results keep their lengths and layout, and profile() reports the stage as "volume".  A bad
        entry raises OperationError naming the utterance and the id, and leaves the job's contours as they were."""
        self._set(self._lib.sb200_job_set_volume_contour, _ptr(_volume_arrays(self._lens, contours), C.c_float))

    def set_breaks(self, breaks: Optional[Sequence]) -> None:
        """Per-id pauses in ms for the next run (see VitsModel.infer_batch_with_values): breaks[b] holds one break per
        id of utterance b, or is None; None for the whole list, or breaks that are all None / NaN / 0, turn pauses off.
        The results, their lengths and prosody_bounds count the pauses, and profile() reports the stage as "break".  A
        bad entry raises OperationError naming the utterance and the id, and leaves the job's breaks as they were."""
        self._set(self._lib.sb200_job_set_breaks, _ptr(_break_arrays(self._lens, breaks), C.c_float))

    def set_target_durations(self, targets: Optional[Sequence]) -> None:
        """Target durations for the next run (see VitsModel.infer_batch_with_values): per utterance None, a duration in
        ms for the whole utterance or a list of (first, last, ms) spans of ids; None for the whole list, or entries
        that all ask for nothing, turn fitting off.  A bad entry, or one on an utterance with a tempo ratio, raises
        OperationError naming the utterance and the span, and leaves the job's targets as they were."""
        t = _target_arrays(self._lens, _check_target_list(targets, self.batch, None, self._lens))
        self._set(self._lib.sb200_job_set_targets, *_target_images(t))
        self._spans = None if t is None else [int(x) for x in t[3]]

    def targets(self) -> List[List[Tuple[float, int]]]:
        """Per utterance, each target span's (u, delivered length) of the last run: u the factor its predicted
        durations got, and the span's samples at the voice's rate, breaks included (NaN and -1 for a span that asked
        for nothing).  OperationError when the last run had no targets."""
        if self._spans is None:
            raise OperationError("the job's last run had no target durations")
        n = self._spans[-1]
        u, ln = np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.int64)
        err = N.sb200_error()
        _check(self._lib.sb200_job_targets(self._h, _ptr(u, C.c_float), _ptr(ln, C.c_int64), n, C.byref(err)), err)
        return [[(float(u[k]), int(ln[k])) for k in range(self._spans[b], self._spans[b + 1])]
                for b in range(self.batch)]

    def set_speaker_blends(self, blends: Optional[Sequence]) -> None:
        """Per-utterance speaker blends for the next run (see VitsModel.infer_batch_with_values): a mapping
        {speaker: weight} or None per utterance, or None for none.  A blend replaces the utterance's config speaker.  A
        bad entry raises OperationError naming the utterance and leaves the job's blends as they were."""
        s, w, o = _blend_arrays(self._m, blends, self.batch)
        self._set(self._lib.sb200_job_set_speaker_blends, _ptr(s, C.c_int64), _ptr(w, C.c_float), _ptr(o, C.c_size_t))

    def prosody_bounds(self) -> List[np.ndarray]:
        """Each id's delivered end in the last run, at the voice's rate, one int64 array per utterance (see
        sb200_job_prosody_bounds)."""
        total = int(sum(self._lens))
        out = np.zeros(total, np.int64)
        err = N.sb200_error()
        _check(self._lib.sb200_job_prosody_bounds(self._h, _ptr(out, C.c_int64), total, C.byref(err)), err)
        offs = np.concatenate([[0], np.cumsum(self._lens)]).astype(int)
        return [out[offs[b]:offs[b + 1]].copy() for b in range(self.batch)]

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
        return self._fetch_bytes(self._lib.sb200_job_fetch_g711, G711_LAW[law],
                                 _ptr(_gain_array(gains, self.batch), C.c_float))

    def fetch_flac(self, gains: Optional[Sequence] = None) -> List[bytes]:
        """One complete FLAC stream per utterance (see sb200_job_fetch_flac): lossless, of exactly the 16-bit samples
        fetch_i16 returns after gains[b] (None: 1), at the utterance's delivered rate.  Analysed, laid out and packed on
        the device; only the compressed bytes leave the card."""
        return self._fetch_bytes(self._lib.sb200_job_fetch_flac, _ptr(_gain_array(gains, self.batch), C.c_float))

    def _fetch_bytes(self, fn, *args) -> List[bytes]:
        """One byte buffer per utterance from fetch entry point `fn` (sb200_job_fetch_g711 / _flac) with `args`."""
        outs = (C.POINTER(C.c_uint8) * self.batch)()
        lens = (C.c_size_t * self.batch)()
        err = N.sb200_error()
        _check(fn(self._h, *args, outs, lens, C.byref(err)), err)
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
