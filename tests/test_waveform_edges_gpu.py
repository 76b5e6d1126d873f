"""GPU (-m gpu): the formant, pitch / tempo, resampling and loudness kernels against their float64 specifications at
the length, run and ratio edges of tests/waveform_edges.py (whose host test shows each case reaches its edge): every
sample within the bound the stage's own tests use, and bits where the header promises bits (exact zeros, offsets,
lengths, skipped stages, identity rates, the scaled samples of a loudness target).  Prints, per stage, the worst
|got - ref| / bound."""
import ctypes as C
import math

import numpy as np
import pytest

import waveform_edges as we
from waveform_edges import f32p, fr, i64p, lr, pc, pr, rr

import sonata_b200
from sonata_b200 import PiperSynthesisConfig, voicegen, workload
from sonata_b200 import _native as N
from sonata_b200.job import SynthesisJob

pytestmark = pytest.mark.gpu

DEFAULT = PiperSynthesisConfig(None, 0.667, 1.0, 0.8)
TOL_LU = 1e-6          # test_loudness_gpu.py's tolerance against the reference meter

worst = {}


def _note(stage, ratio):
    worst[stage] = max(worst.get(stage, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for stage, r in sorted(worst.items()):
        print(f"worst |gpu - spec| / bound, {stage}: {r:.6f}")


@pytest.fixture(scope="module")
def voices(lib_built):
    d = voicegen.default_voice_dir()
    paths = {q: voicegen.write_voice(d, q) for q in ("medium", "x_low")}
    ms = {}

    def get(q):
        if q not in ms:
            ms[q] = sonata_b200.from_config_path(paths[q], device=0)
            ms[q].set_fallback_synthesis_config(DEFAULT)
        return ms[q]
    yield get
    for m in ms.values():
        m.close()


def _ids(n, utt):
    return list(workload.synthetic_ids(n, utt=utt))


# ---------------------------------------------------------------- formant stage

def _hold_formant(stage, y, pre, rate, phi, pitch=None, Q=None, P=None, what=()):
    assert len(y) == len(pre), what
    if not fr.asks(len(pre), phi, pitch, Q, P):
        np.testing.assert_array_equal(y, pre, err_msg=str(what))
        return
    ref = fr.apply(pre, rate, phi, pitch, Q, P)
    ratio = float(np.max(np.abs(y.astype(np.float64) - ref) / fr.bound(ref)))
    _note(stage, ratio)
    assert ratio <= 1.0, (what, ratio)
    if not np.any(pre):
        assert not np.any(y), what                          # silence in, exact zeros out


@pytest.mark.parametrize("rate", we.RATES)
def test_formant_batch_kernel(lib_built, rate):
    for n in we.FORMANT_LENGTHS:
        for sname, x in we.signals(n, rate, seed=1).items():
            for name, p, t, phi in we.FORMANT_RATIOS:
                pre, y = we.formant_debug(lib_built, x, rate, phi, pitch=p, tempo=t)
                assert len(pre) == pr.plan(rate, n, p, t)["n2"]
                _hold_formant("formant", y, pre, rate, phi, pitch=p, what=(rate, n, sname, name))


@pytest.mark.parametrize("rate", we.RATES)
def test_formant_batch_kernel_contours(lib_built, rate):
    for n in we.FORMANT_LENGTHS:
        sig = we.signals(n, rate, seed=2)
        for cname, ends, ratios, Q, m, d in we.formant_contours(n):
            pl = pc.plan(rate, n, ends, ratios, None)
            for sname in ("impulse_last", "impulse_hop", "noise", "vowel", "square"):
                for phi in (0.5, 1.0, 2.0):
                    pre, y = we.formant_debug(lib_built, sig[sname], rate, phi, ends=ends, ratios=ratios)
                    assert len(pre) == pl["n2"] == n
                    _hold_formant("formant contour", y, pre, rate, phi, Q=pl["Q"], P=pl["p"],
                                  what=(rate, n, cname, sname, phi))


@pytest.mark.parametrize("quality", ["medium", "x_low"])
def test_formant_job_path(voices, quality):
    """One job, run plain, with its prosody and with prosody and formants: each utterance's formant output is within
    bound of the specification applied to its pre-formant signal from the same job, and the bits of
    sb200_debug_formant over its decoder output."""
    m = voices(quality)
    rate = m.audio_output_info().sample_rate
    table = we.FORMANT_JOB
    B = len(table)
    batches = [_ids(len(frames), 70 + b)[:len(frames)] for b, (frames, *_) in enumerate(table)]     # one id per entry
    frames = [list(f) for f, *_ in table]
    pitches = [p for _, p, *_ in table]
    tempos = [t for _, _, t, *_ in table]
    contours = [c for *_, c, _, _ in table]
    phis = [phi for *_, phi, _ in table]
    job = SynthesisJob(m, batches, seeds=[700 + b for b in range(B)])
    try:
        job.set_durations(None, frames)
        job.run()
        xs = [np.asarray(a.samples.as_slice()).copy() for a in job.fetch()]
        job.set_prosody(pitches, tempos)
        job.set_pitch_contours(contours)
        job.run()
        pres = [np.asarray(a.samples.as_slice()).copy() for a in job.fetch()]
        job.set_formants(phis)
        job.run()
        ys = [np.asarray(a.samples.as_slice()).copy() for a in job.fetch()]
        assert any(r["name"] == "formant" for r in job.profile())
    finally:
        job.close()
    for b, (fr_b, p, t, contour, phi, n2) in enumerate(table):
        x, pre, y = xs[b], pres[b], ys[b]
        assert len(x) == 256 * sum(fr_b)
        assert len(pre) == len(y) == n2, (quality, b, len(y))
        if contour is None:
            Q = P = None
        else:
            pl = pc.plan(rate, len(x), we.job_ends(fr_b), contour, t)
            Q, P = pl["Q"], pl["p"]
        _hold_formant("formant job", y, pre, rate, phi, pitch=p if contour is None else None, Q=Q, P=P,
                      what=(quality, b))
        e, r = (None, None) if contour is None else (we.job_ends(fr_b), contour)
        dpre, dy = we.formant_debug(N.lib(), x, rate, phi, pitch=p, tempo=t, ends=e, ratios=r)
        np.testing.assert_array_equal(dpre, pre)
        np.testing.assert_array_equal(dy, y)


# ---------------------------------------------------------------- resampler

def _resample(lib, x, in_rate, out_rate):
    up, down = rr.ratio(in_rate, out_rate)
    x = np.ascontiguousarray(x, np.float32)
    y = np.full(rr.n_out(len(x), up, down) + 1, np.float32(7.0))      # one sentinel past the end
    err = N.sb200_error()
    rc = lib.sb200_debug_resample(0, f32p(x), x.size, in_rate, out_rate, f32p(y), C.byref(err))
    assert rc == 0, C.string_at(err.message) if err.message else rc
    assert y[-1] == np.float32(7.0)
    return y[:-1]


@pytest.mark.parametrize("in_rate,out_rate", we.RS_PAIRS)
def test_resample_kernel(lib_built, in_rate, out_rate):
    up, down = rr.ratio(in_rate, out_rate)
    for lname, n in we.resample_lengths(in_rate, out_rate):
        for sname, x in we.resample_signals(n, seed=3).items():
            y = _resample(lib_built, x, in_rate, out_rate)
            assert len(y) == rr.n_out(n, up, down)
            if sname == "silence":
                assert not np.any(y)
                continue
            ref = rr.resample64(x, up, down)
            tol = rr.bound(x, up, down)
            err = np.abs(y.astype(np.float64) - ref)
            ratio = float(np.max(np.where(tol > 0, err / np.where(tol > 0, tol, 1.0), np.where(err > 0, np.inf, 0.0))))
            _note("resample", ratio)
            assert ratio <= 1.0, (lname, n, sname, ratio)


def test_resample_identity_rates_copy_bits(voices):
    """The two identity pairs: the hook refuses them (no ratio), and a job asked for its voice's own rate copies its
    samples bit for bit."""
    err = N.sb200_error()
    x = np.ones(8, np.float32)
    y = np.zeros(8, np.float32)
    for rate in we.RATES:
        assert N.lib().sb200_debug_resample(0, f32p(x), 8, rate, rate, f32p(y), C.byref(err)) == 19
        N.lib().sb200_string_free(err.message)
    for quality in ("medium", "x_low"):
        m = voices(quality)
        rate = m.audio_output_info().sample_rate
        batches = [_ids(9, 80), _ids(3, 81)]
        plain = m.infer_batch_with_values(batches, seeds=[1, 2])
        same = m.infer_batch_with_values(batches, seeds=[1, 2], output_rates=[rate, rate])
        for a, b in zip(plain, same):
            assert b.info.sample_rate == rate
            np.testing.assert_array_equal(np.asarray(a.samples.as_slice()), np.asarray(b.samples.as_slice()))


# ---------------------------------------------------------------- loudness

def _measure(lib, x, rate):
    x = np.ascontiguousarray(x, np.float32)
    out = C.c_double()
    err = N.sb200_error()
    rc = lib.sb200_debug_loudness(0, f32p(x), x.size, rate, C.byref(out), C.byref(err))
    assert rc == 0, C.string_at(err.message) if err.message else rc
    return out.value


@pytest.mark.parametrize("rate", lr.RATES)
def test_loudness_kernel(lib_built, rate):
    for lname, n in we.loudness_lengths(rate):
        for sname, x in (("level_step", we.level_step(rate, n)), ("at_-70", we.at_absolute_gate(rate, n))):
            got, ref = _measure(lib_built, x, rate), lr.integrated(x, rate)
            assert math.isfinite(ref)
            _note("loudness (LU / 1e-6)", abs(got - ref) / TOL_LU)
            assert abs(got - ref) <= TOL_LU, (lname, sname, got, ref)


def test_loudness_peak_limited_gain(voices):
    """Targets the peak limit must cap: g is min(10^((T - L) / 20), 1 / peak) rounded to f32 and stepped down while
    f32(peak g) > 1, so f32(peak g) <= 1, and either g is f32(1 / peak) or one ulp more breaks the limit; the
    delivered samples are the unscaled ones times g, bit for bit."""
    m = voices("medium")
    batches = [_ids(20, 90), _ids(31, 91), _ids(12, 92)]
    seeds = [9, 10, 11]
    plain = m.infer_batch_with_values(batches, seeds=seeds, output_rates=[0, 48000, 8000])
    job = SynthesisJob(m, batches, seeds=seeds, output_rates=[0, 48000, 8000], loudness=[0.0, -1.0, 0.0])
    try:
        job.run()
        got = [np.asarray(a.samples.as_slice()).copy() for a in job.fetch()]
        lufs, gains = job.loudness()
    finally:
        job.close()
    for b, a in enumerate(plain):
        x = np.asarray(a.samples.as_slice())
        peak = np.float32(np.max(np.abs(x)))
        g = np.float32(gains[b])
        T = (0.0, -1.0, 0.0)[b]
        assert abs(lufs[b] - lr.integrated(x, a.info.sample_rate)) <= TOL_LU
        assert 10 ** ((T - lufs[b]) / 20) > 1 / float(peak), b          # the cap decides
        assert np.float32(peak * g) <= 1.0
        assert g == np.float32(1.0 / float(peak)) or np.float32(peak * np.nextafter(g, np.float32(np.inf))) > 1.0
        spec = np.float32(min(10 ** ((T - lufs[b]) / 20), 1.0 / float(peak)))
        while np.float32(peak * spec) > 1.0:
            spec = np.nextafter(spec, np.float32(0))
        assert g == spec, (b, g, spec)
        np.testing.assert_array_equal(got[b], x * g)


# ---------------------------------------------------------------- pitch / tempo

def _prosody(lib, x, rate, p, t):
    x = np.ascontiguousarray(x, np.float32)
    pl = pr.plan(rate, len(x), p, t)
    y = np.zeros(pl["n2"] + 1, np.float32)
    off = np.zeros(pl["F"] + 1, np.int32)
    s = np.zeros(pl["n1"] + 1, np.float32)
    err = N.sb200_error()
    rc = lib.sb200_debug_prosody(0, f32p(x), x.size, rate, we._nan(p), we._nan(t), f32p(y), y.size,
                                 off.ctypes.data_as(C.POINTER(C.c_int32)), off.size, f32p(s), s.size, C.byref(err))
    assert rc == 0, C.string_at(err.message) if err.message else rc
    return y[:pl["n2"]], off[:pl["F"]], (s[:pl["n1"]] if pl["stretch"] else None), pl


def _prosody_contour(lib, x, rate, ends, ratios, t):
    x = np.ascontiguousarray(x, np.float32)
    e = np.ascontiguousarray(ends, np.int64)
    r = np.ascontiguousarray(ratios, np.float32)
    pl = pc.plan(rate, len(x), e, r, t)
    y = np.zeros(pl["n2"] + 1, np.float32)
    off = np.zeros(pl["F"] + 1, np.int32)
    s = np.zeros(pl["n1"] + 1, np.float32)
    err = N.sb200_error()
    rc = lib.sb200_debug_prosody_contour(0, f32p(x), x.size, rate, i64p(e), f32p(r), len(e), we._nan(t), f32p(y),
                                         y.size, off.ctypes.data_as(C.POINTER(C.c_int32)), off.size, f32p(s), s.size,
                                         C.byref(err))
    assert rc == 0, C.string_at(err.message) if err.message else rc
    return y[:pl["n2"]], off[:pl["F"]], s[:pl["n1"]], pl


def _hold_prosody(stage, x, y, off, s, pl, pitch_resample, what):
    """Offsets exactly, the stretched signal within ola_bound and the output within pitch_bound of the resampler over
    the device's own stretched signal; the stages that do not run keep bits."""
    assert len(y) == pl["n2"], what
    cur = np.asarray(x, np.float64)
    if pl["stretch"]:
        np.testing.assert_array_equal(off, pr.offsets(x, pl), err_msg=str(what))
        ref, bound = pr.overlap_add(x, pl, off.astype(np.int64))
        if len(ref):
            r = float(np.max(np.abs(s - ref) / np.maximum(bound, np.finfo(np.float64).tiny)))
            assert np.all(np.abs(s - ref) <= bound), (what, r)
            _note(stage + " ola", r if np.isfinite(r) else 0.0)
        cur = s.astype(np.float64)
        if not pl["pitch"]:
            np.testing.assert_array_equal(y, s, err_msg=str(what))
    if pl["pitch"]:
        ref, bound = pitch_resample(cur, pl)
        if len(ref):
            r = float(np.max(np.abs(y - ref) / bound))
            _note(stage + " pitch", r)
            assert r <= 1.0, (what, r)
    if not pl["stretch"] and not pl["pitch"]:
        np.testing.assert_array_equal(y, x, err_msg=str(what))
    if not np.any(x):
        assert not np.any(y), what


@pytest.mark.parametrize("rate", we.RATES)
def test_prosody_kernels(lib_built, rate):
    for cname, p, t in we.PROSODY_CORNERS:
        for lname, n in we.prosody_lengths(rate, p, t):
            for sname, x in we.signals(n, rate, seed=4, loud=True).items():
                # not the f32 denormal: the overlap-add's f32 products of it round at an absolute 2^-150, where no f32
                # evaluation can meet ola_bound's relative 2^-22 (the formant stage, double inside, does take it)
                if sname == "denormal":
                    continue
                y, off, s, pl = _prosody(lib_built, x, rate, p, t)
                _hold_prosody("prosody", x, y, off, s, pl, pr.pitch_resample, (rate, cname, lname, n, sname))


@pytest.mark.parametrize("rate", we.RATES)
def test_prosody_contour_kernels(lib_built, rate):
    Hs = rate // 100
    for n in (Hs + 1, 2 * Hs + 1, 3 * Hs + 7):
        sig = we.signals(n, rate, seed=5, loud=True)
        for cname, ends, ratios in we.prosody_contours(n, rate):
            for t in (None, 0.25, 4.0):
                for sname in ("impulse_first", "impulse_last", "noise", "vowel", "loud", "tied", "silence"):
                    y, off, s, pl = _prosody_contour(lib_built, sig[sname], rate, ends, ratios, t)
                    assert pl["one"] is None
                    _hold_prosody("contour", sig[sname], y, off, s, pl, pc.pitch_resample,
                                  (rate, n, cname, t, sname))
