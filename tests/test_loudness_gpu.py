"""GPU (-m gpu): loudness normalisation measured and applied on the device.

The kernel's integrated loudness against the float64 reference meter (known answers, gate edges, lengths), synthesised
audio of every voice quality at every output rate (measurement, gain, scaled samples, re-measured loudness), jobs
without targets unchanged, an utterance in a mixed C2-sized batch equal to itself alone, the i16 paths at the fixed
scale, and the frontends."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import loudness_reference as lr
import sonata_b200
from sonata_b200 import PiperSynthesisConfig, cli, voicegen, workload
from sonata_b200 import _native as N
from sonata_b200.core import AudioSamples
from sonata_b200.job import SynthesisJob
from sonata_b200.piper import _loudness_array
from sonata_b200.synth import SonataSpeechSynthesizer

pytestmark = pytest.mark.gpu

DEFAULT = PiperSynthesisConfig(None, 0.667, 1.0, 0.8)
TOL_LU = 1e-6


@pytest.fixture(scope="module")
def voices(lib_built):
    d = voicegen.default_voice_dir()
    paths = {q: voicegen.write_voice(d, q) for q in ("medium", "high", "low", "x_low")}
    paths["medium4"] = voicegen.write_voice(d, "medium", n_speakers=4)
    ms = {}

    def get(q):
        if q not in ms:
            ms[q] = sonata_b200.from_config_path(paths[q], device=0)
            ms[q].set_fallback_synthesis_config(DEFAULT)
        return ms[q]
    get.paths = paths
    yield get
    for m in ms.values():
        m.close()


def _ids(n, utt):
    return list(workload.synthetic_ids(n, utt=utt))


def _measure(x, rate):
    x = np.ascontiguousarray(x, np.float32)
    out = C.c_double()
    err = N.sb200_error()
    rc = N.lib().sb200_debug_loudness(0, x.ctypes.data_as(C.POINTER(C.c_float)), x.size, rate, C.byref(out),
                                      C.byref(err))
    assert rc == 0
    return out.value


def _close(got, ref):
    if ref == -math.inf:
        return got == -math.inf
    return abs(got - ref) <= TOL_LU


def _run(m, batches, seeds, rates=None, targets=None, configs=None):
    job = SynthesisJob(m, batches, seeds=seeds, output_rates=rates, loudness=targets, configs=configs)
    n0 = N.lib().sb200_launch_count()
    job.run()
    launches = N.lib().sb200_launch_count() - n0
    audio = job.fetch()
    out = dict(wav=[a.samples.as_slice().copy() for a in audio], sr=[a.info.sample_rate for a in audio],
               i16=job.fetch_i16(), profile=job.profile(), launches=launches)
    total = sum(len(w) for w in out["wav"])
    i16 = np.zeros(total, np.int16)
    assert job.copy_out(i16.ctypes.data, i16.nbytes, 1) == i16.nbytes
    out["i16_copy"] = i16
    out["offs"] = job.lengths()[2]
    out["loud"] = job.loudness() if _loudness_array(targets, len(batches)) is not None else None
    job.close()
    return out


@pytest.mark.parametrize("rate", lr.RATES)
def test_known_answers(lib_built, rate):
    x = lr.sine(rate, 5.0)
    got = _measure(x, rate)
    assert abs(got + 23.01) <= 0.1
    assert _close(got, lr.integrated(x, rate))
    S = lr.step(rate)
    assert _measure(np.zeros(rate, np.float32), rate) == -math.inf
    assert _measure(x[:4 * S - 1], rate) == -math.inf
    assert _measure(lr.sine(rate, 1.0, peak=1e-4), rate) == -math.inf
    for n in (4 * S, 4 * S + 1, 7 * S - 1, 7 * S, 7 * S + 1, 23 * S - 1, 23 * S + 1):
        assert _close(_measure(x[:n], rate), lr.integrated(x[:n], rate)), n
    loud, quiet = lr.sine(rate, 2.0, peak=0.1 * 10 ** 0.15), lr.sine(rate, 2.0, peak=0.1 * 10 ** -0.85)
    both = np.concatenate([loud, quiet])
    assert _close(_measure(both, rate), lr.integrated(both, rate))
    noise = (np.random.default_rng(rate).standard_normal(3 * rate) * 0.05).astype(np.float32)
    assert _close(_measure(noise, rate), lr.integrated(noise, rate))


@pytest.mark.parametrize("quality", ["medium", "high", "low", "x_low"])
def test_synthesised_audio(voices, quality):
    m = voices(quality)
    vr = m.audio_output_info().sample_rate
    rates = [None] + list(lr.RATES)
    B = len(rates)
    batches = [_ids(12 + 5 * b, 40 + b) for b in range(B)]
    seeds = [500 + b for b in range(B)]
    targets = [(-30.0, -23.0, -16.0, -9.0)[b % 4] for b in range(B)]
    targets[3] = None
    base = _run(m, batches, seeds, rates)
    got = _run(m, batches, seeds, rates, targets)
    lufs, gains = got["loud"]
    assert [r["name"] for r in got["profile"]].count("loudness") == 1
    assert got["launches"] == base["launches"] + 1
    for b in range(B):
        x, y, rate = base["wav"][b], got["wav"][b], base["sr"][b]
        assert rate == (rates[b] or vr) and got["sr"][b] == rate
        L = lr.integrated(x, rate)
        assert _close(lufs[b], L), (quality, b, lufs[b], L)
        if targets[b] is None:
            assert gains[b] == 1.0
            np.testing.assert_array_equal(y, x)
            np.testing.assert_array_equal(got["i16"][b], AudioSamples(y).to_i16_vec())
            continue
        g = lr.gain(x, targets[b], L)
        assert abs(float(gains[b]) - float(g)) <= float(np.spacing(g)), (quality, b, gains[b], g)
        np.testing.assert_array_equal(y, x * gains[b])
        assert float(np.max(np.abs(y))) <= 1.0
        peak = float(np.max(np.abs(x)))
        if L > -math.inf and 10 ** ((targets[b] - L) / 20) < 1 / peak:
            assert abs(lr.integrated(y, rate) - targets[b]) < 0.01
        fixed = AudioSamples(y).to_i16_fixed()
        np.testing.assert_array_equal(got["i16"][b], fixed)
        o = got["offs"][b]
        np.testing.assert_array_equal(got["i16_copy"][o:o + len(y)], fixed)


def test_no_targets_change_nothing(voices):
    m = voices("medium")
    batches = [_ids(30, 3), _ids(9, 4), _ids(14, 5)]
    base = _run(m, batches, [1, 2, 3], [0, 48000, 8000])
    for t in ([None, None, None], [float("nan")] * 3):
        same = _run(m, batches, [1, 2, 3], [0, 48000, 8000], t)
        for key in ("wav", "i16"):
            for a, b in zip(base[key], same[key]):
                np.testing.assert_array_equal(a, b)
        np.testing.assert_array_equal(base["i16_copy"], same["i16_copy"])
        assert same["launches"] == base["launches"]
        assert [r["name"] for r in same["profile"]] == [r["name"] for r in base["profile"]]
        assert not any(r["name"] == "loudness" for r in same["profile"])
    # a job whose targets are switched off again, and its results before a run with targets
    job = SynthesisJob(m, batches, seeds=[1, 2, 3], output_rates=[0, 48000, 8000], loudness=[-20, None, -20])
    job.set_loudness(None)
    job.run()
    for a, b in zip(base["wav"], job.fetch()):
        np.testing.assert_array_equal(a, b.samples.as_slice())
    with pytest.raises(sonata_b200.OperationError, match="no loudness"):
        job.loudness()
    job.close()


def test_bad_targets_leave_the_job_as_it_was(voices):
    m = voices("medium")
    batches = [_ids(20, 6), _ids(21, 7)]
    job = SynthesisJob(m, batches, seeds=[6, 7], loudness=[-20, None])
    bad = np.array([-20, 5], np.float32)
    err = N.sb200_error()
    rc = m._lib.sb200_job_set_loudness(job._h, bad.ctypes.data_as(C.POINTER(C.c_float)), C.byref(err))
    assert rc == 19
    msg = C.string_at(err.message).decode()
    N.lib().sb200_string_free(err.message)
    assert "utterance 1" in msg
    job.run()
    lufs, gains = job.loudness()
    assert gains[1] == 1.0 and np.isfinite(lufs).all()
    job.close()


@pytest.mark.parametrize("size", ["small", "c2"])
def test_mixed_batch_equals_alone(voices, size):
    m = voices("medium4")
    B, n = (6, 24) if size == "small" else (32, 256)
    batches = [_ids(n - 3 * (b % 5), 200 + b) for b in range(B)]
    rates = [(0, 8000, 48000, 22050, 11025, 44100, 24000, 16000, 32000)[b % 9] for b in range(B)]
    targets = [(None, -23.0, -16.0, -30.0, -9.0, -45.0, -1.0)[b % 7] for b in range(B)]
    configs = [PiperSynthesisConfig(b % 4, 0.667, 1.0, 0.8) for b in range(B)]
    seeds = [3000 + b for b in range(B)]
    mixed = _run(m, batches, seeds, rates, targets, configs)
    for b in range(B):
        alone = _run(m, [batches[b]], [seeds[b]], [rates[b]], [targets[b]], [configs[b]])
        np.testing.assert_array_equal(mixed["wav"][b], alone["wav"][0])
        np.testing.assert_array_equal(mixed["i16"][b], alone["i16"][0])
        if targets[b] is not None:
            assert mixed["loud"][0][b] == alone["loud"][0][0]
            assert mixed["loud"][1][b] == alone["loud"][1][0]


def test_frontends_match_the_job_path(voices, tmp_path):
    import wave
    m = voices("medium")
    phs = ["hɛloʊ wɜːld ðɪs ɪz ə lɔŋɡɚ sɛntəns", "ænd ə sɛkənd wʌn"]
    ids = [m.phonemes_to_input_ids(p) for p in phs]
    job = _run(m, ids, [5, 6], None, [-20.0, -20.0])
    sb = m.speak_batch(phs, seeds=[5, 6], loudness=[-20.0, -20.0])
    for a, w in zip(sb, job["wav"]):
        np.testing.assert_array_equal(a.samples.as_slice(), w)
    al = m.speak_batch_with_alignment(phs, seeds=[5, 6], loudness=[-20.0, -20.0])
    plain = m.speak_batch_with_alignment(phs, seeds=[5, 6])
    for (a, x), (_, y), w in zip(al, plain, job["wav"]):
        np.testing.assert_array_equal(a.samples.as_slice(), w)
        assert [(p.start_sample, p.num_samples) for p in x] == [(p.start_sample, p.num_samples) for p in y]
    synth = SonataSpeechSynthesizer(m)
    par = list(synth.synthesize_parallel("\n".join(phs), seed=5, loudness=-20.0))
    lazy = list(synth.synthesize_lazy("\n".join(phs), seed=5, loudness=-20.0))
    for a, c, w in zip(par, lazy, job["wav"]):
        np.testing.assert_array_equal(a.samples.as_slice(), w)
        np.testing.assert_array_equal(c.samples.as_slice(), w)
    f = tmp_path / "s.wav"
    synth.synthesize_to_file(f, "\n".join(phs), seed=5, loudness=-20.0)
    with wave.open(str(f)) as r:
        data = np.frombuffer(r.readframes(r.getnframes()), "<i2")
    np.testing.assert_array_equal(data, AudioSamples(np.concatenate(job["wav"])).to_i16_fixed())
    m.set_fallback_synthesis_config(DEFAULT)
    (tmp_path / "in.txt").write_text("\n".join(phs) + "\n", encoding="utf-8")
    out = tmp_path / "c.wav"
    assert cli.main([voices.paths["medium"], "-f", str(tmp_path / "in.txt"), "-o", str(out), "--loudness", "-20",
                     "--seed", "5"]) == 0
    with wave.open(str(out)) as r:
        np.testing.assert_array_equal(np.frombuffer(r.readframes(r.getnframes()), "<i2"), data)
    m.set_fallback_synthesis_config(DEFAULT)
