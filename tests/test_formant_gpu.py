"""GPU (-m gpu): the formant stage on the device against its float64 specification (tests/formant_reference.py),
applied to the device's own pre-formant signal; bit-for-bit checks of batches, skipped utterances and the one-shot
call against the job path; and its composition with the output stage."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import flac_reference as flr
import formant_reference as fr
import loudness_reference as lr
import prosody_contour_reference as pc
import sonata_b200
from sonata_b200 import PiperSynthesisConfig, voicegen, workload
from sonata_b200 import _native as N
from sonata_b200.core import AudioSamples
from sonata_b200.job import SynthesisJob

pytestmark = pytest.mark.gpu

DEFAULT = PiperSynthesisConfig(None, 0.667, 1.0, 0.8)
NAN = float("nan")
f32p = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
i64p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))


@pytest.fixture(scope="module")
def voices(lib_built):
    d = voicegen.default_voice_dir()
    paths = {q: voicegen.write_voice(d, q) for q in ("medium", "high", "low", "x_low")}
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


def _debug(x, rate, phi, pitch=NAN, tempo=NAN, ends=None, ratios=None):
    x = np.ascontiguousarray(x, np.float32)
    cap = 3 * len(x) + 4096
    pre, y = np.zeros(cap, np.float32), np.zeros(cap, np.float32)
    n2 = C.c_int64()
    err = N.sb200_error()
    e = None if ends is None else np.ascontiguousarray(ends, np.int64)
    r = None if ratios is None else np.ascontiguousarray(ratios, np.float32)
    rc = N.lib().sb200_debug_formant(0, f32p(x), len(x), rate, pitch, tempo, None if e is None else i64p(e),
                                     None if r is None else f32p(r), 0 if e is None else len(e), phi, f32p(pre),
                                     f32p(y), cap, C.byref(n2), C.byref(err))
    assert rc == 0, err.message
    return pre[:n2.value], y[:n2.value]


worst = {"ratio": 0.0}


def _hold(y, pre, rate, phi, pitch=None, Q=None, P=None):
    ref = fr.apply(pre, rate, phi, pitch, Q, P)
    ratio = float(np.max(np.abs(y.astype(np.float64) - ref) / fr.bound(ref)))
    worst["ratio"] = max(worst["ratio"], ratio)
    assert ratio <= 1.0, ratio


@pytest.mark.parametrize("tempo", [NAN, 1.3])
def test_vowel_grid(lib_built, tempo):
    rate = 22050
    x = fr.vowel(rate, seconds=0.6)
    for p in (0.5, 0.8, 1.0, 1.25, 2.0):
        for phi in (0.5, 0.8, 1.0, 1.25, 2.0):
            pre, y = _debug(x, rate, phi, pitch=p if p != 1.0 else NAN, tempo=tempo)
            if not fr.asks(len(pre), phi, pitch=p):
                np.testing.assert_array_equal(y, pre)
                continue
            _hold(y, pre, rate, phi, pitch=p)
    print("worst |gpu - spec| / bound:", worst["ratio"])


def test_vowel_question_contour(lib_built):
    rate = 22050
    x = fr.vowel(rate, seconds=0.8)
    n = len(x)
    ends = np.linspace(0, n, 9)[1:].astype(np.int64)
    ratios = np.array([1, 1, 1, 1, 1, 1.1, 1.2, 1.3], np.float32)
    for tempo in (NAN, 0.8):
        pre, y = _debug(x, rate, 1.0, tempo=tempo, ends=ends, ratios=ratios)
        pl = pc.plan(rate, n, ends, ratios, None if np.isnan(tempo) else tempo)
        assert len(pre) == pl["n2"]
        _hold(y, pre, rate, 1.0, Q=pl["Q"], P=pl["p"])


@pytest.mark.parametrize("quality", ["medium", "high", "low", "x_low"])
def test_voices_against_spec(voices, quality):
    m = voices(quality)
    rate = m.audio_output_info().sample_rate
    batches = [_ids(40, 900), _ids(28, 901), _ids(33, 902)]
    seeds = [11, 12, 13]
    pitches = [1.25, None, 0.8]
    formants = [1.0, 1.2, 0.9]
    plain = m.infer_batch_with_values(batches, seeds=seeds, pitches=pitches)
    got = m.infer_batch_with_values(batches, seeds=seeds, pitches=pitches, formants=formants)
    for a, b, p, phi in zip(plain, got, pitches, formants):
        pre, y = a.samples.as_slice(), b.samples.as_slice()
        assert len(pre) == len(y) and b.info.sample_rate == rate
        _hold(np.asarray(y), np.asarray(pre), rate, phi, pitch=p)


def _run(m, batches, seeds, keep=False, **kw):
    job = SynthesisJob(m, batches, seeds=seeds, **kw)
    n0 = N.lib().sb200_launch_count()
    job.run()
    launches = N.lib().sb200_launch_count() - n0
    r = dict(wav=[np.asarray(a.samples.as_slice()).copy() for a in job.fetch()], launches=launches,
             profile=job.profile(), i16=job.fetch_i16(), job=job)
    if not keep:
        job.close()
    return r


def test_mixed_batch_equals_alone_and_skips_keep_bits(voices):
    m = voices("medium")
    batches = [_ids(30 + 3 * b, 950 + b) for b in range(5)]
    seeds = [300 + b for b in range(5)]
    pitches = [None, 1.25, 1.25, None, 0.8]
    tempos = [None, None, 1.4, 1.2, None]
    formants = [1.2, 1.0, NAN, None, 0.8]       # the last one equals its pitch ratio: skipped
    got = _run(m, batches, seeds, pitches=pitches, tempos=tempos, formants=formants)
    assert any(r["name"] == "formant" for r in got["profile"])
    for b in range(5):
        alone = _run(m, [batches[b]], [seeds[b]], pitches=[pitches[b]], tempos=[tempos[b]], formants=[formants[b]])
        np.testing.assert_array_equal(got["wav"][b], alone["wav"][0])
    base = _run(m, batches, seeds, pitches=pitches, tempos=tempos)
    for kw in ({}, {"formants": [NAN] * 5}, {"formants": [None, 1.25, None, None, 0.8]}):
        r = _run(m, batches, seeds, pitches=pitches, tempos=tempos, **kw)
        assert r["launches"] == base["launches"]
        assert not any(p["name"] == "formant" for p in r["profile"])
        for a, b in zip(r["wav"], base["wav"]):
            np.testing.assert_array_equal(a, b)
    assert got["launches"] == base["launches"] + 1
    for b in (3, 4):
        np.testing.assert_array_equal(got["wav"][b], base["wav"][b])


def test_one_shot_equals_job_and_composition(voices):
    m = voices("medium")
    batches = [_ids(35, 990), _ids(29, 991)]
    seeds = [21, 22]
    kw = dict(pitches=[1.25, None], formants=[1.0, 1.15])
    job = _run(m, batches, seeds, **kw)
    one = m.infer_batch_with_values(batches, seeds=seeds, **kw)
    for a, b in zip(job["wav"], one):
        np.testing.assert_array_equal(a, np.asarray(b.samples.as_slice()))
    # lengths, frame counts and alignments do not change; the output stage runs on the formant stage's output
    plain = m.infer_batch_with_durations(batches, seeds=seeds, pitches=kw["pitches"])
    got = m.infer_batch_with_durations(batches, seeds=seeds, **kw)
    for (a, fa), (b, fb) in zip(plain, got):
        assert len(a.samples.as_slice()) == len(b.samples.as_slice())
        np.testing.assert_array_equal(fa, fb)
    rates = m.infer_batch_with_values(batches, seeds=seeds, output_rates=[16000, 16000], loudness=[-20, None], **kw)
    plain_rates = m.infer_batch_with_values(batches, seeds=seeds, output_rates=[16000, 16000], loudness=[-20, None],
                                            pitches=kw["pitches"])
    for a, b in zip(rates, plain_rates):
        assert a.info.sample_rate == 16000 and len(a.samples.as_slice()) == len(b.samples.as_slice())
        assert not np.array_equal(np.asarray(a.samples.as_slice()), np.asarray(b.samples.as_slice()))
    assert [len(x) for x in job["i16"]] == [len(x) for x in job["wav"]]
    phs = ["həlˈoʊ wˈɜːld", "ðɪs ɪz ɐ tˈɛst"]
    al0 = m.speak_batch_with_alignment(phs, seeds=seeds, pitches=kw["pitches"])
    al1 = m.speak_batch_with_alignment(phs, seeds=seeds, **kw)
    for (a, x), (b, y) in zip(al0, al1):
        assert len(a.samples.as_slice()) == len(b.samples.as_slice())
        assert [(e.start_sample, e.num_samples) for e in x] == [(e.start_sample, e.num_samples) for e in y]


def test_result_layout_fetches_and_output_stage(voices):
    """The formant stage keeps the job's result compact (the utterances back to back, sum(samples) long): a caller's
    d_out of exactly that size and copy_out give what fetch gives; i16, G.711 and FLAC are those of the delivered
    samples; loudness measures and scales the formant output; bounds and lengths are those without formants."""
    import torch
    m = voices("medium")
    batches = [_ids(34, 1200), _ids(27, 1201), _ids(31, 1202)]
    seeds = [41, 42, 43]
    for kw in (dict(pitches=[1.25, None, 0.8], formants=[1.0, 1.2, NAN]),
               dict(formants=[1.3, None, 0.9]),
               dict(tempos=[1.5, None, None], formants=[None, 0.8, None])):
        r = _run(m, batches, seeds, keep=True, **kw)
        job = r["job"]
        total = sum(len(w) for w in r["wav"])
        _, samples, offs = job.lengths()
        assert int(sum(samples)) == total and list(offs) == list(np.cumsum([0] + list(samples))[:-1])
        flat = np.zeros(total, np.float32)
        assert job.copy_out(flat.ctypes.data, total * 4, 0) == total * 4
        np.testing.assert_array_equal(flat, np.concatenate(r["wav"]))
        i16 = np.zeros(total, np.int16)
        assert job.copy_out(i16.ctypes.data, total * 2, 1) == total * 2
        np.testing.assert_array_equal(i16, np.concatenate(r["i16"]))
        flac = job.fetch_flac()
        al = job.fetch_g711("alaw")
        for b in range(3):
            ref16 = AudioSamples(r["wav"][b]).to_i16_vec()
            np.testing.assert_array_equal(r["i16"][b], ref16)
            np.testing.assert_array_equal(flr.decode(flac[b]).samples, ref16)
            np.testing.assert_array_equal(np.frombuffer(al[b], np.uint8),
                                          np.frombuffer(AudioSamples(r["wav"][b]).as_g711_bytes("alaw"), np.uint8))
        buf = torch.zeros(total, dtype=torch.float32, device="cuda")
        j2 = SynthesisJob(m, batches, seeds=seeds, **kw)
        with pytest.raises(sonata_b200.OperationError, match="too small"):
            j2.run(buf.data_ptr(), total - 1)
        j2.run(buf.data_ptr(), total)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(buf.cpu().numpy(), np.concatenate(r["wav"]))
        j2.close()
        job.close()
    # loudness and output rates act on the formant output
    kw = dict(pitches=[1.25, None, None], formants=[1.0, 1.2, None])
    rated = _run(m, batches, seeds, output_rates=[16000, 0, 24000], **kw)
    loud = _run(m, batches, seeds, keep=True, output_rates=[16000, 0, 24000], loudness=[-20.0, -23.0, None], **kw)
    lufs, gains = loud["job"].loudness()
    loud["job"].close()
    for b, rate in enumerate((16000, 22050, 24000)):
        assert abs(lufs[b] - lr.integrated(rated["wav"][b], rate)) <= 1e-6
        np.testing.assert_array_equal(loud["wav"][b], rated["wav"][b] * gains[b])
    # a contour with formants: the same bounds and lengths as without
    contours = [[1.0] * (len(x) - 6) + [1.1, 1.15, 1.2, 1.25, 1.3, 1.3] for x in batches]
    plain = SynthesisJob(m, batches, seeds=seeds, pitch_contours=contours)
    plain.run()
    shaped = SynthesisJob(m, batches, seeds=seeds, pitch_contours=contours, formants=[1.0, 1.0, 1.0])
    shaped.run()
    for a, b in zip(plain.prosody_bounds(), shaped.prosody_bounds()):
        np.testing.assert_array_equal(a, b)
    assert list(plain.lengths()[1]) == list(shaped.lengths()[1])
    assert any(p["name"] == "formant" for p in shaped.profile())
    plain.close()
    shaped.close()
