"""GPU (-m gpu): pitch contours on the device against the numpy specification (tests/prosody_contour_reference.py).

Offsets exactly and waveforms within the per-sample bounds, on constructed signals and on synthesised audio of every
voice quality; a uniform contour against the utterance ratio and a neutral one against none, bit for bit; a mixed batch
against each utterance alone; alignments from the delivered ends; and the output stage applied to a contoured job."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import flac_reference as fr
import loudness_reference as lr
import prosody_contour_reference as pc
import prosody_reference as pr
import sonata_b200
from sonata_b200 import PiperSynthesisConfig, voicegen, workload
from sonata_b200 import _native as N
from sonata_b200.core import AudioSamples
from sonata_b200.job import SynthesisJob
from sonata_b200.piper import _alignment, rate_ratio

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


def _device(x, rate, ends, ratios, tempo):
    """(y, offsets, stretched or None, plan) of the kernels over one buffer."""
    x = np.ascontiguousarray(x, np.float32)
    ends = np.ascontiguousarray(ends, np.int64)
    ratios = np.ascontiguousarray(ratios, np.float32)
    pl = pc.plan(rate, len(x), ends, ratios, tempo)
    y = np.zeros(pl["n2"] + 1, np.float32)
    off = np.zeros(pl["F"] + 1, np.int32)
    s = np.zeros(pl["n1"] + 1, np.float32)
    err = N.sb200_error()
    rc = N.lib().sb200_debug_prosody_contour(0, f32p(x), x.size, rate, i64p(ends), f32p(ratios), len(ends),
                                             NAN if tempo is None else tempo, f32p(y), y.size,
                                             off.ctypes.data_as(C.POINTER(C.c_int32)), off.size, f32p(s), s.size,
                                             C.byref(err))
    assert rc == 0, C.string_at(err.message) if err.message else rc
    return y[:pl["n2"]], off[:pl["F"]], s[:pl["n1"]] if pl["stretch"] else None, pl


def _utterance_ratio(x, rate, p, tempo):
    x = np.ascontiguousarray(x, np.float32)
    pl = pr.plan(rate, len(x), p, tempo)
    y = np.zeros(pl["n2"] + 1, np.float32)
    err = N.sb200_error()
    assert N.lib().sb200_debug_prosody(0, f32p(x), x.size, rate, NAN if p is None else p,
                                       NAN if tempo is None else tempo, f32p(y), y.size, None, 0, None, 0,
                                       C.byref(err)) == 0
    return y[:pl["n2"]]


def _check_against_reference(x, rate, ends, ratios, tempo):
    y, off, s, pl = _device(x, rate, ends, ratios, tempo)
    assert len(y) == pl["n2"]
    if pl["one"] is not None:           # one piece: the utterance ratio it equals, bit for bit
        p = float(pl["p"][0])
        np.testing.assert_array_equal(y, _utterance_ratio(x, rate, None if p == 1.0 else p, tempo))
        return y, pl
    np.testing.assert_array_equal(off, pr.offsets(x, pl))
    ref, bound = pr.overlap_add(x, pl, off.astype(np.int64))
    assert np.all(np.abs(s - ref) <= bound), (rate, tempo, float(np.max(np.abs(s - ref) - bound)))
    ref, bound = pc.pitch_resample(s.astype(np.float64), pl)
    assert np.all(np.abs(y - ref) <= bound), (rate, tempo, float(np.max(np.abs(y - ref) - bound)))
    return y, pl


@pytest.mark.parametrize("rate", [22050, 16000])
def test_constructed_signals(lib_built, rate):
    rng = np.random.default_rng(rate)
    x = pr.tone(rate, 150, 0.6) + 0.5 * pr.tone(rate, 450, 0.6)
    noise = (rng.standard_normal(len(x)) * 0.2).astype(np.float32)
    n = len(x)
    cases = [
        ([n // 3, n], [0.5, 2.0]),                                             # the extremes meet inside a pitch block
        ([n // 4, n // 2, 3 * n // 4, n], [1.0, 1.3, 0.8, 1.3]),
        (list(np.cumsum([37, 90, 0, 150, 11, 200]).tolist()) + [n], [2.0, 0.5, 0.9, 1.7, 0.6, 2.0, 1.1]),  # < Hs
        (list(np.linspace(0, n, 41).astype(np.int64)[1:]), list(rng.uniform(0.5, 2.0, 40))),
        ([n // 2, n], [1.25, 1.25]),                                           # one piece
        ([n // 2, n], [1.0, NAN]),                                             # neutral
    ]
    knots_inside = 0
    for sig in (x, noise):
        for ends, ratios in cases:
            for tempo in (None, 0.5, 2.5):
                _, pl = _check_against_reference(sig, rate, ends, ratios, tempo)
                if pl["m"] > 1:
                    knots_inside += int(np.sum(np.ceil(pl["Q"][1:]) % 256 != 0))
    assert knots_inside > 10


@pytest.mark.parametrize("quality", ["medium", "high", "low", "x_low"])
def test_synthesised_audio(voices, quality):
    m = voices(quality)
    rate = m.audio_output_info().sample_rate
    rng = np.random.default_rng(11)
    batches = [_ids(22, 7), _ids(31, 8), _ids(17, 9)]
    seeds = [70, 71, 72]
    contours = [list(rng.choice([0.8, 1.0, 1.25], len(b))) for b in batches]
    contours[2] = [1.0] * (len(batches[2]) - 4) + [1.06, 1.12, 1.18, 1.3]    # a question's rise
    tempos = [None, 1.5, 0.8]
    plain = m.infer_batch_with_durations(batches, seeds=seeds)
    got = m.infer_batch_with_durations(batches, seeds=seeds, tempos=tempos, pitch_contours=contours)
    for b in range(len(batches)):
        (x, frames), (a, f) = plain[b], got[b]
        np.testing.assert_array_equal(f, frames)
        x = x.samples.as_slice().copy()
        ends = 256 * np.cumsum(frames)
        y, pl = _check_against_reference(x, rate, ends, contours[b], tempos[b])
        np.testing.assert_array_equal(a.samples.as_slice(), y)
        assert len(a.samples.as_slice()) == pl["n2"] and a.info.sample_rate == rate


def _run(m, batches, seeds, **kw):
    durations = kw.pop("durations", None)
    job = SynthesisJob(m, batches, seeds=seeds, **kw)
    if durations is not None:
        job.set_durations(None, durations)
    n0 = N.lib().sb200_launch_count()
    job.run()
    launches = N.lib().sb200_launch_count() - n0
    return dict(wav=[a.samples.as_slice().copy() for a in job.fetch()], i16=job.fetch_i16(), profile=job.profile(),
                launches=launches, lengths=job.lengths(), job=job)


def test_uniform_is_the_utterance_ratio_and_neutral_is_none(voices):
    m = voices("medium")
    B = 4
    batches = [_ids(30 - 4 * b, 500 + b) for b in range(B)]
    seeds = [5000 + b for b in range(B)]
    base = _run(m, batches, seeds)
    for tempos in (None, [None, 1.5, 0.5, 2.5]):
        tkw = {} if tempos is None else dict(tempos=tempos)
        ratio = _run(m, batches, seeds, pitches=[1.25] * B, **tkw)
        uni = _run(m, batches, seeds, pitch_contours=[[1.25] * len(x) for x in batches], **tkw)
        for a, b in zip(uni["wav"], ratio["wav"]):
            np.testing.assert_array_equal(a, b)
        assert uni["launches"] == ratio["launches"]
        for a, b in zip(uni["job"].prosody(), ratio["job"].prosody()):
            np.testing.assert_array_equal(a, b)
        vals = m.infer_batch_with_values(batches, seeds=seeds, pitch_contours=[[1.25] * len(x) for x in batches], **tkw)
        for a, b in zip(vals, ratio["wav"]):
            np.testing.assert_array_equal(a.samples.as_slice(), b)
        for r in (ratio, uni):
            r["job"].close()
    # all 1 / NaN: nothing new laid out or launched, the same bits
    for contours in ([[1.0] * len(x) for x in batches], [None, [NAN] * len(batches[1]), None, None]):
        same = _run(m, batches, seeds, pitch_contours=contours)
        assert same["launches"] == base["launches"]
        assert [r["name"] for r in same["profile"]] == [r["name"] for r in base["profile"]]
        for a, b in zip(same["wav"], base["wav"]):
            np.testing.assert_array_equal(a, b)
        same["job"].close()
    base["job"].close()


def test_mixed_batch_equals_alone(voices):
    m = voices("medium")
    rng = np.random.default_rng(3)
    B = 6
    batches = [_ids(36 - 3 * b, 700 + b) for b in range(B)]
    seeds = [7000 + b for b in range(B)]
    contours = [list(rng.choice([0.8, 1.0, 1.25], len(x))) for x in batches]
    contours[1] = contours[4] = None
    pitches = [None, 1.25, None, None, None, None]
    tempos = [None, None, 1.5, None, 0.8, 2.0]
    durations = [None] * B
    durations[3] = [-1, 0, 0] + [-1] * (len(batches[3]) - 3)          # ids without frames
    kw = dict(pitch_contours=contours, pitches=pitches, tempos=tempos, durations=durations)
    mixed = _run(m, batches, seeds, **kw)
    names = [r["name"] for r in mixed["profile"]]
    assert names.count("stretch") == 1 and names.count("pitch") == 1
    n1, n2, frames = mixed["job"].prosody()
    bounds = mixed["job"].prosody_bounds()
    id_frames = mixed["job"].id_frames()
    for b in range(B):
        alone = _run(m, [batches[b]], [seeds[b]], **{k: [v[b]] for k, v in kw.items()})
        np.testing.assert_array_equal(mixed["wav"][b], alone["wav"][0])
        np.testing.assert_array_equal(mixed["i16"][b], alone["i16"][0])
        np.testing.assert_array_equal(bounds[b], alone["job"].prosody_bounds()[0])
        alone["job"].close()
        ends = 256 * np.cumsum(id_frames[b])
        n = 256 * max(int(ends[-1]) // 256, 1)
        ratios = [pitches[b] or NAN] * len(batches[b]) if contours[b] is None else contours[b]
        pl = pc.plan(22050, n, ends, ratios, tempos[b])
        assert (n1[b], n2[b], frames[b]) == (pl["n1"], pl["n2"], pl["F"]) and len(mixed["wav"][b]) == pl["n2"]
        np.testing.assert_array_equal(bounds[b], pl["bounds"])
    # argument checks at the C and job levels: the utterance and the id, and the job as it was
    job = mixed["job"]
    packed = np.concatenate([np.asarray(c if c is not None else [NAN] * len(x), np.float32)
                             for c, x in zip(contours, batches)])
    bad = packed.copy()
    bad[len(batches[0]) + 2] = 2.5
    err = N.sb200_error()
    assert m._lib.sb200_job_set_pitch_contour(job._h, f32p(bad), C.byref(err)) == 19
    msg = C.string_at(err.message).decode()
    N.lib().sb200_string_free(err.message)
    assert "utterance 1, id 2" in msg and "pitch ratio" in msg
    clash = packed.copy()
    clash[len(batches[0]) + 1] = 0.8                                    # utterance 1 has a pitch ratio
    assert m._lib.sb200_job_set_pitch_contour(job._h, f32p(clash), C.byref(err)) == 19
    msg = C.string_at(err.message).decode()
    N.lib().sb200_string_free(err.message)
    assert "utterance 1: a pitch contour and a pitch ratio" in msg
    with pytest.raises(sonata_b200.OperationError, match="utterance 2, id 0: pitch ratio 0.1"):
        job.set_pitch_contours([None, None, [0.1] * len(batches[2]), None, None, None])
    with pytest.raises(sonata_b200.OperationError, match="utterance 0: a pitch contour and a pitch ratio"):
        job.set_prosody([1.5] + [None] * (B - 1), tempos)
    with pytest.raises(sonata_b200.OperationError, match="utterance 0: a pitch contour and a pitch ratio"):
        m.infer_batch_with_values(batches[:1], pitches=[1.5], pitch_contours=[contours[0]])
    job.run()
    for a, w in zip(job.fetch(), mixed["wav"]):
        np.testing.assert_array_equal(a.samples.as_slice(), w)
    job.close()


def _resample(x, in_rate, out_rate):
    x = np.ascontiguousarray(x, np.float32)
    g = np.gcd(in_rate, out_rate)
    y = np.zeros(-(-len(x) * (out_rate // g) // (in_rate // g)), np.float32)
    err = N.sb200_error()
    assert N.lib().sb200_debug_resample(0, f32p(x), x.size, in_rate, out_rate, f32p(y), C.byref(err)) == 0
    return y


def test_alignment_follows_the_delivered_ends(voices):
    m = voices("medium")
    phs = ["hɛloʊ wɜːld ðɪs ɪz ə lɔŋɡɚ sɛntəns", "ænd ə sɛkənd wʌn"]
    char_contours = [[1.0] * (3 * len(p) // 4) + [1.06, 1.12, 1.18, 1.24, 1.3] * len(p) for p in phs]
    char_contours = [c[:len(p)] for c, p in zip(char_contours, phs)]
    plain = m.speak_batch_with_alignment(phs, seeds=[5, 6])
    got = m.speak_batch_with_alignment(phs, seeds=[5, 6], pitch_contours=char_contours)
    for (a0, al0), (a, al) in zip(plain, got):
        assert [x.phoneme for x in al] == [x.phoneme for x in al0]
        assert [x.start_sample for x in al] == [x.start_sample for x in al0]     # no tempo: the boundaries stay
        assert sum(x.num_samples for x in al) == len(a.samples.as_slice())
    maps = [m.phonemes_to_input_ids_map(p) for p in phs]
    frames = [f for _, f in m.infer_batch_with_durations([i for i, _ in maps], seeds=[5, 6])]
    id_ratios = [[1.0 if c < 0 else cc[c] for c in src] for cc, (_, src) in zip(char_contours, maps)]
    for kw in (dict(tempos=[1.5, 0.8]), dict(tempos=[None, 2.0], output_rates=[48000, 16000])):
        got = m.speak_batch_with_alignment(phs, seeds=[5, 6], pitch_contours=char_contours, **kw)
        wav = m.speak_batch(phs, seeds=[5, 6], pitch_contours=char_contours, **kw)
        for b, (a, al) in enumerate(got):
            n = len(a.samples.as_slice())
            np.testing.assert_array_equal(a.samples.as_slice(), wav[b].samples.as_slice())
            pl = pc.plan(22050, 256 * int(np.sum(frames[b])), 256 * np.cumsum(frames[b]), id_ratios[b],
                         kw["tempos"][b])
            up, down = rate_ratio(22050, a.info.sample_rate)
            want = _alignment(phs[b], maps[b][1], frames[b], n, up, down, bounds=pl["bounds"])
            assert [(x.start_sample, x.num_samples) for x in al] == [(x.start_sample, x.num_samples) for x in want]
            assert al[0].start_sample == 0 and sum(x.num_samples for x in al) == n
            assert all(y.start_sample == x.start_sample + x.num_samples for x, y in zip(al, al[1:]))


def test_composes_with_the_output_stage(voices):
    m = voices("medium")
    rng = np.random.default_rng(9)
    batches = [_ids(30, 50), _ids(22, 51), _ids(26, 52)]
    seeds = [50, 51, 52]
    kw = dict(pitch_contours=[list(rng.choice([0.8, 1.25], len(x))) for x in batches], tempos=[1.5, None, 0.8])
    pros = _run(m, batches, seeds, **kw)
    rates = [48000, 8000, None]
    both = _run(m, batches, seeds, output_rates=rates, **kw)
    for b in range(3):
        want = pros["wav"][b] if rates[b] is None else _resample(pros["wav"][b], 22050, rates[b])
        np.testing.assert_array_equal(both["wav"][b], want)
    loud = _run(m, batches, seeds, output_rates=rates, loudness=[-20.0, -23.0, None], **kw)
    lufs, gains = loud["job"].loudness()
    for b in range(3):
        assert abs(lufs[b] - lr.integrated(both["wav"][b], rates[b] or 22050)) <= 1e-6
        np.testing.assert_array_equal(loud["wav"][b], both["wav"][b] * gains[b])
    job = both["job"]
    flac = job.fetch_flac()
    mu = job.fetch_g711("mulaw")
    for b in range(3):
        i16 = AudioSamples(both["wav"][b]).to_i16_vec()
        np.testing.assert_array_equal(both["i16"][b], i16)
        np.testing.assert_array_equal(fr.decode(flac[b]).samples, i16)
        np.testing.assert_array_equal(np.frombuffer(mu[b], np.uint8),
                                      np.frombuffer(AudioSamples(both["wav"][b]).as_g711_bytes("mulaw"), np.uint8))
    for r in (pros, both, loud):
        r["job"].close()
