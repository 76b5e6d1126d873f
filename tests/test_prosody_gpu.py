"""GPU (-m gpu): pitch and tempo on the device against the numpy specification (tests/prosody_reference.py).

Offsets exactly, then the overlap-add and the pitch resampler within their per-sample bounds, on synthesised audio of
every voice quality and on constructed signals; a mixed batch against each utterance alone; jobs without ratios
unchanged; and the stage composed with output rates, loudness, the i16 / G.711 / FLAC fetches, d_out, alignments and the
one-shot C call."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import flac_reference as fr
import loudness_reference as lr
import prosody_reference as pr
import sonata_b200
from sonata_b200 import PiperSynthesisConfig, voicegen, workload
from sonata_b200 import _native as N
from sonata_b200.core import AudioSamples
from sonata_b200.job import SynthesisJob
from sonata_b200.synth import SonataSpeechSynthesizer

pytestmark = pytest.mark.gpu

DEFAULT = PiperSynthesisConfig(None, 0.667, 1.0, 0.8)
GRID = (0.5, 0.8, 1.0, 1.25, 2.0)


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
    get.paths = paths
    yield get
    for m in ms.values():
        m.close()


def _ids(n, utt):
    return list(workload.synthetic_ids(n, utt=utt))


def _device(x, rate, p, t):
    """(y, offsets, stretched or None) of the kernels over one buffer."""
    x = np.ascontiguousarray(x, np.float32)
    pl = pr.plan(rate, len(x), p, t)
    y = np.zeros(pl["n2"] + 1, np.float32)
    off = np.zeros(pl["F"] + 1, np.int32)
    s = np.zeros(pl["n1"] + 1, np.float32)
    err = N.sb200_error()
    f = lambda v: float("nan") if v is None else float(v)
    rc = N.lib().sb200_debug_prosody(0, x.ctypes.data_as(C.POINTER(C.c_float)), x.size, rate, f(p), f(t),
                                     y.ctypes.data_as(C.POINTER(C.c_float)), y.size,
                                     off.ctypes.data_as(C.POINTER(C.c_int32)), off.size,
                                     s.ctypes.data_as(C.POINTER(C.c_float)), s.size, C.byref(err))
    assert rc == 0, C.string_at(err.message) if err.message else rc
    return y[:pl["n2"]], off[:pl["F"]], s[:pl["n1"]] if pl["stretch"] else None


def _check_against_reference(x, rate, p, t):
    y, off, s = _device(x, rate, p, t)
    pl = pr.plan(rate, len(x), p, t)
    cur = np.asarray(x, np.float64)
    if pl["stretch"]:
        np.testing.assert_array_equal(off, pr.offsets(x, pl))
        ref, bound = pr.overlap_add(x, pl, off.astype(np.int64))
        assert np.all(np.abs(s - ref) <= bound), (rate, p, t, float(np.max(np.abs(s - ref) - bound)))
        cur = s.astype(np.float64)       # the pitch stage is held to the float64 sum over the signal it was given
        if not pl["pitch"]:
            np.testing.assert_array_equal(y, s)
    if pl["pitch"]:
        ref, bound = pr.pitch_resample(cur, pl)
        assert np.all(np.abs(y - ref) <= bound), (rate, p, t, float(np.max(np.abs(y - ref) - bound)))
    if not pl["stretch"] and not pl["pitch"]:
        np.testing.assert_array_equal(y, x)
    return y


@pytest.mark.parametrize("rate", [22050, 16000])
def test_constructed_signals(lib_built, rate):
    rng = np.random.default_rng(rate)
    tone = pr.tone(rate, 150, 0.6) + 0.5 * pr.tone(rate, 450, 0.6)
    noise = (rng.standard_normal(rate // 2) * 0.2).astype(np.float32)
    square = np.tile(np.array([0.5, 0.5, -0.5, -0.5], np.float32), rate // 8)     # every frame has tied lags
    loud = np.clip(rng.standard_normal(rate // 3) * 2.0, -3, 3).astype(np.float32)  # clamps in the quantiser
    for p in GRID:
        for t in GRID + (0.25, 4.0):
            _check_against_reference(tone, rate, p, t)
    for x in (noise, square, loud, np.zeros(3000, np.float32), tone[:7]):
        for p, t in ((None, 2.0), (1.25, None), (0.8, 0.5), (2.0, 0.25), (0.5, 4.0), (None, 1.01)):
            _check_against_reference(x, rate, p, t)


@pytest.mark.parametrize("quality", ["medium", "high", "low", "x_low"])
def test_synthesised_audio(voices, quality):
    m = voices(quality)
    rate = m.audio_output_info().sample_rate
    combos = [(p, t) for p in GRID for t in GRID + (0.25, 4.0) if (p, t) != (1.0, 1.0)]
    base = m.infer_batch_with_values([_ids(20, 7), _ids(33, 8)], seeds=[70, 71])
    xs = [a.samples.as_slice().copy() for a in base]
    for i, (p, t) in enumerate(combos):
        _check_against_reference(xs[i % 2], rate, p, t)
    # a job gives an utterance what the kernels give its waveform alone
    B = 6
    batches = [_ids(14 + 3 * b, 20 + b) for b in range(B)]
    seeds = [900 + b for b in range(B)]
    pitches = [1.25, None, 0.8, None, 2.0, 0.5]
    tempos = [None, 1.5, 2.0, None, 2.0, 0.25]
    plain = m.infer_batch_with_values(batches, seeds=seeds)
    got = m.infer_batch_with_values(batches, seeds=seeds, pitches=pitches, tempos=tempos)
    for b in range(B):
        x = plain[b].samples.as_slice()
        np.testing.assert_array_equal(got[b].samples.as_slice(), _device(x, rate, pitches[b], tempos[b])[0])
        assert got[b].info.sample_rate == rate


def _run(m, batches, seeds, **kw):
    job = SynthesisJob(m, batches, seeds=seeds, **kw)
    n0 = N.lib().sb200_launch_count()
    job.run()
    launches = N.lib().sb200_launch_count() - n0
    out = dict(wav=[a.samples.as_slice().copy() for a in job.fetch()], i16=job.fetch_i16(), profile=job.profile(),
               launches=launches, lengths=job.lengths(), job=job)
    return out


def test_mixed_batch_equals_alone_and_neutral_changes_nothing(voices):
    m = voices("medium")
    B = 8
    batches = [_ids(40 - 3 * b, 300 + b) for b in range(B)]
    seeds = [4000 + b for b in range(B)]
    pitches = [1.25, None, 0.8, None, 2.0, 1.0, None, 0.5]
    tempos = [None, 1.5, 2.0, None, 2.0, float("nan"), 0.25, 4.0]
    base = _run(m, batches, seeds)
    mixed = _run(m, batches, seeds, pitches=pitches, tempos=tempos)
    names = [r["name"] for r in mixed["profile"]]
    assert names.count("stretch") == 1 and names.count("pitch") == 1
    assert mixed["launches"] == base["launches"] + 3
    n1, n2, frames = mixed["job"].prosody()
    for b in range(B):
        alone = _run(m, [batches[b]], [seeds[b]], pitches=[pitches[b]], tempos=[tempos[b]])
        np.testing.assert_array_equal(mixed["wav"][b], alone["wav"][0])
        np.testing.assert_array_equal(mixed["i16"][b], alone["i16"][0])
        alone["job"].close()
        pl = pr.plan(22050, len(base["wav"][b]), pitches[b], tempos[b])
        assert (n1[b], n2[b], frames[b]) == (pl["n1"], pl["n2"], pl["F"]) and len(mixed["wav"][b]) == pl["n2"]
        assert mixed["lengths"][1][b] == pl["n2"]
        if b in (1, 3, 5):
            np.testing.assert_array_equal(mixed["wav"][3], base["wav"][3])
    np.testing.assert_array_equal(mixed["wav"][5], base["wav"][5])
    # no utterance asks: same launches, regions, workspace and bits as a job that never heard of the stage
    for kw in (dict(pitches=[None] * B, tempos=[1.0] * B), dict(pitches=[float("nan")] * B), dict(tempos=None)):
        same = _run(m, batches, seeds, **kw)
        assert same["launches"] == base["launches"]
        assert [r["name"] for r in same["profile"]] == [r["name"] for r in base["profile"]]
        for a, b in zip(same["wav"], base["wav"]):
            np.testing.assert_array_equal(a, b)
        with pytest.raises(sonata_b200.OperationError, match="no prosody"):
            same["job"].prosody()
        same["job"].close()
    # a bad entry names the utterance and leaves the job's ratios as they were
    job = mixed["job"]
    bad = np.array([1.0] * (B - 1) + [7.0], np.float32)
    err = N.sb200_error()
    assert m._lib.sb200_job_set_prosody(job._h, None, bad.ctypes.data_as(C.POINTER(C.c_float)), C.byref(err)) == 19
    msg = C.string_at(err.message).decode()
    N.lib().sb200_string_free(err.message)
    assert f"utterance {B - 1}" in msg and "tempo" in msg
    job.run()
    for a, b in zip(job.fetch(), mixed["wav"]):
        np.testing.assert_array_equal(a.samples.as_slice(), b)
    job.set_prosody(None, None)
    job.run()
    for a, b in zip(job.fetch(), base["wav"]):
        np.testing.assert_array_equal(a.samples.as_slice(), b)
    job.close()
    base["job"].close()


def _resample(x, in_rate, out_rate):
    x = np.ascontiguousarray(x, np.float32)
    g = np.gcd(in_rate, out_rate)
    y = np.zeros(-(-len(x) * (out_rate // g) // (in_rate // g)), np.float32)
    err = N.sb200_error()
    assert N.lib().sb200_debug_resample(0, x.ctypes.data_as(C.POINTER(C.c_float)), x.size, in_rate, out_rate,
                                        y.ctypes.data_as(C.POINTER(C.c_float)), C.byref(err)) == 0
    return y


def test_composes_with_the_output_stage(voices):
    import torch
    m = voices("medium")
    batches = [_ids(30, 50), _ids(22, 51), _ids(26, 52)]
    seeds = [50, 51, 52]
    kw = dict(pitches=[1.25, None, 0.8], tempos=[1.5, 2.0, None])
    pros = _run(m, batches, seeds, **kw)
    # output rates: the resample launch reads the prosody output
    rates = [48000, 8000, None]
    both = _run(m, batches, seeds, output_rates=rates, **kw)
    for b in range(3):
        want = pros["wav"][b] if rates[b] is None else _resample(pros["wav"][b], 22050, rates[b])
        np.testing.assert_array_equal(both["wav"][b], want)
    # loudness: measured on the delivered signal
    loud = _run(m, batches, seeds, output_rates=rates, loudness=[-20.0, -23.0, None], **kw)
    lufs, gains = loud["job"].loudness()
    for b in range(3):
        assert abs(lufs[b] - lr.integrated(both["wav"][b], rates[b] or 22050)) <= 1e-6
        np.testing.assert_array_equal(loud["wav"][b], both["wav"][b] * gains[b])
    # i16, G.711 and FLAC of the delivered samples
    job = both["job"]
    flac = job.fetch_flac()
    mu = job.fetch_g711("mulaw")
    for b in range(3):
        i16 = AudioSamples(both["wav"][b]).to_i16_vec()
        np.testing.assert_array_equal(both["i16"][b], i16)
        np.testing.assert_array_equal(fr.decode(flac[b]).samples, i16)
        np.testing.assert_array_equal(np.frombuffer(mu[b], np.uint8),
                                      np.frombuffer(AudioSamples(both["wav"][b]).as_g711_bytes("mulaw"), np.uint8))
    # d_out: capacity counts delivered samples
    total = sum(len(w) for w in pros["wav"])
    buf = torch.zeros(total, dtype=torch.float32, device="cuda")
    j2 = SynthesisJob(m, batches, seeds=seeds, **kw)
    with pytest.raises(sonata_b200.OperationError, match="too small"):
        j2.run(buf.data_ptr(), total - 1)
    j2.run(buf.data_ptr(), total)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(buf.cpu().numpy(), np.concatenate(pros["wav"]))
    j2.close()
    for r in (pros, both, loud):
        r["job"].close()


def test_frontends(voices, tmp_path):
    import wave
    m = voices("medium")
    phs = ["hɛloʊ wɜːld ðɪs ɪz ə lɔŋɡɚ sɛntəns", "ænd ə sɛkənd wʌn"]
    ids = [m.phonemes_to_input_ids(p) for p in phs]
    kw = dict(pitches=[1.25, 1.25], tempos=[1.5, 1.5])
    job = _run(m, ids, [5, 6], **kw)
    job["job"].close()
    for a, w in zip(m.speak_batch(phs, seeds=[5, 6], **kw), job["wav"]):
        np.testing.assert_array_equal(a.samples.as_slice(), w)
    # the one-shot C call (infer_batch_with_durations) and its frame counts, which stay frame counts
    plain = m.infer_batch_with_durations(ids, seeds=[5, 6])
    for (a, f), (_, f0), w in zip(m.infer_batch_with_durations(ids, seeds=[5, 6], **kw), plain, job["wav"]):
        np.testing.assert_array_equal(a.samples.as_slice(), w)
        np.testing.assert_array_equal(f, f0)
    for (a, al), w in zip(m.speak_batch_with_alignment(phs, seeds=[5, 6], **kw), job["wav"]):
        np.testing.assert_array_equal(a.samples.as_slice(), w)
        assert al[0].start_sample == 0 and sum(x.num_samples for x in al) == len(w)
        assert all(y.start_sample == x.start_sample + x.num_samples for x, y in zip(al, al[1:]))
    assert [bytes(b) for b in m.speak_batch_g711(phs, "alaw", seeds=[5, 6], **kw)] == \
        [AudioSamples(w).as_g711_bytes("alaw") for w in job["wav"]]
    for f, w in zip(m.speak_batch_flac(phs, seeds=[5, 6], **kw), job["wav"]):
        np.testing.assert_array_equal(fr.decode(f).samples, AudioSamples(w).to_i16_vec())
    synth = SonataSpeechSynthesizer(m)
    text = "\n".join(phs)
    for mode in (synth.synthesize_parallel, synth.synthesize_lazy):
        for a, w in zip(mode(text, seed=5, pitch_ratio=1.25, tempo=1.5), job["wav"]):
            np.testing.assert_array_equal(a.samples.as_slice(), w)
    f = tmp_path / "s.wav"
    synth.synthesize_to_file(f, text, seed=5, pitch_ratio=1.25, tempo=1.5)
    with wave.open(str(f)) as r:
        data = np.frombuffer(r.readframes(r.getnframes()), "<i2")
    np.testing.assert_array_equal(data, AudioSamples(np.concatenate(job["wav"])).to_i16_vec())
    from sonata_b200 import cli
    (tmp_path / "in.txt").write_text(text + "\n", encoding="utf-8")
    out = tmp_path / "c.wav"
    assert cli.main([voices.paths["medium"], "-f", str(tmp_path / "in.txt"), "-o", str(out), "--mode", "parallel",
                     "--pitch-ratio", "1.25", "--tempo", "1.5", "--seed", "5"]) == 0
    with wave.open(str(out)) as r:
        np.testing.assert_array_equal(np.frombuffer(r.readframes(r.getnframes()), "<i2"), data)
    m.set_fallback_synthesis_config(DEFAULT)
