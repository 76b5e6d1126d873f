"""GPU (-m gpu): per-phoneme duration control and timings.

Neutral controls (all scales 1.0, all frames -1) and frames fixed to the predicted ones give the bits of a run without
controls; fixed durations match the oracle's path given the same w_ceil (tests/durations_reference.py); scaled durations follow ceil((exp(logw) * ls) * s)
from the job's own logw; a batch mixing controlled and plain utterances equals each utterance run alone; and the
frames per id the library reports agree with its cum, its sample counts, the alignment of phoneme strings and the
streaming encoder's p_duration."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import durations_reference as dr
import sonata_b200
from oracle import vits_oracle as vo
from sonata_b200 import OperationError, PiperSynthesisConfig, voicegen, workload
from sonata_b200 import _native as N
from sonata_b200.job import SynthesisJob

pytestmark = pytest.mark.gpu

LENS = [1, 7, 64, 65, 130, 513, 33, 200, 2, 97, 300, 16]
SPEAKERS = [0, 3, 1, 3, None, 2, 0, None, 1, 2, 3, 0]
QUALITY = {"medium": "medium", "high": "high", "x_low": "x_low", "medium4": "medium"}
CAPTURES = ("logw", "z_p", "z")
HOP = 256


def _ids(n, utt):
    return workload.synthetic_ids(n // 2 + 1, utt=utt)[:n]


@pytest.fixture(scope="module")
def voices(lib_built):
    d = voicegen.default_voice_dir()
    paths = {"medium": voicegen.write_voice(d, "medium"), "high": voicegen.write_voice(d, "high"),
             "x_low": voicegen.write_voice(d, "x_low"), "medium4": voicegen.write_voice(d, "medium", n_speakers=4)}
    ms = {}

    def get(name):
        if name not in ms:
            ms[name] = sonata_b200.from_config_path(paths[name], device=0)
        return ms[name]
    get.paths = paths
    yield get
    for m in ms.values():
        m.close()


def _configs(voice, noise):
    ns, nw = (0.667, 0.8) if noise else (0.0, 0.0)
    spk = (lambda b: None if SPEAKERS[b] is None else SPEAKERS[b]) if voice == "medium4" else (lambda b: None)
    return [PiperSynthesisConfig(spk(b), ns, (0.8, 1.0, 1.25)[b % 3], nw) for b in range(len(LENS))]


def _capture(job):
    out = []
    wavs = job.fetch()
    for b in range(job.batch):
        r = {"wav": wavs[b].samples.as_slice().copy(), "cum": job.durations(b)}
        for k in CAPTURES:
            r[k] = job.debug_fetch(k, b)
        out.append(r)
    i16 = job.fetch_i16()
    for b, r in enumerate(out):
        r["i16"] = i16[b]
    return out


def _same(a, b, keys, what):
    for i, (x, y) in enumerate(zip(a, b)):
        for k in keys:
            assert x[k].shape == y[k].shape and np.array_equal(x[k], y[k]), (what, i, k)


# ---------------------------------------------------------------- 1, 2 and the timings of a plain job
@pytest.mark.parametrize("voice", ["medium", "high", "x_low", "medium4"])
@pytest.mark.parametrize("backend", [1, 0])
def test_neutral_and_own_frames_change_nothing(voices, voice, backend):
    """One job (so Philox draws are the same in every run): no controls, then all-1.0 scales with all -1 frames, then
    every id fixed to its own predicted frame count.  Also: id_frames == diff(cum) and sum(frames) * 256 == samples."""
    m = voices(voice)
    m.set_backend(backend)
    try:
        batches = [_ids(n, 300 + i) for i, n in enumerate(LENS)]
        for noise in (False, True):
            job = SynthesisJob(m, batches, debug=True, configs=_configs(voice, noise))
            job.run()
            plain = _capture(job)
            frames = job.id_frames()
            _, samples, _ = job.lengths()
            for b in range(len(batches)):
                assert np.array_equal(frames[b], np.diff(np.concatenate([[0], plain[b]["cum"]]))), b
                assert int(frames[b].sum()) * HOP == samples[b] == len(plain[b]["wav"]), b
            job.set_durations([np.ones(n, np.float32) for n in LENS], [np.full(n, -1, np.int32) for n in LENS])
            job.run()
            _same(_capture(job), plain, ("wav", "cum", "i16") + CAPTURES, ("neutral", voice, backend, noise))
            job.set_durations(None, frames)
            job.run()
            _same(_capture(job), plain, ("wav", "cum", "logw", "z_p", "z"), ("own frames", voice, backend, noise))
            job.close()
    finally:
        m.set_backend(1)


# ---------------------------------------------------------------- 3: fixed durations against the oracle
def _fixed_counts(n, seed, long_id=None):
    r = np.random.default_rng(seed)
    f = r.integers(0, 13, size=n).astype(np.int32)
    for s in range(0, n, 37):                          # runs of zeros
        f[s:s + 5] = 0
    if long_id is not None:
        f[long_id] = 300
    return f


@pytest.mark.parametrize("size,noise,backend", [("C1", False, 1), ("C1", True, 1), ("C2", True, 1), ("C1", True, 0)])
def test_fixed_durations_against_oracle(voices, oracle_weights, size, noise, backend):
    from test_gpu_parity import TOL_WAV
    m = voices("medium")
    m.set_backend(backend)
    W = oracle_weights("medium")
    I = voicegen.ARCH["medium"]["inter"]
    nph = workload.CONFIGS[size][2]
    batches = [vo.synthetic_ids(nph, utt=5), vo.synthetic_ids(6, utt=6)]
    fixed = [_fixed_counts(len(batches[0]), 11, long_id=len(batches[0]) // 3), np.zeros(len(batches[1]), np.int32)]
    y_len = [max(int(f.sum()), 1) for f in fixed]
    ns = 0.667 if noise else 0.0
    rng = np.random.default_rng(21)
    eps_w = [rng.standard_normal((len(ids), 2)).astype(np.float32) for ids in batches]
    eps_z = [rng.standard_normal((y, I)).astype(np.float32) for y in y_len] if noise else None
    cfg = [PiperSynthesisConfig(None, ns, 1.0, 0.8)] * 2
    job = SynthesisJob(m, batches, eps_w, eps_z, configs=cfg)
    job.set_durations(None, fixed)
    try:
        job.run()
        wavs = job.fetch()
        got_frames = job.id_frames()
        assert job.lengths()[0] == y_len
        for b, ids in enumerate(batches):
            assert np.array_equal(got_frames[b], fixed[b]), b
            ez = None if eps_z is None else torch.from_numpy(eps_z[b].T.copy()).view(1, I, -1)
            ref = dr.infer(W, ids, [ns, 1.0, 0.8], eps_w=torch.from_numpy(eps_w[b].T.copy()).view(1, 2, -1), eps_z=ez,
                           w_ceil=torch.from_numpy(fixed[b].astype(np.float32))).numpy()
            got = wavs[b].samples.as_slice()
            assert got.shape == ref.shape, b
            err = float(np.abs(got.astype(np.float64) - ref).max())
            assert err < TOL_WAV, (b, err)
        assert len(wavs[1]) == HOP and not got_frames[1].any()          # every id 0 frames: one frame
    finally:
        job.close()
        m.set_backend(1)


# ---------------------------------------------------------------- 4: scaled durations
@pytest.mark.parametrize("voice,backend", [("medium", 1), ("medium", 0), ("high", 1), ("x_low", 1), ("medium4", 0)])
def test_scaled_durations_follow_the_jobs_own_logw(voices, voice, backend):
    m = voices(voice)
    m.set_backend(backend)
    rng = np.random.default_rng(8)
    batches = [_ids(n, 400 + i) for i, n in enumerate(LENS)]
    configs = _configs(voice, True)
    scales = []
    for b, n in enumerate(LENS):
        pick = rng.choice(np.array([0, 0.5, 1, 1.7, 3], np.float32), size=n)
        free = rng.uniform(0, 3, size=n).astype(np.float32)
        scales.append(np.where(rng.random(n) < 0.5, pick, free).astype(np.float32))
    job = SynthesisJob(m, batches, debug=True, configs=configs)
    job.set_durations(scales, None)
    near = 0
    try:
        job.run()
        frames = job.id_frames()
        _, samples, _ = job.lengths()
        for b in range(len(batches)):
            lw = job.debug_fetch("logw", b)[:, 0].astype(np.float64)
            w = np.exp(lw) * float(np.float32(configs[b].length_scale)) * scales[b].astype(np.float64)
            wc = np.ceil(w)
            nr = (np.abs(w - np.rint(w)) <= 1e-6 * np.maximum(w, 1.0)) & (w != 0)     # 0 scales give exact zeros
            assert np.all((frames[b] == wc) | (nr & (np.abs(frames[b] - wc) <= 1))), (b, np.nonzero((frames[b] != wc) & ~nr))
            assert not frames[b][scales[b] == 0].any(), b
            assert samples[b] == max(int(frames[b].sum()), 1) * HOP, b
            near += int(nr.sum())
    finally:
        job.close()
        m.set_backend(1)
    print(f"{voice} backend {backend}: {near} ids within 1e-6 of an integer (exempt)")


# ---------------------------------------------------------------- 5: mixed batch
@pytest.mark.parametrize("backend", [1, 0, 2])
def test_mixed_controlled_and_plain_equal_each_alone(voices, backend):
    m = voices("medium4")
    m.set_backend(backend)
    rng = np.random.default_rng(13)
    batches = [_ids(n, 500 + i) for i, n in enumerate(LENS)]
    configs = _configs("medium4", True)
    scales, fixed = [], []
    for b, n in enumerate(LENS):
        kind = b % 4             # plain, scaled, fixed, both
        scales.append(rng.uniform(0.3, 2.5, n).astype(np.float32) if kind in (1, 3) else None)
        f = np.where(rng.random(n) < 0.5, rng.integers(0, 13, n), -1).astype(np.int32) if kind in (2, 3) else None
        fixed.append(f)
    eps_w = [rng.standard_normal((len(ids), 2)).astype(np.float32) for ids in batches]
    first = SynthesisJob(m, batches, eps_w, None, configs=configs)
    first.set_durations(scales, fixed)
    first.run()
    I = voicegen.ARCH["medium"]["inter"]
    eps_z = [rng.standard_normal((f, I)).astype(np.float32) for f in first.lengths()[0]]
    first.close()
    job = SynthesisJob(m, batches, eps_w, eps_z, debug=True, configs=configs)
    job.set_durations(scales, fixed)
    try:
        job.run()
        got = _capture(job)
        got_frames = job.id_frames()
        for b, ids in enumerate(batches):
            alone = SynthesisJob(m, [ids], [eps_w[b]], [eps_z[b]], debug=True, configs=[configs[b]])
            if scales[b] is not None or fixed[b] is not None:
                alone.set_durations([scales[b]] if scales[b] is not None else None,
                                    [fixed[b]] if fixed[b] is not None else None)
            alone.run()
            _same([got[b]], _capture(alone), ("wav", "cum", "i16") + CAPTURES, ("mixed", backend, b))
            assert np.array_equal(got_frames[b], alone.id_frames()[0]), b
            if fixed[b] is not None:
                assert np.array_equal(got_frames[b][fixed[b] >= 0], fixed[b][fixed[b] >= 0]), b
            alone.close()
    finally:
        job.close()
        m.set_backend(1)


# ---------------------------------------------------------------- 6: timings through the public interface
PHRASES = ["hɛloʊ wɜːld", "a", "", "ðɪs ɪz ɐ tˈɛst.", "kəmpjˈuːtɚ"]


def _quiet(m):
    m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.0, 1.0, 0.0))


@pytest.mark.parametrize("voice", ["medium", "x_low"])
def test_alignment_of_phoneme_strings(voices, voice):
    m = voices(voice)
    _quiet(m)
    try:
        plain = [a.samples.as_slice().copy() for a in m.speak_batch(PHRASES)]
        res = m.speak_batch_with_alignment(PHRASES)
        for ph, (audio, al), ref in zip(PHRASES, res, plain):
            wav = audio.samples.as_slice()
            assert np.array_equal(wav, ref)
            assert audio.info.sample_rate == (16000 if voice == "x_low" else 22050)
            ids, src = m.phonemes_to_input_ids_map(ph)
            kept = sorted(set(c for c in src if c >= 0))
            assert [a.phoneme for a in al] == ["^"] + [ph[c] for c in kept] + ["$"]
            assert al[0].start_sample == 0 and al[-1].start_sample + al[-1].num_samples == len(wav)
            assert all(x.start_sample + x.num_samples == y.start_sample for x, y in zip(al, al[1:]))
            assert all(a.num_samples % HOP == 0 for a in al)
        # per-character scales: 0 silences a character, and the other characters keep their place in the order
        ph = PHRASES[0]
        sc = [0.0 if ch == "l" else 1.5 for ch in ph]
        audio, al = m.speak_batch_with_alignment([ph], duration_scales=[sc])[0]
        assert all(a.num_samples == 0 for a in al if a.phoneme == "l")
        assert al[-1].start_sample + al[-1].num_samples == len(audio)
        ids, src = m.phonemes_to_input_ids_map(ph)
        id_sc = [1.0 if c < 0 else sc[c] for c in src]
        (ref_audio, ref_frames), = m.infer_batch_with_durations([ids], duration_scales=[id_sc])
        assert np.array_equal(audio.samples.as_slice(), ref_audio.samples.as_slice())
        assert [a.num_samples for a in al][1:-1] == [HOP * int(ref_frames[2 * k + 1] + ref_frames[2 * k + 2])
                                                      for k in range(len(al) - 2)]
    finally:
        m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.667, 1.0, 0.8))


def test_all_zero_utterance_is_one_frame(voices):
    m = voices("medium")
    _quiet(m)
    try:
        batches = [_ids(n, 600 + i) for i, n in enumerate((9, 40))]
        res = m.infer_batch_with_durations(batches, durations=[np.zeros(9, np.int32), None])
        (a0, f0), (a1, f1) = res
        assert not f0.any() and len(a0) == HOP                          # the y_len clamp: sum 0 -> one frame
        assert int(f1.sum()) * HOP == len(a1)
        alone = m.infer_batch_with_values([batches[1]])[0]
        assert np.array_equal(a1.samples.as_slice(), alone.samples.as_slice())
    finally:
        m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.667, 1.0, 0.8))


@pytest.mark.parametrize("voice", ["medium", "medium4"])
def test_latent_p_duration_equals_job_id_frames(voices, voice):
    path = voices.paths[voice]
    sm = sonata_b200.VitsStreamingModel(path, device=0)
    m = voices(voice)
    rng = np.random.default_rng(4)
    batches = [_ids(n, 700 + i) for i, n in enumerate((5, 130, 33))]
    cfgs = [PiperSynthesisConfig(3 if voice == "medium4" else None, 0.0, ls, 0.0) for ls in (1.0, 0.8, 1.3)]
    scales = [None, rng.uniform(0.5, 2, 130).astype(np.float32), None]
    fixed = [np.array([2, 0, 7, -1, 1], np.int32), None, None]
    try:
        encs = sm.infer_encoder_batch(batches, cfgs, duration_scales=scales, durations=fixed)
        job = SynthesisJob(m, batches, configs=cfgs)
        job.set_durations(scales, fixed)
        job.run()
        frames = job.id_frames()
        for b, e in enumerate(encs):
            assert e.p_duration.dtype == np.int32 and np.array_equal(e.p_duration, frames[b]), b
            assert int(e.p_duration.sum()) == e.num_frames == job.lengths()[0][b], b
        job.close()
        plain = sm.infer_encoder_batch(batches, cfgs)
        job = SynthesisJob(m, batches, configs=cfgs)
        job.run()
        assert all(np.array_equal(e.p_duration, f) for e, f in zip(plain, job.id_frames()))
        job.close()
        del encs, plain
    finally:
        sm.close()


# ---------------------------------------------------------------- 7: errors
def _raw_set(job, scales, frames):
    err = N.sb200_error()
    sc = None if scales is None else np.ascontiguousarray(scales, np.float32)
    fr = None if frames is None else np.ascontiguousarray(frames, np.int32)
    from sonata_b200.piper import _check, _ptr
    _check(job._lib.sb200_job_set_durations(job._h, _ptr(sc, C.c_float), _ptr(fr, C.c_int32), C.byref(err)), err)


def test_bad_controls_raise_and_leave_the_job_as_it_was(voices):
    m = voices("medium")
    _quiet(m)
    batches = [_ids(n, 800 + i) for i, n in enumerate((20, 31, 12))]
    total = sum(len(b) for b in batches)
    job = SynthesisJob(m, batches)
    with pytest.raises(OperationError, match="has not run"):
        job.id_frames()
    good = [np.full(20, 1.3, np.float32), None, np.full(12, 0.7, np.float32)]
    job.set_durations(good, [None, np.full(31, 4, np.int32), None])
    job.run()
    before = [a.samples.as_slice().copy() for a in job.fetch()]
    before_frames = job.id_frames()
    # the library's own checks (the raw entry point, past Python's)
    for bad, msg in ((np.nan, "nan"), (np.inf, "inf"), (-0.5, "-0.5")):
        sc = np.ones(total, np.float32)
        sc[20 + 31 + 4] = bad
        with pytest.raises(OperationError, match=f"utterance 2, id 4: duration scale {msg}"):
            _raw_set(job, sc, None)
    fr = np.full(total, -1, np.int32)
    fr[20 + 7] = -2
    with pytest.raises(OperationError, match="utterance 1, id 7: fixed duration -2"):
        _raw_set(job, None, fr)
    # Python's checks, before any native call
    with pytest.raises(OperationError, match="utterance 0: 19 duration scales for 20 ids"):
        job.set_durations([np.ones(19)] + [None] * 2)
    with pytest.raises(OperationError, match="utterance 1, id 3: duration scale nan"):
        job.set_durations([None, [1.0] * 3 + [float("nan")] + [1.0] * 27, None])
    with pytest.raises(OperationError, match="utterance 2, id 0: fixed duration -5"):
        job.set_durations(None, [None, None, [-5] + [0] * 11])
    job.run()
    assert all(np.array_equal(a.samples.as_slice(), b) for a, b in zip(job.fetch(), before))
    assert all(np.array_equal(x, y) for x, y in zip(job.id_frames(), before_frames))
    out = np.zeros(total, np.int32)
    err = N.sb200_error()
    from sonata_b200.piper import _check, _ptr
    with pytest.raises(OperationError, match=f"capacity {total - 1} is smaller than the job's {total} ids"):
        _check(job._lib.sb200_job_id_frames(job._h, _ptr(out, C.c_int32), total - 1, C.byref(err)), err)
    job.set_durations(None, None)                                  # back to the default
    job.run()
    plain = m.infer_batch_with_values(batches)
    assert all(np.array_equal(a.samples.as_slice(), p.samples.as_slice()) for a, p in zip(job.fetch(), plain))
    job.close()
    m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.667, 1.0, 0.8))
