"""GPU (-m gpu): per-utterance noise seeds.

A seeded utterance's eps_w / eps_z are keyed Philox draws of its seed, the tensor, the row within the utterance and the
column (tests/noise_reference.py restates them), so under default noise it comes out bit for bit as itself run alone,
whatever shares its batch, on every backend, call and voice handle; unseeded utterances keep their positional noise
bit for bit."""
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import noise_reference as nr
import sonata_b200
from oracle import vits_oracle as vo
from sonata_b200 import OperationError, PiperSynthesisConfig, voicegen, workload
from sonata_b200.job import SynthesisJob
from sonata_b200.piper import StreamBatch

pytestmark = pytest.mark.gpu

DEFAULT = PiperSynthesisConfig(None, 0.667, 1.0, 0.8)
CAPTURES = ("eps_w", "eps_z", "logw", "z_p", "z")
QUALITY = {"medium4": "medium", "high3": "high", "x_low3": "x_low", "medium": "medium"}


@pytest.fixture(scope="module")
def voices(lib_built):
    d = voicegen.default_voice_dir()
    paths = {"medium4": voicegen.write_voice(d, "medium", n_speakers=4),
             "high3": voicegen.write_voice(d, "high", n_speakers=3),
             "x_low3": voicegen.write_voice(d, "x_low", n_speakers=3),
             "medium": voicegen.write_voice(d, "medium")}
    ms = {}

    def get(name):
        if name not in ms:
            ms[name] = sonata_b200.from_config_path(paths[name], device=0)
        return ms[name]
    get.paths = paths
    yield get
    for m in ms.values():
        m.close()


def _ids(n, utt):
    return workload.synthetic_ids(n // 2 + 1, utt=utt)[:n]


def _close_to_reference(got, ref):
    """Within 8 float32 ulp of the float64 value, plus 2^-30."""
    ref32 = np.abs(ref).astype(np.float32)
    tol = 8.0 * np.spacing(ref32).astype(np.float64) + 2.0 ** -30
    err = np.abs(got.astype(np.float64) - ref)
    return bool((err <= tol).all()), float(err.max()) if err.size else 0.0


def _run(m, batches, configs=None, seeds=None, durations=None, scales=None):
    job = SynthesisJob(m, batches, debug=True, configs=configs, seeds=seeds)
    if durations is not None or scales is not None:
        job.set_durations(scales, durations)
    job.run()
    wavs = job.fetch()
    i16 = job.fetch_i16()
    out = []
    for b in range(len(batches)):
        r = {"wav": wavs[b].samples.as_slice().copy(), "cum": job.durations(b), "i16": i16[b]}
        for name in CAPTURES:
            try:
                r[name] = job.debug_fetch(name, b)
            except OperationError:          # a noise tensor no utterance of the pass scales by more than 0
                assert name.startswith("eps_")
        out.append(r)
    job.close()
    return out


def _same(a, b, what):
    """Equal bits in every capture both runs have (a pass draws a noise tensor only when some utterance uses it)."""
    assert {"wav", "cum", "i16", "logw", "z_p", "z"} <= set(a) & set(b)
    for k in set(a) & set(b):
        assert a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), (what, k)


# ---------------------------------------------------------------- 1. the draws
FRAMES = (1, 127, 128, 129, 257, 3)
SEEDS = (0, 1, 2**64 - 1, 0x0123456789ABCDEF, None, 77)


def test_seeded_draws_equal_the_host_restatement_on_every_backend(voices):
    """Frame counts fixed through the duration controls: 1, 127, 128, 129, 257 frames put segment ends on both sides of
    the 128-frame granule; one utterance is unseeded and utterance lengths are odd and even (id-level gap rows)."""
    m = voices("medium")
    inter = voicegen.ARCH["medium"]["inter"]
    batches = [_ids(n, 300 + i) for i, n in enumerate((5, 64, 33, 130, 7, 1))]
    durations = [[f] + [0] * (len(ids) - 1) for ids, f in zip(batches, FRAMES)]
    caps = {}
    try:
        for backend in (1, 0, 2):
            m.set_backend(backend)
            caps[backend] = _run(m, batches, [DEFAULT] * len(batches), list(SEEDS), durations)
    finally:
        m.set_backend(1)
    for b, (ids, f, s) in enumerate(zip(batches, FRAMES, SEEDS)):
        got_w, got_z = caps[1][b]["eps_w"], caps[1][b]["eps_z"]
        assert got_w.shape == (len(ids), 2) and got_z.shape == (f, inter), b
        assert np.array_equal(caps[1][b]["cum"], np.full(len(ids), f)), b
        if s is None:           # positional noise: each run on the handle is a new call
            continue
        for backend in (0, 2):
            assert np.array_equal(caps[backend][b]["eps_w"], got_w) and np.array_equal(caps[backend][b]["eps_z"], got_z)
        ok, err = _close_to_reference(got_w, nr.eps_w(s, len(ids)))
        assert ok, (b, "eps_w", err)
        ok, err = _close_to_reference(got_z, nr.eps_z(s, f, inter))
        assert ok, (b, "eps_z", err)


# ---------------------------------------------------------------- 2. batch independence under default noise
def _cases(n_speakers):
    spk = lambda s: None if n_speakers <= 1 else s % n_speakers
    cfgs = [PiperSynthesisConfig(spk(1), 0.667, 1.0, 0.8), PiperSynthesisConfig(spk(3), 0.8, 0.8, 0.6),
            PiperSynthesisConfig(None, 0.667, 1.25, 0.8), PiperSynthesisConfig(spk(2), 0.5, 1.0, 0.8),
            PiperSynthesisConfig(spk(0), 0.667, 1.0, 0.0), PiperSynthesisConfig(spk(2), 0.0, 1.1, 0.8)]
    lens = [23, 64, 9, 130, 41, 17]
    seeds = [11, None, 2**64 - 5, 11, None, 123456789]
    return lens, cfgs, seeds


@pytest.mark.parametrize("voice,backend", [("medium4", 1), ("medium4", 0), ("medium4", 2), ("high3", 1), ("x_low3", 1)])
def test_seeded_utterance_in_a_batch_equals_itself_alone(voices, voice, backend):
    m = voices(voice)
    m.set_backend(backend)
    lens, cfgs, seeds = _cases(int(voice[-1]))
    batches = [_ids(n, 400 + i) for i, n in enumerate(lens)]
    scales = [None] * len(lens)
    scales[3] = np.linspace(0.5, 1.5, lens[3]).tolist()          # duration controls on one seeded utterance
    try:
        batch = _run(m, batches, cfgs, seeds, scales=scales)
        for b in (0, 2, 3, 5):                                     # first, middle and last positions
            alone = _run(m, [batches[b]], [cfgs[b]], [seeds[b]], scales=[scales[b]])[0]
            _same(batch[b], alone, (voice, backend, b))
        # utterances 0 and 3 share a seed: their first frames hold the same noise (prefix stability)
        n = min(batch[0]["eps_z"].shape[0], batch[3]["eps_z"].shape[0])
        assert np.array_equal(batch[0]["eps_z"][:n], batch[3]["eps_z"][:n])
        # reversed order: the seeded utterances keep their bits
        rev = _run(m, batches[::-1], cfgs[::-1], seeds[::-1], scales=scales[::-1])
        for b in (0, 2, 3, 5):
            _same(batch[b], rev[len(lens) - 1 - b], (voice, backend, "reversed", b))
    finally:
        m.set_backend(1)


# ---------------------------------------------------------------- 3. reproducible across calls and handles
def test_same_seed_same_bits_across_calls_and_handles(voices):
    m = voices("medium")
    other = sonata_b200.from_config_path(voices.paths["medium"], device=0)
    batches = [_ids(n, 500 + i) for i, n in enumerate((31, 12, 57))]
    try:
        first = m.infer_batch_with_values(batches, seeds=[7, 8, 9])
        again = m.infer_batch_with_values(batches, seeds=[7, 8, 9])
        there = other.infer_batch_with_values(batches, seeds=[7, 8, 9])
        for a, b, c in zip(first, again, there):
            assert np.array_equal(a.samples.as_slice(), b.samples.as_slice())
            assert np.array_equal(a.samples.as_slice(), c.samples.as_slice())
        diff = m.infer_batch_with_values(batches[:1], seeds=[70])[0].samples.as_slice()
        same = first[0].samples.as_slice()
        assert diff.shape != same.shape or float(np.abs(diff - same).max()) > 1e-3
        # the other entry points agree with each other
        ph = m.speak_batch(["hɛloʊ", "wɜld"], seeds=[5, 6])
        ids = [m.phonemes_to_input_ids(p) for p in ("hɛloʊ", "wɜld")]
        ref = m.infer_batch_with_values(ids, seeds=[5, 6])
        assert all(np.array_equal(a.samples.as_slice(), b.samples.as_slice()) for a, b in zip(ph, ref))
        al = m.speak_batch_with_alignment(["hɛloʊ"], seeds=[5])
        assert np.array_equal(al[0][0].samples.as_slice(), ref[0].samples.as_slice())
    finally:
        other.close()


# ---------------------------------------------------------------- 4. unseeded utterances keep their bits
def test_unseeded_neighbours_keep_their_positional_noise(voices):
    path = voices.paths["medium"]
    a = sonata_b200.from_config_path(path, device=0)
    b = sonata_b200.from_config_path(path, device=0)
    batches = [_ids(n, 600 + i) for i, n in enumerate((20, 45, 9, 70))]
    try:
        plain = _run(a, batches, [DEFAULT] * 4)                       # first call on each handle: same call counter
        half = _run(b, batches, [DEFAULT] * 4, seeds=[None, 3, None, 4])
        for i in (0, 2):
            _same(plain[i], half[i], ("unseeded", i))
        assert not np.array_equal(plain[1]["eps_w"], half[1]["eps_w"])
    finally:
        a.close()
        b.close()


def test_seed_errors_leave_the_job_as_it_was(voices):
    m = voices("medium")
    batches = [_ids(n, 700 + i) for i, n in enumerate((15, 26))]
    job = SynthesisJob(m, batches, seeds=[1, 2])
    job.run()
    before = [x.samples.as_slice().copy() for x in job.fetch()]
    with pytest.raises(OperationError, match="utterance 1"):
        job.set_seeds([1, -3])
    job.run()
    after = [x.samples.as_slice().copy() for x in job.fetch()]
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
    job.close()
    inj = SynthesisJob(m, batches, eps_w=[np.zeros((15, 2), np.float32), None])
    with pytest.raises(OperationError, match="utterance 1: a noise seed on a job with injected"):
        inj.set_seeds([None, 4])
    inj.set_seeds(None)
    inj.close()


# ---------------------------------------------------------------- 5. against the oracle
MARGIN = 1e-3
ORACLE_CASE = [(14, 3, 0.8), (30, 0, 1.0), (9, None, 1.25), (22, 1, 1.0)]    # phonemes, speaker, length_scale


def _oracle_case(W, W64, a, n, spk, ls, utt, seed0):
    """The first seed from seed0 up whose durations stay MARGIN away from the ceil cliff in fp32 and fp64."""
    ids = vo.synthetic_ids(n, utt=utt)
    for seed in range(seed0, seed0 + 40):
        ew = nr.eps_w(seed, len(ids)).astype(np.float32)
        tw = torch.from_numpy(ew.T.copy()).view(1, 2, -1)
        st = {}
        vo.infer(W, ids, [0.0, ls, 0.8], eps_w=tw, stages=st, sid=spk)
        fr = st["w"].view(-1).double()
        ok = float(torch.minimum(fr - torch.floor(fr), torch.ceil(fr) - fr).min()) >= MARGIN
        st64 = {}
        vo.infer(W64, ids, [0.0, ls, 0.8], eps_w=tw.double(), stages=st64, sid=spk)
        fr64 = st64["w"].view(-1)
        ok = ok and float(torch.minimum(fr64 - torch.floor(fr64), torch.ceil(fr64) - fr64).min()) >= MARGIN
        if not ok:
            continue
        ez = torch.from_numpy(nr.eps_z(seed, st["y_len"], a["inter"]).astype(np.float32).T.copy()).unsqueeze(0)
        ref = {}
        vo.infer(W, ids, [0.667, ls, 0.8], eps_w=tw, eps_z=ez, stages=ref, sid=spk)
        return ids, seed, ref
    raise AssertionError("no screened seed")


@pytest.mark.parametrize("backend", [1, 0])
def test_seeded_batch_against_oracle(voices, backend):
    from test_gpu_parity import TOL_LOGW_MAX, TOL_STAGE, TOL_WAV
    m = voices("medium4")
    m.set_backend(backend)
    tensors = voicegen.make_tensors("medium", n_speakers=4)
    W, W64 = vo.to_torch(tensors), vo.to_torch(tensors, dtype=torch.float64)
    a = vo.arch_of(W)
    cases = [_oracle_case(W, W64, a, n, spk, ls, 800 + b, 1000 * b) for b, (n, spk, ls) in enumerate(ORACLE_CASE)]
    batches = [c[0] for c in cases]
    configs = [PiperSynthesisConfig(spk, 0.667, ls, 0.8) for _, spk, ls in ORACLE_CASE]
    job = SynthesisJob(m, batches, debug=True, configs=configs, seeds=[c[1] for c in cases])
    tm = lambda t: t[0].T.numpy()
    try:
        job.run()
        wavs = job.fetch()
        for b, (_, _, st) in enumerate(cases):
            ref_cum = np.cumsum(st["w_ceil"].view(-1).numpy()).astype(np.int64)
            assert np.array_equal(job.durations(b).astype(np.int64), ref_cum), b
            pairs = [("logw", job.debug_fetch("logw", b), tm(st["logw"]), TOL_LOGW_MAX),
                     ("z_p", job.debug_fetch("z_p", b), tm(st["z_p"]), TOL_STAGE),
                     ("z", job.debug_fetch("z", b), tm(st["z"]), TOL_STAGE),
                     ("wav", wavs[b].samples.as_slice(), st["wav"].view(-1).numpy(), TOL_WAV)]
            for name, got, ref, tol in pairs:
                assert got.shape == ref.shape, (b, name)
                err = float(np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64)).max())
                assert err < tol, (b, name, err)
    finally:
        job.close()
        m.set_backend(1)


# ---------------------------------------------------------------- 6. streaming
def test_seeded_latents_equal_alone_and_the_synthesis_z(voices):
    m = voices("medium")
    from sonata_b200.piper import VitsStreamingModel
    s = VitsStreamingModel(voices.paths["medium"], device=0)
    batches = [_ids(n, 900 + i) for i, n in enumerate((25, 60, 11))]
    seeds = [21, None, 22]
    try:
        encs = s.infer_encoder_batch(batches, seeds=seeds)
        full = _run(m, batches, seeds=seeds)
        for b in (0, 2):
            alone = s.infer_encoder_batch([batches[b]], seeds=[seeds[b]])[0]
            got = encs[b].infer_decoder().as_slice()
            assert np.array_equal(got, alone.infer_decoder().as_slice())
            assert encs[b].num_frames == full[b]["z"].shape[0]
            assert np.array_equal(got, full[b]["wav"]), b     # decoder of the latent == the seeded synthesis
    finally:
        s.close()


@pytest.mark.parametrize("noise", [(0.0, 0.0), (0.667, 0.8)])
def test_seeded_stream_batch_equals_stream_synthesis(voices, noise):
    from sonata_b200.piper import VitsStreamingModel
    s = VitsStreamingModel(voices.paths["medium"], device=0)
    s.set_fallback_synthesis_config(PiperSynthesisConfig(None, noise[0], 1.0, noise[1]))
    sentences = ["hɛloʊ wɜld ðɪs ɪz ɐ tɛst", "ʃɔɹt", "ɐ lɔŋɡɚ sɛntəns ðæt ɡoʊz ɔn fɔɹ ɐ waɪl"]
    seeds = [31, None, 32]
    try:
        sb = StreamBatch(s, 45, 3)
        keys = [sb.add(p, seed=sd) for p, sd in zip(sentences, seeds)]
        got = {k: [] for k in keys}
        while len(sb):
            for k, a in sb.step():
                got[k].append(a.as_slice().copy())
        for k, p, sd in zip(keys, sentences, seeds):
            if sd is None:
                continue
            want = [a.as_slice().copy() for a in s.stream_synthesis(p, 45, 3, seed=sd)]
            assert len(got[k]) == len(want) and all(np.array_equal(x, y) for x, y in zip(got[k], want)), k
    finally:
        s.close()


def test_bench_seeds_runs(tmp_path):
    import subprocess
    env = dict(os.environ, SONATA_B200_VOICE_DIR=str(tmp_path))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_seeds.py"), "--steps", "1", "--warmup", "1",
                        "--rounds", "1", "--utts", "4", "--phonemes", "24"], capture_output=True, text=True, env=env,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    arms = [json.loads(line)["arm"] for line in r.stdout.splitlines() if '"arm"' in line]
    assert arms == ["a_unseeded", "b_seeded", "c_half"]
