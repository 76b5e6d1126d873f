"""GPU (-m gpu): speaker blends (include/sonata_b200.h, sb200_speak_batch_ids_blends).

- The device's blended embedding g and effective biases (sb200_debug_speaker_blend) against float64, within bounds
  derived from the kernels' operation counts; g also bit for bit against the numpy statement of the contract.
- Whole passes against the oracle fed the same g (a speaker-embedding row appended to the voice), stage by stage with
  the mixed-batch test's tolerances and exact durations.
- Bit-for-bit identities with seeded noise: one-speaker blends are that speaker, equal canonical forms give equal bits,
  a blended utterance does not depend on its batch, a blend replaces only the config's speaker, jobs without blends keep
  their bits and launches, and a refused set_speaker_blends changes nothing.
- Streams: a StreamBatch of blended and plain streams equals each stream_synthesis, a whole-latent chunk equals the
  blended job, a one-speaker blend stream is the plain speaker's, and chunk passes hold the chunk tests' bounds."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import blend_reference as br  # noqa: E402
import sonata_b200  # noqa: E402
from oracle import vits_oracle as vo  # noqa: E402
from sonata_b200 import OperationError, PiperSynthesisConfig, voicegen, workload  # noqa: E402
from sonata_b200 import _native as N  # noqa: E402
from sonata_b200.job import SynthesisJob  # noqa: E402
from sonata_b200.piper import StreamBatch, _check  # noqa: E402

pytestmark = pytest.mark.gpu

VOICES = {"medium4": ("medium", 4), "high3": ("high", 3), "x_low3": ("x_low", 3)}
DEFAULT = PiperSynthesisConfig(None, 0.667, 1.0, 0.8)
U = 2.0 ** -24


@pytest.fixture(scope="module")
def voices(lib_built):
    d = voicegen.default_voice_dir()
    paths = {k: voicegen.write_voice(d, q, n_speakers=n) for k, (q, n) in VOICES.items()}
    ms = {}

    def get(name, streaming=False):
        key = (name, streaming)
        if key not in ms:
            cls = sonata_b200.VitsStreamingModel if streaming else sonata_b200.VitsModel
            ms[key] = cls(paths[name], device=0)
        ms[key].set_fallback_synthesis_config(DEFAULT)
        ms[key].set_backend(1)
        return ms[key]
    yield get
    for m in ms.values():
        m.close()


_T = {}


def _tensors(name):
    if name not in _T:
        q, n = VOICES[name]
        _T[name] = voicegen.make_tensors(q, n_speakers=n)
    return _T[name]


def _ids(n, utt):
    return workload.synthetic_ids(n // 2 + 1, utt=utt)[:n]


def _hook(m, pairs, rows):
    """(g, biases) of the blend `pairs` as a pass forms them."""
    s = np.array([p[0] for p in pairs], np.int64)
    w = np.array([p[1] for p in pairs], np.float32)
    g = np.zeros(voicegen.GIN_CHANNELS, np.float32)
    b = np.zeros(rows, np.float32)
    err = N.sb200_error()
    _check(m._lib.sb200_debug_speaker_blend(m._h, s.ctypes.data_as(C.POINTER(C.c_int64)),
                                            w.ctypes.data_as(C.POINTER(C.c_float)), len(s),
                                            g.ctypes.data_as(C.POINTER(C.c_float)), g.size,
                                            b.ctypes.data_as(C.POINTER(C.c_float)), b.size, C.byref(err)), err)
    return g, b


def _stacked_cond(T, a):
    """The conditioning weights W [rows][gin] in the order the voice stacks them: dp.cond, each coupling layer's WaveNet
    cond_layer in application order with every layer's 2H rows interleaved (tanh row j, sigmoid row j), then dec.cond.
    Every width here is a multiple of its column tile, so no row is padding."""
    H = a["hidden"]
    perm = np.empty(2 * H, np.int64)
    perm[0::2], perm[1::2] = np.arange(H), H + np.arange(H)
    rows = [T["dp.cond.weight"][:, :, 0]]
    for step in range(a["flow_n"]):
        cw = T[f"flow.flows.{2 * (a['flow_n'] - 1 - step)}.enc.cond_layer.weight"][:, :, 0]
        for l in range(a["wn_layers"]):
            rows.append(cw[2 * H * l + perm])
    rows.append(T["dec.cond.weight"][:, :, 0])
    return np.concatenate(rows).astype(np.float64)


BLENDS = {"two": [(1, 0.7), (2, 0.3)], "three": [(0, 0.25), (1, 1.5), (2, 0.125)]}


def _all_speakers(n):
    return [(k, 1.0 + k) for k in range(n)]


@pytest.mark.parametrize("name", ["medium4", "x_low3"])
def test_blend_g_and_biases_against_float64(voices, name):
    m = voices(name)
    T = _tensors(name)
    a = voicegen.ARCH[VOICES[name][0]]
    Wc = _stacked_cond(T, a)
    E = np.asarray(T["emb_g.weight"], np.float32)
    nspk = VOICES[name][1]
    gin = E.shape[1]
    mdot = (gin + 31) // 32 + 5 + 1          # fmaf terms per lane, the 5 shuffle adds and the bias add
    g0, b0 = _hook(m, [(0, 1.0)], Wc.shape[0])
    assert np.array_equal(g0, E[0])
    for label, pairs in list(BLENDS.items()) + [("all", _all_speakers(nspk))]:
        g, b = _hook(m, pairs, Wc.shape[0])
        s, w = br.canonical(pairs)
        assert np.array_equal(g, br.blend_g(E, s, w)), label           # the contract, bit for bit
        g64, bound = br.blend_g64(E, s, w)
        assert np.all(np.abs(g.astype(np.float64) - g64) <= bound), label
        # biases: the difference to speaker 0's cancels the base; each side's error is its dot product's (gamma_mdot
        # sum |W g|) plus the rounding of its final add (u |b|)
        d_dev = b.astype(np.float64) - b0.astype(np.float64)
        d_ref = Wc @ (g.astype(np.float64) - E[0].astype(np.float64))
        gam = mdot * U / (1 - mdot * U)
        lim = (gam * (np.abs(Wc) @ np.abs(g.astype(np.float64))) + U * np.abs(b)
               + gam * (np.abs(Wc) @ np.abs(E[0].astype(np.float64))) + U * np.abs(b0))
        assert np.all(np.abs(d_dev - d_ref) <= lim * 1.01), (label, float(np.max(np.abs(d_dev - d_ref) / lim)))
        assert float(np.abs(d_dev).max()) > 1e-3, label                 # the blend moved the biases


# ---------------------------------------------------------------------------------------------------- oracle parity
MARGIN = 1e-3


def _oracle_blends(nspk):
    """A 50/50 pair, a 3-speaker blend and an all-speaker blend."""
    return [[(0, 0.5), (nspk - 1, 0.5)], [(0, 0.2), (1, 0.3), (2, 0.5)], [(k, 1.0 + k) for k in range(nspk)]]


ORACLE_SCALES = [(0.667, 1.0, 0.8), (0.0, 1.2, 0.0), (0.667, 0.8, 0.8)]


def _oracle_cases(m, name, rows):
    """Per blend: ids, scales, eps_w, eps_z and the oracle's stages under a voice with g appended as an extra speaker,
    the first candidate utterance whose every duration is at least MARGIN from the ceil() cliff."""
    nspk = VOICES[name][1]
    T = dict(_tensors(name))
    cases = []
    gs = []
    for pairs in _oracle_blends(nspk):
        gs.append((pairs, _hook(m, pairs, rows)[0]))
    T["emb_g.weight"] = np.concatenate([np.asarray(T["emb_g.weight"], np.float32)] + [g[None] for _, g in gs], 0)
    W = vo.to_torch(T)
    a = vo.arch_of(W)
    for b, (pairs, _) in enumerate(gs):
        nsc, ls, nw = ORACLE_SCALES[b]
        for k in range(12):
            ids = vo.synthetic_ids(10 + 7 * b + k, utt=300 + 17 * b + k)
            ew = np.random.default_rng(600 + 31 * b + k).standard_normal((len(ids), 2)).astype(np.float32)
            ew_t = torch.from_numpy(ew.T.copy()).view(1, 2, -1)
            probe = {}
            vo.infer(W, ids, [0.0, ls, nw], eps_w=ew_t, stages=probe, sid=nspk + b)
            w = probe["w"].view(-1).double()
            fr = w - torch.floor(w)
            if float(torch.minimum(fr, 1 - fr).min()) < MARGIN:
                continue
            ez = torch.randn(1, a["inter"], probe["y_len"], generator=torch.Generator().manual_seed(900 + b))
            st = {}
            vo.infer(W, ids, [nsc, ls, nw], eps_w=ew_t, eps_z=ez, stages=st, sid=nspk + b)
            cases.append(dict(ids=ids, pairs=pairs, cfg=PiperSynthesisConfig(None, nsc, ls, nw), ew=ew,
                              ez=ez[0].T.contiguous().numpy(), st=st))
            break
        else:
            raise AssertionError(f"no candidate utterance clears the duration margin for blend {b}")
    return cases, a


@pytest.mark.parametrize("name,backend", [("medium4", 1), ("medium4", 0), ("high3", 1), ("x_low3", 1)])
def test_blended_batch_against_oracle(voices, name, backend):
    from test_gpu_parity import TOL_LOGW_MAX, TOL_STAGE, TOL_WAV
    m = voices(name)
    rows = _stacked_cond(_tensors(name), voicegen.ARCH[VOICES[name][0]]).shape[0]
    cases, a = _oracle_cases(m, name, rows)
    m.set_backend(backend)
    job = SynthesisJob(m, [c["ids"] for c in cases], [c["ew"] for c in cases], [c["ez"] for c in cases], debug=True,
                       configs=[c["cfg"] for c in cases], speaker_blends=[dict(c["pairs"]) for c in cases])
    job.run()
    frames_got = job.lengths()[0]
    wavs = job.fetch()
    tm = lambda t: t[0].T.numpy()
    try:
        for b, c in enumerate(cases):
            st = c["st"]
            ref_cum = np.cumsum(st["w_ceil"].view(-1).numpy()).astype(np.int64)
            assert np.array_equal(job.durations(b).astype(np.int64), ref_cum) and frames_got[b] == st["y_len"], b
            pairs = [("x", job.debug_fetch("x", b), tm(st["x"]), TOL_STAGE),
                     ("stats", job.debug_fetch("stats", b), np.concatenate([tm(st["m_p"]), tm(st["logs_p"])], 1),
                      TOL_STAGE),
                     ("logw", job.debug_fetch("logw", b), tm(st["logw"]), TOL_LOGW_MAX),
                     ("z_p", job.debug_fetch("z_p", b), tm(st["z_p"]), TOL_STAGE),
                     ("z", job.debug_fetch("z", b), tm(st["z"]), TOL_STAGE),
                     ("dec.pre", job.debug_fetch("dec.pre", b), tm(st["dec.pre"]), TOL_STAGE)]
            for i in range(len(a["up_rates"])):
                pairs.append((f"dec.mrf{i}", job.debug_fetch(f"dec.mrf{i}", b), tm(st[f"dec.mrf{i}"]), TOL_STAGE))
            pairs.append(("wav", wavs[b].samples.as_slice(), st["wav"].view(-1).numpy(), TOL_WAV))
            for stage, got, ref, tol in pairs:
                assert got.shape == ref.shape, (b, stage)
                err = float(np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64)).max())
                assert err < tol, (b, stage, err)
    finally:
        job.close()
        m.set_backend(1)


# ---------------------------------------------------------------------------------------------------- identities
def _wavs(m, batches, configs=None, seeds=None, blends=None):
    return [a.samples.as_slice().copy() for a in m.infer_batch_with_values(batches, configs, seeds=seeds,
                                                                            speaker_blends=blends)]


def _same(xs, ys):
    return len(xs) == len(ys) and all(x.shape == y.shape and np.array_equal(x, y) for x, y in zip(xs, ys))


@pytest.mark.parametrize("name", ["medium4", "high3"])
def test_one_speaker_blends_are_that_speaker(voices, name):
    m = voices(name)
    ids = [_ids(n, 10 + i) for i, n in enumerate((40, 90))]
    seeds = [11, 12]
    for s in range(VOICES[name][1]):
        cfg = PiperSynthesisConfig(s, 0.667, 1.1, 0.8)
        ref = _wavs(m, ids, [cfg, cfg], seeds)
        other = PiperSynthesisConfig((s + 1) % VOICES[name][1], 0.667, 1.1, 0.8)
        for blend in ({s: 0.3}, {f"speaker_{s}": 5.0, (s + 1) % VOICES[name][1]: 0.0}):
            assert _same(_wavs(m, ids, [other, other], seeds, [blend, blend]), ref), (s, blend)


def test_equal_canonical_forms_give_equal_bits(voices):
    m = voices("medium4")
    ids = [_ids(n, 20 + i) for i, n in enumerate((33, 120, 64))]
    seeds = [5, 6, 7]
    base = {1: 0.3, 3: 0.7}
    ref = _wavs(m, ids, seeds=seeds, blends=[base] * 3)
    variants = [{3: 0.7, 1: 0.3}, {"speaker_3": 0.7, 0: 0.0, 1: 0.3}, {1: 0.3 * 4, 3: 0.7 * 4},
                {3: np.float32(0.7) / 8, 2: 0.0, 1: np.float32(0.3) / 8}]
    for v in variants:
        assert _same(_wavs(m, ids, seeds=seeds, blends=[v] * 3), ref), v
    # the blend is neither of its speakers, nor the other blend
    assert not _same(_wavs(m, ids, seeds=seeds, blends=[{1: 0.7, 3: 0.3}] * 3), ref)


def test_mixed_batch_equals_each_utterance_alone(voices):
    m = voices("medium4")
    lens = [1, 7, 64, 65, 130, 513, 33, 200, 2, 97, 300, 16]
    ids = [_ids(n, 40 + i) for i, n in enumerate(lens)]
    seeds = [1000 + i for i in range(len(lens))]
    blends = [None, {0: 0.5, 1: 0.5}, {2: 1.0}, {0: 0.5, 1: 0.5}, {3: 0.1, 0: 0.2, 1: 0.3, 2: 0.4}, None,
              {"speaker_1": 0.25, "speaker_2": 0.75}, {0: 0.5, 1: 0.5}, None, {3: 2.0, 2: 1.0}, {2: 1.0, 3: 2.0},
              {1: 1.0}]
    configs = [PiperSynthesisConfig(i % 4 if i % 3 else None, (0.0, 0.667)[i % 2], (0.8, 1.0, 1.3)[i % 3],
                                    (0.0, 0.8)[(i // 2) % 2]) for i in range(len(lens))]
    for backend in (1, 0):
        m.set_backend(backend)
        got = _wavs(m, ids, configs, seeds, blends)
        for b in range(len(lens)):
            assert _same(got[b:b + 1], _wavs(m, [ids[b]], [configs[b]], [seeds[b]], [blends[b]])), (backend, b)
        # the same batch reversed: each utterance keeps its bits next to other neighbours
        rev = _wavs(m, ids[::-1], configs[::-1], seeds[::-1], blends[::-1])
        assert _same(rev[::-1], got), backend
    m.set_backend(1)


def test_the_blend_replaces_only_the_config_speaker(voices):
    m = voices("medium4")
    ids = [_ids(80, 3)]
    blend = [{0: 0.6, 2: 0.4}]
    a = _wavs(m, ids, [PiperSynthesisConfig(3, 0.5, 1.25, 0.6)], [9], blend)
    b = _wavs(m, ids, [PiperSynthesisConfig(None, 0.5, 1.25, 0.6)], [9], blend)
    c = _wavs(m, ids, [PiperSynthesisConfig(1, 0.667, 1.0, 0.8)], [9], blend)
    assert _same(a, b)
    assert a[0].shape != c[0].shape                       # length_scale 1.25 still applies


def _run_counted(m, batches, **kw):
    lib = m._lib
    job = SynthesisJob(m, batches, **kw)
    l0 = lib.sb200_launch_count()
    job.run()
    n = lib.sb200_launch_count() - l0
    out = [a.samples.as_slice().copy() for a in job.fetch()]
    return job, n, out


def test_jobs_without_blends_keep_their_bits_and_launches(voices):
    m = voices("medium4")
    batches = [_ids(n, 60 + i) for i, n in enumerate((40, 90, 17))]
    cfgs = [PiperSynthesisConfig(s, 0.667, 1.0, 0.8) for s in (2, 0, 3)]
    seeds = [1, 2, 3]
    job, n_plain, plain = _run_counted(m, batches, configs=cfgs, seeds=seeds)
    job.close()
    job, n_none, none = _run_counted(m, batches, configs=cfgs, seeds=seeds, speaker_blends=[None] * 3)
    job.set_speaker_blends([{1: 0.5, 2: 0.5}, None, None])
    job.set_speaker_blends(None)
    l0 = m._lib.sb200_launch_count()
    job.run()
    n_reset = m._lib.sb200_launch_count() - l0
    reset = [a.samples.as_slice().copy() for a in job.fetch()]
    job.close()
    assert n_none == n_plain == n_reset and _same(none, plain) and _same(reset, plain)
    # one-speaker blends take the plain path: same launches and bits
    one = [{2: 3.0}, {0: 1.0, 1: 0.0}, {"speaker_3": 0.5}]
    job, n_one, out = _run_counted(m, batches, configs=[PiperSynthesisConfig(None, 0.667, 1.0, 0.8)] * 3, seeds=seeds,
                                   speaker_blends=one)
    job.close()
    assert n_one == n_plain and _same(out, plain)
    # a real blend adds the blend-table launch and nothing else
    job, n_blend, _ = _run_counted(m, batches, configs=cfgs, seeds=seeds, speaker_blends=[{1: 0.5, 2: 0.5}, None, None])
    job.close()
    assert n_blend == n_plain + 1


def test_a_refused_set_speaker_blends_leaves_the_job_as_it_was(voices):
    m = voices("medium4")
    batches = [_ids(n, 80 + i) for i, n in enumerate((30, 50))]
    blends = [{0: 0.4, 3: 0.6}, None]
    job = SynthesisJob(m, batches, seeds=[4, 5], speaker_blends=blends)
    job.run()
    before = [a.samples.as_slice().copy() for a in job.fetch()]
    for bad, msg in (([None, {7: 1.0}], "utterance 1"), ([{1: -1.0}, None], "utterance 0"),
                     ([{1: 0.0, 2: 0.0}, None], "utterance 0"), ([None], "1 entries for 2")):
        with pytest.raises(OperationError, match=msg):
            job.set_speaker_blends(bad)
    # the C call checks every entry before any change, too
    s = np.array([1, 1], np.int64)
    w = np.array([0.5, 0.5], np.float32)
    o = np.array([0, 0, 2], np.uint64)
    err = N.sb200_error()
    rc = m._lib.sb200_job_set_speaker_blends(job._h, s.ctypes.data_as(C.POINTER(C.c_int64)),
                                             w.ctypes.data_as(C.POINTER(C.c_float)),
                                             o.ctypes.data_as(C.POINTER(C.c_size_t)), C.byref(err))
    with pytest.raises(OperationError, match="utterance 1: speaker blend: speaker 1 appears more than once"):
        _check(rc, err)
    job.run()
    after = [a.samples.as_slice().copy() for a in job.fetch()]
    job.close()
    assert _same(before, after)


def test_the_blend_matters(voices):
    m = voices("medium4")
    ids = [_ids(60, 9)]
    cfg = [PiperSynthesisConfig(None, 0.0, 1.0, 0.0)]
    mix = _wavs(m, ids, cfg, [1], [{0: 0.5, 2: 0.5}])[0]
    for s in (0, 2):
        alone = _wavs(m, ids, [PiperSynthesisConfig(s, 0.0, 1.0, 0.0)], [1])[0]
        assert mix.shape != alone.shape or float(np.abs(mix - alone).max()) > 1e-2, s


# ---------------------------------------------------------------------------------------------------- streams
PHONEMES = ["ðə kwɪk braʊn fɒks dʒʌmps", "həloʊ", "ɪt wʌz ðə bɛst ʌv taɪmz ɪt wʌz ðə wɜːst ʌv taɪmz",
            "aɪ æm", "ə lɔːŋ ˈsɛntəns wɪð meni wɜːdz ænd ə lɒt ʌv fɹeɪmz tuː dɪˈkoʊd ɪn tʃʌŋks"]


def test_stream_batch_equals_stream_synthesis(voices):
    sm = voices("medium4", streaming=True)
    cs, pad = 44, 3
    specs = [({0: 0.5, 3: 0.5}, 1), (None, 2), ({1: 0.2, 2: 0.8}, 3), ({"speaker_3": 1.0, 0: 1.0}, 4),
             ({0: 0.5, 3: 0.5}, 5)]
    sb = StreamBatch(sm, cs, pad)
    keys = [sb.add(ph, seed=seed, speaker_blend=bl) for ph, (bl, seed) in zip(PHONEMES, specs)]
    got = {}
    while len(sb):
        for key, a in sb.step():
            assert not isinstance(a, Exception), a
            got.setdefault(key, []).append(a.as_slice().copy())
    for k, ph, (bl, seed) in zip(keys, PHONEMES, specs):
        alone = [a.as_slice().copy() for a in sm.stream_synthesis(ph, cs, pad, seed=seed, speaker_blend=bl)]
        assert _same(got[k], alone), (k, bl)


def test_whole_latent_chunk_equals_the_blended_job(voices):
    m, sm = voices("medium4"), voices("medium4", streaming=True)
    ids = _ids(57, 5)
    blend = {1: 0.35, 3: 0.65}
    ref = _wavs(m, [ids], seeds=[8], blends=[blend])[0]
    enc = sm.infer_encoder_batch([ids], seeds=[8], speaker_blends=[blend])[0]
    got = enc.infer_decoder(0, enc.num_frames).as_slice()
    assert got.shape == ref.shape and np.array_equal(got, ref)
    # the latent keeps its blend: decoded next to plain and other blended latents, it keeps its bits
    others = sm.infer_encoder_batch([_ids(30, 6), _ids(44, 7)], seeds=[1, 2], speaker_blends=[None, {0: 1.0, 2: 1.0}])
    res = sm.infer_decoder_batch([(others[0], 0, others[0].num_frames), (enc, 0, enc.num_frames),
                                  (others[1], 0, others[1].num_frames)])
    assert np.array_equal(res[1].as_slice(), ref)


def test_one_speaker_blend_stream_is_the_plain_speaker(voices):
    sm = voices("medium4", streaming=True)
    ph = PHONEMES[2]
    sm.set_fallback_synthesis_config(PiperSynthesisConfig(2, 0.667, 1.0, 0.8))
    plain = [a.as_slice().copy() for a in sm.stream_synthesis(ph, 44, 3, seed=3)]
    sm.set_fallback_synthesis_config(DEFAULT)
    blended = [a.as_slice().copy() for a in sm.stream_synthesis(ph, 44, 3, seed=3, speaker_blend={2: 0.25})]
    assert _same(plain, blended)


def test_chunk_passes_against_the_oracle_decoder(voices):
    """Chunks of a blended latent through the debug chunk pass, every decoder stage held to the chunk tests' bounds
    (tests/dec_reference.py) under a voice with the blend's g appended as an extra speaker."""
    import test_chunk_decoder_gpu as tcd
    sm = voices("medium4", streaming=True)
    T = _tensors("medium4")
    rows = _stacked_cond(T, voicegen.ARCH["medium"]).shape[0]
    pairs = [(0, 0.3), (1, 0.3), (3, 0.4)]
    g, _ = _hook(sm, pairs, rows)
    Tx = dict(T)
    Tx["emb_g.weight"] = np.concatenate([np.asarray(T["emb_g.weight"], np.float32), g[None]], 0)
    tcd.VOICES["medium4_blend"] = ("medium", 5)
    tcd._TENSORS["medium4_blend"] = Tx
    try:
        enc = sm.infer_encoder_batch([_ids(90, 12)], configs=[PiperSynthesisConfig(None, 0.0, 1.0, 0.0)],
                                     speaker_blends=[dict(pairs)])[0]
        F = enc.num_frames
        chunks = [(enc, 0, F), (enc, 0, 45), (enc, 40, 91), (enc, F - 50, F)]
        fails, table = [], {}
        for backend in (1, 0):
            sm.set_backend(backend)
            caps, _ = tcd._debug_pass(sm, chunks)
            for k, u in enumerate(caps):
                fails += tcd._check_chunk("medium4_blend", backend, u, 4, f"chunk {k}", table)
        assert not fails, fails
    finally:
        sm.set_backend(1)
        del tcd.VOICES["medium4_blend"], tcd._TENSORS["medium4_blend"]
