"""GPU (-m gpu): Piper's 16 kHz qualities through the C ABI.  x_low (96-wide encoder and flow, 48-wide attention heads
on the tensor-core attention, coupling halves of 48 channels zero-padded to 96 at load) and low (the medium
architecture at 16 kHz) against the oracle and the goldens of tests/golden/qualities/, the 48-wide attention against
float64, the bit-identity properties the medium voice is held to, streaming, and the libsonata facade at 16 kHz."""
import ctypes as C
import glob
import json
import os
import sys
import wave

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import sonata_b200  # noqa: E402
from oracle import vits_oracle as vo  # noqa: E402
from sonata_b200 import PiperSynthesisConfig, voicegen, workload  # noqa: E402
from sonata_b200.job import SynthesisJob  # noqa: E402

pytestmark = pytest.mark.gpu
BACKENDS = [1, 0]
TOL_WAV = 1e-3
TOL_STAGE = 2e-4
TOL_LOGW_MAX = 2e-3
TOL_LOGW_MEDIAN = 1e-5
QGOLD = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "qualities", "*.npz")))


def _stage_tol(name):
    return TOL_WAV if name == "wav" else TOL_LOGW_MAX if name == "logw" else TOL_STAGE


@pytest.fixture(scope="module")
def qpaths(lib_built):
    d = voicegen.default_voice_dir()
    return {q: voicegen.write_voice(d, q) for q in ("x_low", "low")}


@pytest.fixture(scope="module")
def models(qpaths):
    ms = {}

    def get(q):
        if q not in ms:
            ms[q] = sonata_b200.from_config_path(qpaths[q], device=0)
        return ms[q]
    yield get
    for m in ms.values():
        m.close()


def _det(m):
    m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.0, 1.0, 0.0))


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("path", QGOLD, ids=[os.path.basename(p) for p in QGOLD])
def test_cuda_matches_quality_goldens(path, backend, models):
    g = np.load(path)
    m = models(str(g["quality"]))
    m.set_backend(backend)
    assert m.audio_output_info().sample_rate == 16000
    sc = g["scales"]
    m.set_fallback_synthesis_config(PiperSynthesisConfig(None, float(sc[0]), float(sc[1]), float(sc[2])))
    ew = [g["eps_w"]] if "eps_w" in g else None
    ez = [g["eps_z"]] if "eps_z" in g else None
    job = SynthesisJob(m, [g["ids"]], ew, ez, debug=True)
    job.run()
    frames, samples, _ = job.lengths()
    assert np.array_equal(job.durations(0), g["cum"]), "durations must be exact"
    assert frames[0] == int(g["y_len"]) and samples[0] == 256 * int(g["y_len"])
    assert float(np.abs(job.debug_fetch("z", 0) - g["z"]).max()) < TOL_STAGE
    a = job.fetch()[0]
    assert a.info.sample_rate == 16000
    assert float(np.abs(a.samples.as_slice() - g["wav"]).max()) < TOL_WAV
    job.close()
    m.set_backend(1)


def _check_report(rep, seeds=None):
    for i, u in enumerate(rep["utts"]):
        if seeds is not None:
            assert u["ceil_margin"] >= 1e-3 and u["y_len_ref"] == seeds[i][1], ("screening is stale", u)
        assert u["durations_exact"] and u["y_len_ref"] == u["y_len_got"], u
        names = [s[0] for s in u["stages"]]
        assert {"x", "stats", "logw", "z_p", "z", "dec.pre", "dec.mrf0", "wav"} <= set(names), names
        for name, err, ref_max in u["stages"]:
            assert err != "SHAPE" and err < _stage_tol(name), (name, err, u["n_ids"])
        assert u["logw_median_err"] < TOL_LOGW_MEDIAN, u["logw_median_err"]


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("quality,ns,noise", [("x_low", (16, 40, 5, 0, 1), False), ("x_low", (9, 21), True),
                                               ("low", (12, 3), False)])
def test_every_stage_against_oracle_16k(quality, ns, noise, backend):
    from stage_report import stage_report
    _check_report(stage_report(quality, ns, noise, backend=backend, verbose=False))


# (seed, frames) from `python tests/screen_margin.py x_low <phonemes> <count>`: every duration >= 1e-3 from the ceil()
# cliff in the fp32 oracle and its fp64 shadow
SCREENED_X_LOW = {
    "C1": (128, [(0, 713)]),                                        # 1 x 128 phonemes, T_x = 258
    "C2": (256, [(0, 1503), (2, 1490), (5, 1480), (14, 1464)]),     # 4 x 256 phonemes in ONE batch, T_x = 514
}


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("cfg", list(SCREENED_X_LOW))
def test_x_low_baseline_sizes_against_oracle(cfg, backend):
    from stage_report import stage_report
    n, seeds = SCREENED_X_LOW[cfg]
    rep = stage_report("x_low", [n] * len(seeds), False, backend=backend, verbose=False, utts=[s for s, _ in seeds])
    _check_report(rep, seeds)


def test_x_low_takes_the_tensor_core_attention(models):
    """The default backend runs x_low's 48-wide heads on the tensor-core attention (the capture `p0` of its softmax
    exists), backend 0 on the fp32 kernel; both give the same durations here."""
    m = models("x_low"); _det(m)
    ids = workload.synthetic_ids(30, utt=5)
    cums = []
    for backend, has_p0 in ((1, True), (0, False)):
        m.set_backend(backend)
        job = SynthesisJob(m, [ids], debug=True)
        job.run()
        try:
            job.debug_fetch("p0", 0)
            got = True
        except sonata_b200.OperationError:
            got = False
        assert got == has_p0, backend
        cums.append(job.durations(0))
        job.close()
    m.set_backend(1)
    assert np.array_equal(cums[0], cums[1])


def _ids_of_length(n, utt):
    return workload.synthetic_ids(n // 2 + 1, utt=utt)[:n]


def _attention_job(m, lens, simt, monkeypatch):
    if simt:
        monkeypatch.setenv("SB200_ATT_SIMT", "1")
    else:
        monkeypatch.delenv("SB200_ATT_SIMT", raising=False)
    ids = [_ids_of_length(n, 300 + i) for i, n in enumerate(lens)]
    job = SynthesisJob(m, ids, debug=True)
    job.run()
    out = []
    for b in range(len(ids)):
        d = {k: job.debug_fetch(k, b) for k in ("qkv0", "att0")}
        for k in ("p0", "vt0"):
            try:
                d[k] = job.debug_fetch(k, b)
            except sonata_b200.OperationError:
                pass
        d["ids"] = ids[b]
        out.append(d)
    job.close()
    monkeypatch.delenv("SB200_ATT_SIMT", raising=False)
    return out


# the lengths of test_gpu_parity.py's test_tensor_core_attention_against_fp64
ATT_JOBS = {
    "nreg20": (1, 2, 31, 32, 33, 63, 65, 97, 127, 128, 129, 255, 257, 639, 640),
    "nreg40": (3, 95, 641, 1279, 1280),
    "fp32_fallback": (1281, 33),
}


@pytest.mark.parametrize("regime", list(ATT_JOBS))
def test_48_wide_attention_against_fp64(regime, models, monkeypatch):
    """Layer 0 of the x_low text encoder (2 heads of 48) against float64, with the bounds of the 96-wide test: Q.K^T over
    K = 48 (the second 32-channel K-block half used, zero-filled in both operands), P.V on 48-column tiles.  p0 keys
    [T, round_up(T, 32)) are exactly zero."""
    import att_reference as ar
    from conv_unit import TF_TOL
    m = models("x_low"); _det(m)
    m.set_backend(1)
    lens = ATT_JOBS[regime]
    t = voicegen.make_tensors("x_low")
    a = voicegen.ARCH["x_low"]
    H, heads, D = a["hidden"], a["heads"], a["hidden"] // a["heads"]
    assert D == 48
    relk, relv = ar.rel_embeddings(t, 0)
    tc = _attention_job(m, lens, False, monkeypatch)
    simt = _attention_job(m, lens, True, monkeypatch)
    on_tc = regime != "fp32_fallback"
    for n, u, s in zip(lens, tc, simt):
        assert ("vt0" in u) == on_tc and ("p0" in u) == on_tc
        q, k = u["qkv0"][:, :H], u["qkv0"][:, H:2 * H]
        v = u["vt0"].T if on_tc else u["qkv0"][:, 2 * H:]
        _, refs = ar.project_qkv(t, 0, u["ids"])
        for got, ref in zip((q, k, v), refs):
            assert float(np.abs(got - ref).max()) < TF_TOL * max(1.0, float(np.abs(ref).max())), n
        assert np.array_equal(s["qkv0"][:, :2 * H], u["qkv0"][:, :2 * H]), n
        assert np.array_equal(s["qkv0"][:, 2 * H:], v), n
        Ps, ref = ar.attention(q, k, v, relk, relv, heads)
        e_tc = float(np.abs(u["att0"] - ref).max())
        e_simt = float(np.abs(s["att0"] - ref).max())
        scale = float(np.abs(ref).max())
        row = {"T": n, "tc": e_tc, "simt": e_simt, "max_ref": scale}
        assert e_simt <= ar.fp32_att_bound(n, scale), row
        assert on_tc or np.array_equal(u["att0"], s["att0"]), n
        assert e_tc <= ar.ATT_MULT * e_simt + ar.ATT_FLOOR * scale, row
        if on_tc:
            p0 = u["p0"]
            tz = (n + 31) // 32 * 32
            assert p0.shape[1] >= tz and not p0[:, n:tz].any(), n
            sums = p0[:, :n].astype(np.float64).sum(1)
            assert float(np.abs(sums - 1.0).max()) <= (n / 32 + 8) * 2.0 ** -23, n
            P32, _ = ar.attention_head(*(np.asarray(x, dtype=np.float32)[:, :D] for x in (q, k, v)),
                                       relk.astype(np.float32), relv.astype(np.float32))
            e_p = float(np.abs(p0[:, :n] - Ps[0]).max())
            e_p32 = float(np.abs(P32 - Ps[0]).max())
            assert e_p <= ar.ATT_MULT * e_p32 + ar.ATT_FLOOR, (row, e_p, e_p32)


def test_x_low_attention_bits_do_not_depend_on_batch(models):
    """Alone (32-key score tiles) and inside a batch of 32 (64-key tiles, wider conv tiles everywhere): att0, p0, logw
    and the durations are bitwise equal.  P.V always runs on 48-column tiles for 48-wide heads."""
    m = models("x_low"); _det(m)
    m.set_backend(1)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    lens = [202 + 2 * (u % 24) for u in range(32)]
    ids = [_ids_of_length(n, 400 + u) for u, n in enumerate(lens)]
    ws = lambda ls: sum(2 * ((n + 255) // 256) * ((n + 63) // 64) for n in ls) * 2 / sms
    assert ws(lens) > 1.3
    job = SynthesisJob(m, ids, debug=True)
    job.run()
    for b in (0, 13, 31):
        assert ws([lens[b]]) < 0.5
        solo = SynthesisJob(m, [ids[b]], debug=True)
        solo.run()
        tz = (lens[b] + 31) // 32 * 32
        for name in ("att0", "p0", "x", "logw", "stats"):
            x, y = job.debug_fetch(name, b), solo.debug_fetch(name, 0)
            if name == "p0":
                x, y = x[:, :tz], y[:, :tz]
            assert np.array_equal(x, y), (b, name, float(np.abs(x - y).max()))
        assert np.array_equal(job.durations(b), solo.durations(0)), b
        solo.close()
    job.close()


def test_x_low_conv_results_do_not_depend_on_tile_width(lib_built):
    """Every x_low conv shape with more than one tile width, once per width its planner picks: bitwise equal rows."""
    from conv_unit import tile_width_launches, width_invariance
    from test_quality_voices import x_low_tc_layers, x_low_tf_layers
    cases = [(1,) + lay for lay in x_low_tc_layers()] + [(2,) + lay for lay in x_low_tf_layers()]
    ran = 0
    for case in cases:
        if len(tile_width_launches(*case)) < 2:
            continue
        launches, res = width_invariance(*case)
        for nt, rows, same in res:
            assert same, (case, launches, nt, rows)
        ran += 1
    assert ran >= 6, ran


def test_x_low_batched_equals_sequential(models):
    m = models("x_low"); _det(m)
    m.set_backend(1)
    batches = [workload.synthetic_ids(n, utt=50 + i) for i, n in enumerate((30, 7, 64, 18))]
    together = m.infer_batch_with_values(batches)
    for b, ids in enumerate(batches):
        alone = m.infer_with_values(ids)
        assert np.array_equal(alone.samples.as_slice(), together[b].samples.as_slice())


@pytest.mark.parametrize("reversed_", [False, True])
def test_padded_coupling_layers_equal_unpadded(lib_built, reversed_):
    """The loader widens x_low's coupling pre (48 -> 96 input channels) and post (48 -> 96 output channels) with exact
    zeros.  On the fp32 backend they give the same bits as the unpadded layers: pre against its 48 input channels (run
    as one whole 64-channel K-block of the fp32 kernel, the last 16 channels zero), post on the target half, and post
    leaves the conditioning half of z as it was.  A 48-channel input the fp32 kernel refuses outright."""
    from conv_unit import run_conv
    g = torch.Generator().manual_seed(11)
    rows, H, half = 300, 96, 48
    z = torch.randn(rows, 2 * half, generator=g)
    cond, tgt = (slice(half, 2 * half), slice(0, half)) if reversed_ else (slice(0, half), slice(half, 2 * half))
    w_pre, b_pre = torch.randn(H, half, 1, generator=g) / 7, torch.randn(H, generator=g) * 0.1
    w_post, b_post = torch.randn(half, H, 1, generator=g) / 10, torch.randn(half, generator=g) * 0.1
    y = np.zeros((rows, H), np.float32)
    assert "multiple of 32" in run_conv(0, z[:, cond].contiguous(), w_pre, b_pre, 1, y0=y)
    x64, w64 = torch.zeros(rows, 64), torch.zeros(H, 64, 1)
    x64[:, :half], w64[:, :half] = z[:, cond], w_pre
    y_u = np.zeros((rows, H), np.float32)
    assert not run_conv(0, x64, w64, b_pre, 1, y0=y_u)
    wp = torch.zeros(H, 2 * half, 1); wp[:, cond] = w_pre
    y_p = np.zeros((rows, H), np.float32)
    assert not run_conv(0, z, wp, b_pre, 1, y0=y_p)
    assert np.array_equal(y_u, y_p)
    ref = z[:, cond].double() @ w_pre[:, :, 0].double().T + b_pre.double()
    assert float(np.abs(y_p - ref.numpy()).max()) < 1e-5
    # post: z[:, tgt] -= post(h)
    h = torch.randn(rows, H, generator=g)
    zu = z[:, tgt].contiguous().numpy().copy()
    assert not run_conv(0, h, w_post, b_post, 1, scale=-1.0, y0=zu, acc0=True)
    wq = torch.zeros(2 * half, H, 1); wq[tgt] = w_post
    bq = torch.zeros(2 * half); bq[tgt] = b_post
    zp = z.numpy().copy()
    assert not run_conv(0, h, wq, bq, 1, scale=-1.0, y0=zp, acc0=True)
    assert np.array_equal(zp[:, tgt], zu) and np.array_equal(zp[:, cond], z.numpy()[:, cond])


def test_x_low_streaming_chunks_match_oracle(qpaths, tmp_path):
    cfg = json.load(open(qpaths["x_low"], encoding="utf-8"))
    cfg["streaming"] = True
    p = tmp_path / "rt.onnx.json"
    json.dump(cfg, open(p, "w", encoding="utf-8"), ensure_ascii=False)
    os.symlink(qpaths["x_low"].replace(".onnx.json", ".svw"), tmp_path / "rt.svw")
    m = sonata_b200.from_config_path(str(p), device=0)
    assert isinstance(m, sonata_b200.VitsStreamingModel)
    _det(m)
    W = vo.to_torch(voicegen.make_tensors("x_low"))
    ids = workload.synthetic_ids(60, utt=77)
    st = {}
    full_ref = vo.infer(W, ids, [0, 1, 0], stages=st).numpy()
    enc = m.infer_encoder(ids)
    assert enc.num_frames == st["y_len"]
    assert float(np.abs(enc.infer_decoder().as_slice() - full_ref).max()) < TOL_WAV
    chunks = list(sonata_b200.SpeechStreamer(enc, 45, 3))
    assert len(chunks) > 1
    total = 0
    for ((m0, m1), (a0, a1)), got in zip(sonata_b200.AdaptiveMelChunker(enc.num_frames, 45, 3), chunks):
        hi = enc.num_frames if m1 is None else m1
        ref = vo.decode(W, st["z"][:, :, m0:hi]).view(-1).numpy()
        ref = ref[a0:a1] if a1 is not None else ref[a0:]
        exp = sonata_b200.AudioSamples(ref); exp.crossfade(42)
        assert float(np.abs(got.as_slice() - exp.as_slice()).max()) < TOL_WAV
        total += len(got)
    assert total == 256 * enc.num_frames
    m.close()


def test_facade_on_a_16k_voice(lib_built, qpaths, tmp_path):
    """libsonata on the low voice: AudioInfo says 16 kHz, appended silence is counted in 16 kHz samples, and the WAV
    written by speak-to-file has a 16 kHz header."""
    from test_libsonata_facade import CALLBACK, AudioInfoC, ExternError, SynthesisEvent, SynthesisParams
    lib = lib_built
    lib.libsonataLoadVoiceFromConfigPath.restype = C.c_void_p
    lib.libsonataLoadVoiceFromConfigPath.argtypes = [C.c_char_p, C.POINTER(ExternError)]
    lib.libsonataSpeak.argtypes = [C.c_void_p, C.c_char_p, SynthesisParams, C.POINTER(ExternError)]
    lib.libsonataSpeakToFile.argtypes = [C.c_void_p, C.c_char_p, SynthesisParams, C.c_char_p, C.POINTER(ExternError)]
    lib.libsonataSpeakToFile.restype = C.c_uint8
    lib.libsonataGetAudioInfo.argtypes = [C.c_void_p, C.POINTER(AudioInfoC), C.POINTER(ExternError)]
    lib.libsonataFreeSynthesisEvent.argtypes = [SynthesisEvent]
    lib.libsonataUnloadSonataVoice.argtypes = [C.c_void_p]
    err = ExternError()
    v = lib.libsonataLoadVoiceFromConfigPath(qpaths["low"].encode(), C.byref(err))
    assert v and err.code == 0
    ai = AudioInfoC()
    lib.libsonataGetAudioInfo(v, C.byref(ai), C.byref(err))
    assert (ai.sample_rate, ai.num_channels, ai.sample_width) == (16000, 1, 2)
    events = []

    def cb(ev):
        pcm = np.ctypeslib.as_array(ev.data, shape=(max(ev.len, 1),))[:ev.len].copy()
        events.append((ev.event_type, pcm.view("<i2")))
        lib.libsonataFreeSynthesisEvent(ev)
        return 0
    text = "hɛloʊ wɜːld\nðɪs ɪz ə tɛst".encode("utf-8")
    sil = 30 * 16000 // 1000
    lib.libsonataSpeak(v, text, SynthesisParams(1, 10, 100, 50, 30, CALLBACK(cb), 0), C.byref(err))
    assert err.code == 0 and events[-1][0] == 1
    speech = [e[1] for e in events[:-1]]
    assert len(speech) == 2
    for s in speech:
        assert (len(s) - sil) % 256 == 0 and len(s) > sil and not s[-sil:].any() and s[:-sil].any()
    out = tmp_path / "o.wav"
    ok = lib.libsonataSpeakToFile(v, text, SynthesisParams(1, 10, 100, 50, 50, CALLBACK(cb), 0), str(out).encode(), C.byref(err))
    assert ok == 1
    with wave.open(str(out)) as w:
        assert w.getframerate() == 16000 and w.getnchannels() == 1 and w.getsampwidth() == 2
        n = w.getnframes()
    assert (n - 2 * (50 * 16000 // 1000)) % 256 == 0
    lib.libsonataUnloadSonataVoice(v)


def test_imported_x_low_voice_loads_and_speaks(lib_built, tmp_path):
    """`python -m sonata_b200.onnx_import` on a self-written x_low ONNX file: the voice it writes loads through
    `from_config_path`, reports 16 kHz and speaks what the oracle computes from the same tensors."""
    import subprocess
    from test_quality_voices import _onnx_voice
    onnx, cfg, tensors = _onnx_voice(tmp_path, "x_low", seed=5)
    out = subprocess.run([sys.executable, "-m", "sonata_b200.onnx_import", onnx, cfg, str(tmp_path / "out")],
                         cwd=ROOT, capture_output=True, text=True, check=True).stdout.strip().splitlines()[-1]
    m = sonata_b200.from_config_path(out, device=0)
    _det(m)
    assert m.audio_output_info().sample_rate == 16000
    ids = workload.synthetic_ids(20, utt=4)
    got = m.infer_with_values(ids)
    ref = vo.infer(vo.to_torch(tensors), ids, [0.0, 1.0, 0.0]).numpy()
    assert got.info.sample_rate == 16000 and got.samples.as_slice().shape == ref.shape
    assert float(np.abs(got.samples.as_slice() - ref).max()) < TOL_WAV
    m.close()
