"""GPU (-m gpu): the CUDA path, called through the C ABI, against the oracle and the committed
golden vectors.  Two-stage check everywhere (SURVEY facts 3-4): durations EXACT, then waveform
sample-wise max-abs < 1e-3 (the tolerance BASELINE.json states; measured error is ~1e-5)."""
import glob
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))      # conv_unit.py (kernel unit cases, torch reference only)
sys.path.insert(0, os.path.join(ROOT, "tests"))      # stage_report.py (uses the oracle: test infrastructure)

import sonata_b200
from oracle import vits_oracle as vo
from sonata_b200 import PiperSynthesisConfig, voicegen, workload
from sonata_b200.job import SynthesisJob

pytestmark = pytest.mark.gpu
# Test ids stay stable across hardware ports: "tcgen05" names backend 1, the tensor-core backend (wgmma on sm_90a).
BACKEND_IDS = ["tcgen05", "fp32simt"]
TOL_WAV = 1e-3          # BASELINE.json: "waveform max-abs error <1e-3"
TOL_STAGE = 2e-4        # per-stage activations are O(1..5); fp32 path measures ~1e-5
# logw comes out of three inverse rational-quadratic spline flows whose derivative may be as small as 1e-3 (the
# graph's min_derivative), i.e. the INVERSE amplifies its input error by up to 1e3 at a few ids per utterance (the
# fp32 oracle itself is 1.1e-4 away from its fp64 shadow there).  So logw is held to a tight
# MEDIAN and a loose max; what the graph consumes -- ceil(exp(logw)) -- is compared exactly.
TOL_LOGW_MAX = 2e-3
TOL_LOGW_MEDIAN = 1e-5


def _stage_tol(name):
    return TOL_WAV if name == "wav" else TOL_LOGW_MAX if name == "logw" else TOL_STAGE
GOLD = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz")))


@pytest.fixture(scope="module")
def models(voice_paths):
    ms = {}

    def get(q):
        if q not in ms:
            ms[q] = sonata_b200.from_config_path(voice_paths[q], device=0)
        return ms[q]
    yield get
    for m in ms.values():
        m.close()


def _det(m):
    m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.0, 1.0, 0.0))


@pytest.mark.parametrize("backend", [1, 0], ids=BACKEND_IDS)
@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p) for p in GOLD])
def test_cuda_matches_golden_vectors(path, backend, models):
    g = np.load(path)
    q = os.path.basename(path).split("_")[0]
    m = models(q)
    m.set_backend(backend)
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
    wav = job.fetch()[0].samples.as_slice()
    assert float(np.abs(wav - g["wav"]).max()) < TOL_WAV
    job.close()
    m.set_backend(1)


@pytest.mark.parametrize("backend", [1, 0], ids=BACKEND_IDS)
@pytest.mark.parametrize("quality,ns,noise", [("medium", (16, 40, 5, 0, 1), False), ("medium", (9, 21), True),
                                               ("high", (12, 3), False)])
def test_every_stage_against_oracle(quality, ns, noise, backend):
    from stage_report import stage_report
    rep = stage_report(quality, ns, noise, backend=backend, verbose=False)
    for u in rep["utts"]:
        assert u["durations_exact"] and u["y_len_ref"] == u["y_len_got"], u
        names = [s[0] for s in u["stages"]]
        assert "wav" in names and "z" in names and "dec.mrf0" in names
        for name, err, ref_max in u["stages"]:
            assert err != "SHAPE", (name, u)
            assert err < _stage_tol(name), (name, err, u["n_ids"])
        assert u["logw_median_err"] < TOL_LOGW_MEDIAN, u["logw_median_err"]


# Full-size parity (BASELINE.json configs): utterance seeds screened by tests/screen_margin.py so that every duration
# w = exp(logw) stays >= 1e-3 away from an integer in the fp32 oracle AND its fp64 shadow -- there ceil(w) is well
# defined and the frame counts must match EXACTLY.  (seed, frames) pairs as printed by the screening script.
MARGIN = 1e-3
SCREENED = {
    "C1": ("medium", 128, [(2, 854)]),                                   # 1 x 128 phonemes, T_x = 258
    "C2": ("medium", 256, [(0, 1783), (1, 1794), (2, 1742), (5, 1819)]),  # 4 x 256 phonemes in ONE batch, T_x = 514
    "C3": ("high", 512, [(3, 3559)]),                                    # 1 x 512 phonemes, T_x = 1026
}


@pytest.mark.parametrize("backend", [1, 0], ids=BACKEND_IDS)
@pytest.mark.parametrize("cfg", ["C1", "C2", "C3"])
def test_baseline_sizes_against_oracle(cfg, backend):
    """The CUDA path against the oracle at the BASELINE.json utterance sizes: durations exact, every stage
    (x, stats, logw, z_p, z, dec.pre, every dec.up*/dec.mrf*) < 2e-4, waveform < 1e-3.  Exercises the multi-tile
    attention path (T_x = 514 / 1026), the block scan of the duration kernel over long segments and the
    frame-level gap logic at 1.8k / 3.5k-frame segments."""
    from stage_report import stage_report
    quality, n, seeds = SCREENED[cfg]
    rep = stage_report(quality, [n] * len(seeds), False, backend=backend, verbose=False, utts=[s for s, _ in seeds])
    for u, (seed, frames) in zip(rep["utts"], seeds):
        assert u["n_ids"] == 2 * n + 2
        assert u["ceil_margin"] >= MARGIN, ("screening is stale: re-run tests/screen_margin.py", u["utt"], u["ceil_margin"])
        assert u["y_len_ref"] == frames, ("oracle frame count moved", u)
        assert u["durations_exact"] and u["y_len_got"] == frames, (cfg, seed, u["flipped_ids"], u["y_len_got"], frames)
        names = [s[0] for s in u["stages"]]
        assert {"x", "stats", "logw", "z_p", "z", "dec.pre", "dec.mrf0", "wav"} <= set(names), names
        for name, err, ref_max in u["stages"]:
            assert err != "SHAPE", (name, u)
            assert err < _stage_tol(name), (cfg, seed, name, err)
        assert u["logw_median_err"] < TOL_LOGW_MEDIAN, (cfg, seed, u["logw_median_err"])


@pytest.mark.parametrize("backend", [1, 0], ids=BACKEND_IDS)
def test_multi_speaker_voice_against_oracle(backend, voice_paths):
    """SURVEY §8f row N1: a multi-speaker voice (`emb_g`, `dp.cond`, the WaveNets' `cond_layer`, `dec.cond`) -- the graph
    the reference feeds the `sid` tensor to whenever num_speakers > 1 (piper/src/lib.rs:353-358).  Every stage against
    the oracle for two speakers, and the speakers must differ."""
    from stage_report import stage_report
    waves = {}
    for sid in (0, 3):
        rep = stage_report("medium", (21, 40), False, backend=backend, verbose=False, n_speakers=4, sid=sid)
        for u in rep["utts"]:
            assert u["durations_exact"] and u["y_len_ref"] == u["y_len_got"], (sid, u)
            for name, err, ref_max in u["stages"]:
                assert err != "SHAPE" and err < _stage_tol(name), (sid, name, err)
        waves[sid] = [u["y_len_got"] for u in rep["utts"]]
    cfg = voicegen.write_voice(voicegen.default_voice_dir(), "medium", n_speakers=4)
    m = sonata_b200.from_config_path(cfg, device=0)
    assert m.get_speakers() == {i: f"speaker_{i}" for i in range(4)} and m.speaker_name_to_id("speaker_2") == 2
    ids = workload.synthetic_ids(30, utt=9)
    outs = []
    for sid in (None, 0, 2):                                   # speaker: None -> sid 0 (`unwrap_or(0)`)
        m.set_fallback_synthesis_config(PiperSynthesisConfig(sid, 0.0, 1.0, 0.0))
        outs.append(m.infer_with_values(ids).samples.as_slice().copy())
    assert np.array_equal(outs[0], outs[1])
    assert outs[2].shape != outs[1].shape or float(np.abs(outs[2] - outs[1]).max()) > 1e-2
    with pytest.raises(sonata_b200.OperationError):
        m.set_fallback_synthesis_config(PiperSynthesisConfig(9, 0.0, 1.0, 0.0))     # piper/src/lib.rs:215-231
    m.close()


def test_unscreened_duration_flips_are_cliff_cases():
    """Companion of the screened test: 8 x 256-phoneme utterances with ARBITRARY seeds.  A frame count may differ
    from the oracle's only where the oracle's own duration sits on the ceil() cliff (margin < 1e-3, where fp32
    and fp64 disagree among themselves in ~2 % of C2 batches); everywhere else durations are exact and the
    waveform is within tolerance.  The flip counts are reported (gpurun_out/flip_report.json), not failed on."""
    import json
    from stage_report import stage_report
    seeds = list(range(100, 108))
    rep = stage_report("medium", [256] * len(seeds), False, backend=1, verbose=False, utts=seeds)
    out = []
    for u in rep["utts"]:
        out.append({k: u[k] for k in ("utt", "n_ids", "ceil_margin", "durations_exact", "flipped_ids", "y_len_ref", "y_len_got")})
        if u["ceil_margin"] >= MARGIN:
            assert u["durations_exact"], u
        if u["durations_exact"]:
            wav = [s for s in u["stages"] if s[0] == "wav"][0]
            assert wav[1] < TOL_WAV, u
        else:
            assert u["flipped_ids"] <= 2 and abs(u["y_len_ref"] - u["y_len_got"]) <= u["flipped_ids"], u
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "flip_report.json"), "w") as f:
        json.dump({"margin": MARGIN, "utts": out, "flipped_utts": sum(not o["durations_exact"] for o in out)}, f, indent=1)


@pytest.mark.parametrize("backend", [1, 0], ids=BACKEND_IDS)
def test_conv_kernels_against_torch(backend, lib_built):
    """Kernel-level unit check of both contraction backends (same ConvArgs contract): 1x1 / dilated k-tap,
    leaky-ReLU prologue, gate / ReLU / residual / scale / accumulate epilogues, masked rows (exactly 0, or untouched
    under accumulate), and launches of the wgmma kernel on both sides of each tile-narrowing edge."""
    from conv_unit import CASES, run_case
    for c in CASES:
        err, msg = run_case(backend, *c)
        assert err is not None, (c, msg)
        assert err < 1e-4, (c, err)


def _supported(backend, cin, cout, k, dil, act, res, acc):
    if backend == 0:
        return True
    import ctypes
    from sonata_b200 import _native
    o = (ctypes.c_int32 * 16)()
    return _native.lib().sb200_debug_plan(backend, 4096, cin, cout, k, dil, act, int(res), int(acc), o) == 0


@pytest.mark.parametrize("backend", [1, 0, 2], ids=BACKEND_IDS + ["tf32x3"])
def test_conv_multi_segment_row_map(backend, lib_built):
    """Several segments with gap rows in one launch, through the engine's row map (segment end per granule, seg_mul rows
    per frame at decoder levels): ragged ends inside a 128-row tile, a segment shorter than the conv's halo.  Gap rows
    come out exactly 0, or keep their (non-zero) prior contents bit for bit under accumulate."""
    from conv_unit import SEG_CASES, TF_TOL, run_segments
    ran = 0
    for lens, gran, seg_mul, cin, cout, k, dil, slope, act, res, scale, acc in SEG_CASES:
        if not _supported(backend, cin, cout, k, dil, act, res, acc):
            continue
        err, gaps_ok = run_segments(backend, lens, gran, seg_mul, cin, cout, k, dil, slope, act, res, scale, acc)
        assert gaps_ok, (lens, gran, seg_mul, cin, cout, k, acc)
        assert err < (TF_TOL if backend == 2 else 1e-4), (lens, gran, seg_mul, cin, cout, k, err)
        ran += 1
    assert ran >= 3


@pytest.mark.parametrize("backend", [1, 0, 2], ids=BACKEND_IDS + ["tf32x3"])
def test_conv_split_outputs(backend, lib_built):
    """The two-buffer epilogue of the flow's WaveNet res/skip layers: columns [0, H) accumulate into the residual
    stream, [H, 2H) into the skip sum (written on the first layer, accumulated after), each half checked on its own.
    The 3xTF32 kernel has no split epilogue (the encoder never splits): its planner must refuse the launch."""
    from conv_unit import SPLIT_CASES, run_split
    if backend == 2:
        with pytest.raises(AssertionError, match="not supported"):
            run_split(2, *SPLIT_CASES[0], 0)
        return
    for lens, H, k in SPLIT_CASES:
        for acc1 in (0, 1):
            (e0, g0), (e1, g1) = run_split(backend, lens, H, k, acc1)
            assert g0 and g1, (lens, acc1, g0, g1)
            assert e0 < 1e-4 and e1 < 1e-4, (lens, acc1, e0, e1)


def test_conv_results_do_not_depend_on_tile_width(lib_built):
    """Bit-identity across tile widths at kernel level: each flow / decoder shape (bf16x2) and encoder shape (3xTF32) runs
    once per column-tile width its planner can choose (row counts found by asking the planner, on this device's SM
    count), the larger launches fed the same leading rows.  Every output row whose receptive field lies inside all
    inputs must be bitwise equal: a wgmma m64nNk16 / k8 gives an output element the same bits at every N."""
    from conv_unit import WIDTH_CASES, width_invariance
    for case in WIDTH_CASES:
        launches, res = width_invariance(*case)
        assert len(launches) >= 2, (case, launches)
        for nt, rows, same in res:
            assert same, (case, launches, nt, rows)


def test_conv_tf_kernel_fp32_class_accuracy(lib_built):
    """conv_tf.cu (wgmma 3xTF32, chunk-flushed accumulation) on every encoder / duration-predictor shape against an
    fp64 reference: the kernel replaces fp32 CUDA-core GEMMs in front of the ceil() cliff, so it is held to the
    error of an fp32 FMA chain (measured 2e-6 .. 1e-5), not to the 1e-4 of the bf16x2 decoder kernel."""
    from conv_unit import TF_CASES, TF_TOL, run_case
    for c in TF_CASES:
        err, msg = run_case(2, *c)
        assert err is not None, (c, msg)
        assert err < TF_TOL, (c, err)


def _ids_of_length(n, utt):
    """n ids (any n, odd included): a synthetic utterance cut to length."""
    return workload.synthetic_ids(n // 2 + 1, utt=utt)[:n]


def _attention_job(m, lens, simt, monkeypatch):
    """Layer-0 attention captures of one job on the medium voice (debug run), per utterance."""
    if simt:
        monkeypatch.setenv("SB200_ATT_SIMT", "1")
    else:
        monkeypatch.delenv("SB200_ATT_SIMT", raising=False)
    ids = [_ids_of_length(n, 300 + i) for i, n in enumerate(lens)]
    job = SynthesisJob(m, ids, debug=True)
    job.run()
    out = []
    for b in range(len(ids)):
        d = {k: job.debug_fetch(k, b) for k in ("qkv0", "att0", "x", "logw")}
        for k in ("p0", "vt0"):
            try:
                d[k] = job.debug_fetch(k, b)
            except sonata_b200.OperationError:
                pass
        d["ids"], d["cum"] = ids[b], job.durations(b)
        out.append(d)
    job.close()
    monkeypatch.delenv("SB200_ATT_SIMT", raising=False)
    return out


# One job per softmax regime of the tensor-core attention (rows in 20 / 40 registers, kernels_misc.cu), lengths batched so
# segment offsets and gap rows are exercised: T = 1, odd T, T = 32k +- 1 (the softmax zero-fills keys to the next multiple
# of 32, the K extent of P.V), T <= 128 (the second 128-row m-tile of a tile pair has no valid row), T = 640 / 641; and
# T = 1281, past the tensor-core attention's limit, on the fp32 attention.
ATT_JOBS = {
    "nreg20": (1, 2, 31, 32, 33, 63, 65, 97, 127, 128, 129, 255, 257, 639, 640),
    "nreg40": (3, 95, 641, 1279, 1280),
    "fp32_fallback": (1281, 33),
}


@pytest.mark.parametrize("regime", list(ATT_JOBS))
def test_tensor_core_attention_against_fp64(regime, models, monkeypatch):
    """Layer 0 of the text encoder on the default backend against float64 (tests/att_reference.py):
    * q / k / v projection, V through its transposed store, against x0 . Wqkv^T + b at the 3xTF32 conv tolerance;
    * the same job with SB200_ATT_SIMT=1 (V stored untransposed by the same conv kernel): Q / K and V bit for bit;
    * att0 of the fp32 CUDA-core attention (the SB200_ATT_SIMT=1 run, and both runs of the job past 1280 ids, which
      takes that kernel whatever the setting) against the fp64 attention of the kernel's own Q / K / V, within the
      T-scaled fp32 bound att_reference.fp32_att_bound;
    * att0 of the tensor-core attention, both heads, against the same reference, within
      ATT_MULT x (the fp32 attention's error on the same inputs) + ATT_FLOOR x max|ref|;
    * head-0 probabilities p0 against the fp64 softmax, within ATT_MULT x the error of a float32 softmax computed on the
      host + ATT_FLOOR (absolute; probabilities are <= 1), zero keys [T, round_up(T, 32)), rows summing to 1 within a
      T-scaled few ulp.  For p0 the floor is what binds: measured 0 .. 5.3e-7 against a float32 host error of
      0 .. 1.5e-7, while a score GEMM on a single TF32 MMA or two of its three split products is off by 1e-4 or more.
    att0 errors measured on an H100 SXM are listed beside ATT_MULT in tests/att_reference.py.  Run with -s to print the
    per-utterance table."""
    import att_reference as ar
    from conv_unit import TF_TOL
    m = models("medium"); _det(m)
    lens = ATT_JOBS[regime]
    t = voicegen.make_tensors("medium")
    a = voicegen.ARCH["medium"]
    H, heads, D = a["hidden"], a["heads"], a["hidden"] // a["heads"]
    relk, relv = ar.rel_embeddings(t, 0)
    tc = _attention_job(m, lens, False, monkeypatch)
    simt = _attention_job(m, lens, True, monkeypatch)
    on_tc = regime != "fp32_fallback"
    report = []
    for n, u, s in zip(lens, tc, simt):
        assert u["qkv0"].shape == (n, 3 * H) and u["att0"].shape == (n, H)
        assert ("vt0" in u) == on_tc and ("p0" in u) == on_tc
        q, k = u["qkv0"][:, :H], u["qkv0"][:, H:2 * H]
        v = u["vt0"].T if on_tc else u["qkv0"][:, 2 * H:]
        _, refs = ar.project_qkv(t, 0, u["ids"])
        for got, ref in zip((q, k, v), refs):
            assert float(np.abs(got - ref).max()) < TF_TOL * max(1.0, float(np.abs(ref).max())), n
        # transposed store: the fp32-attention run stores V untransposed through the same conv_tf kernel
        assert np.array_equal(s["qkv0"][:, :2 * H], u["qkv0"][:, :2 * H]), n
        assert np.array_equal(s["qkv0"][:, 2 * H:], v), n
        Ps, ref = ar.attention(q, k, v, relk, relv, heads)
        e_tc = float(np.abs(u["att0"] - ref).max())
        e_simt = float(np.abs(s["att0"] - ref).max())
        scale = float(np.abs(ref).max())
        bound = ar.ATT_MULT * e_simt + ar.ATT_FLOOR * scale
        row = {"T": n, "tc": e_tc, "simt": e_simt, "max_ref": scale, "bound": bound,
               "simt_bound": ar.fp32_att_bound(n, scale)}
        assert e_simt <= ar.fp32_att_bound(n, scale), row                             # the fp32 kernel on its own
        assert on_tc or np.array_equal(u["att0"], s["att0"]), n                        # past 1280 ids: the same kernel
        assert e_tc <= bound, row
        if on_tc:
            p0 = u["p0"]
            tz = (n + 31) // 32 * 32
            assert p0.shape[1] >= tz and not p0[:, n:tz].any(), n                    # zero-filled keys of the P.V K extent
            sums = p0[:, :n].astype(np.float64).sum(1)
            assert float(np.abs(sums - 1.0).max()) <= (n / 32 + 8) * 2.0 ** -23, (n, float(np.abs(sums - 1.0).max()))
            P32, _ = ar.attention_head(*(np.asarray(x, dtype=np.float32)[:, :D] for x in (q, k, v)),
                                       relk.astype(np.float32), relv.astype(np.float32))
            e_p = float(np.abs(p0[:, :n] - Ps[0]).max())
            e_p32 = float(np.abs(P32 - Ps[0]).max())
            row.update(p0=e_p, p0_fp32=e_p32)
            assert e_p <= ar.ATT_MULT * e_p32 + ar.ATT_FLOOR, row
        report.append(row)
    print(regime, "\n" + "\n".join(" ".join(f"{k}={v:.3g}" if isinstance(v, float) else f"{k}={v}" for k, v in r.items())
                                   for r in report))


def test_attention_bits_do_not_depend_on_batch(models):
    """Utterances synthesised alone (both attention GEMMs on narrow column tiles: 32 keys / 32 head columns) and inside a
    batch of 32 (64 / 96-column tiles, and wider conv tiles everywhere): att0, p0, x, logw and the durations are bitwise
    equal.  The sizes sit far from the width switch of engine.cu create_job (checked below)."""
    m = models("medium"); _det(m)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    lens = [202 + 2 * (u % 24) for u in range(32)]                   # 202 .. 248 ids
    ids = [_ids_of_length(n, 400 + u) for u, n in enumerate(lens)]

    def widths(ls):     # the attention GEMM tile widths create_job picks (2 heads, 96-wide)
        ws = sum(2 * ((n + 255) // 256) * ((n + 63) // 64) for n in ls)
        wo = sum(2 * ((n + 255) // 256) for n in ls)
        return (32 if ws * 2 <= sms else 64), (32 if wo * 3 <= sms else 96), ws * 2 / sms, wo * 3 / sms
    assert widths(lens)[:2] == (64, 96) and min(widths(lens)[2:]) > 1.3
    job = SynthesisJob(m, ids, debug=True)
    job.run()
    for b in (0, 13, 31):
        assert widths([lens[b]])[:2] == (32, 32) and max(widths([lens[b]])[2:]) < 0.5
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


def test_device_i16_matches_host_to_i16_vec(models):
    """SURVEY §8f row N2: the 16-bit PCM conversion (`to_i16_vec`: per-buffer peak normalisation, clamp, truncating cast,
    audio/ops/src/samples.rs:51-75) done on the device is bit-identical to the host mirror of the reference."""
    m = models("medium"); _det(m)
    batches = [workload.synthetic_ids(n, utt=70 + i) for i, n in enumerate((21, 5, 40))]
    job = SynthesisJob(m, batches)
    job.run()
    f32 = job.fetch()
    i16 = job.fetch_i16()
    assert len(i16) == len(f32)
    for a, q in zip(f32, i16):
        ref = a.samples.to_i16_vec()
        assert q.dtype == np.int16 and q.shape == ref.shape
        assert np.array_equal(q, ref)
        assert int(np.abs(q.astype(np.int32)).max()) >= 32766       # peak-normalised


def test_batched_equals_sequential(models):
    """speak_batch is a sequential B=1 loop in the reference (piper/src/lib.rs:433-435): the packed
    batched pass must give each utterance the result it gets alone."""
    m = models("medium"); _det(m)
    batches = [workload.synthetic_ids(n, utt=50 + i) for i, n in enumerate((30, 7, 64, 18))]
    together = m.infer_batch_with_values(batches)
    for b, ids in enumerate(batches):
        alone = m.infer_with_values(ids)
        assert len(alone) == len(together[b])
        assert np.array_equal(alone.samples.as_slice(), together[b].samples.as_slice())     # DESIGN.md §4: same bits


def test_workspace_growth_keeps_results(voice_paths):
    """A context's two device arenas and its pinned staging are sized from each job's own buffers and grow between jobs.
    Jobs run in turn from one thread (so the voice hands back the same context) must give the bits each gets on a
    freshly loaded model, whose workspace fits that job exactly: a short job, 32 x 256 ids at length_scale 3 (both
    arenas and the staging grow), a short debug job (captures added to both levels), the long job again."""
    short = [workload.synthetic_ids(n, utt=90 + i) for i, n in enumerate((12, 30))]
    long_ = [workload.synthetic_ids(256, utt=u) for u in range(32)]
    calls = [(short, 1.0, False), (long_, 3.0, False), (short, 1.0, True), (long_, 3.0, False)]

    def run(m, ids, length_scale, debug):
        m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.0, length_scale, 0.0))
        job = SynthesisJob(m, ids, debug=debug)
        job.run()
        out = [a.samples.as_slice().copy() for a in job.fetch()]
        job.close()
        return out

    fresh = []
    for call in calls:
        m = sonata_b200.from_config_path(voice_paths["medium"], device=0)
        fresh.append(run(m, *call))
        m.close()
    m = sonata_b200.from_config_path(voice_paths["medium"], device=0)
    for call, want in zip(calls, fresh):
        got = run(m, *call)
        assert len(got) == len(want)
        for g, w in zip(got, want):
            assert np.array_equal(g, w)
    m.close()


def test_speak_api_surface(models, oracle_weights):
    m = models("medium"); _det(m)
    ph = "hɛloʊ wɜːld"
    a1 = m.speak_one_sentence(ph)
    a2 = m.infer_with_values(m.phonemes_to_input_ids(ph))
    assert np.array_equal(a1.samples.as_slice(), a2.samples.as_slice())          # deterministic at scales [0,1,0]
    assert a1.info.sample_rate == 22050 and a1.inference_ms > 0 and 0 < a1.real_time_factor() < 1
    ref = vo.infer(oracle_weights("medium"), m.phonemes_to_input_ids(ph), [0, 1, 0]).numpy()
    assert a1.samples.as_slice().shape == ref.shape and float(np.abs(a1.samples.as_slice() - ref).max()) < TOL_WAV
    outs = m.speak_batch([ph, "", "a"])
    assert len(outs) == 3 and len(outs[1]) % 256 == 0 and len(outs[1]) > 0       # "" -> [bos, eos]
    assert len(a1.as_wave_bytes()) == 2 * len(a1)
    # length_scale stretches durations (w = exp(logw) * length_scale)
    m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.0, 1.7, 0.0))
    assert len(m.speak_one_sentence(ph)) > len(a1)
    _det(m)
    with pytest.raises(sonata_b200.OperationError):
        m.infer_with_values([1, 999, 2])                                        # id outside the embedding table


def test_noise_path_statistics(models):
    """Default scales use the on-device Philox source: results differ call to call (like the graph's
    RandomNormalLike) but stay finite, bounded by tanh, and of plausible length."""
    m = models("medium")
    m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.667, 1.0, 0.8))
    ids = workload.synthetic_ids(40, utt=3)
    a, b = m.infer_with_values(ids), m.infer_with_values(ids)
    for x in (a, b):
        s = x.samples.as_slice()
        assert np.isfinite(s).all() and np.abs(s).max() <= 1.0 and len(s) % 256 == 0
        assert 1.5 < len(s) / 256 / len(ids) < 6.0
    n = min(len(a), len(b))
    assert not np.array_equal(a.samples.as_slice()[:n], b.samples.as_slice()[:n])
    _det(m)


def test_full_size_properties(models):
    """BASELINE config 2 (32 x 256 phonemes) at full size through size-independent properties."""
    m = models("medium"); _det(m)
    batches = [workload.synthetic_ids(256, utt=u) for u in range(32)]
    job = SynthesisJob(m, batches)
    ms = job.run()
    frames, samples, offs = job.lengths()
    assert all(s == 256 * f for s, f in zip(samples, frames))
    assert offs == list(np.concatenate([[0], np.cumsum(samples)[:-1]]))
    for b in (0, 17, 31):
        assert int(job.durations(b)[-1]) == frames[b]                           # sum of ceil'd durations == frames
    auds = job.fetch()
    for a in auds:
        s = a.samples.as_slice()
        assert np.isfinite(s).all() and np.abs(s).max() <= 1.0
    # utterance 5 of the big batch == the same utterance alone (batch-size independence)
    alone = m.infer_with_values(batches[5]).samples.as_slice()
    assert np.array_equal(alone, auds[5].samples.as_slice())
    prof = {p["name"]: p for p in job.profile()}
    assert prof["dec.mrf2"]["launches"] == 6 and prof["dec.mrf2"]["ms"] > 0
    assert prof["dec.up2"]["launches"] == 1          # phase-fused ConvTranspose on the tensor-core backend
    assert ms > 0
    job.close()


def test_streaming_chunks_match_oracle(voice_paths, oracle_weights, tmp_path):
    """VitsStreamingModel: encoder half -> z on device; decoder half on frame slices with the
    reference's chunk schedule, overlap trim and crossfade(42) (piper/src/lib.rs:765-858)."""
    import json
    import shutil
    cfg = json.load(open(voice_paths["medium"], encoding="utf-8"))
    cfg["streaming"] = True
    p = tmp_path / "rt.onnx.json"
    json.dump(cfg, open(p, "w", encoding="utf-8"), ensure_ascii=False)
    os.symlink(voice_paths["medium"].replace(".onnx.json", ".svw"), tmp_path / "rt.svw")
    m = sonata_b200.from_config_path(str(p), device=0)
    assert isinstance(m, sonata_b200.VitsStreamingModel) and m.supports_streaming_output()
    _det(m)
    W = oracle_weights("medium")
    ids = workload.synthetic_ids(60, utt=77)
    st = {}
    full_ref = vo.infer(W, ids, [0, 1, 0], stages=st).numpy()
    z = st["z"]
    enc = m.infer_encoder(ids)
    assert enc.num_frames == st["y_len"]
    full = enc.infer_decoder().as_slice()
    assert float(np.abs(full - full_ref).max()) < TOL_WAV
    chunks = list(sonata_b200.SpeechStreamer(enc, 45, 3))
    assert len(chunks) > 1
    total = 0
    for ((m0, m1), (a0, a1)), got in zip(sonata_b200.AdaptiveMelChunker(enc.num_frames, 45, 3), chunks):
        hi = enc.num_frames if m1 is None else m1
        ref = vo.decode(W, z[:, :, m0:hi]).view(-1).numpy()
        ref = ref[a0:a1] if a1 is not None else ref[a0:]
        exp = sonata_b200.AudioSamples(ref); exp.crossfade(42)
        assert float(np.abs(got.as_slice() - exp.as_slice()).max()) < TOL_WAV
        total += len(got)
    assert total == 256 * enc.num_frames
    # one-shot rule: frames <= 2*chunk + 2*pad -> a single full decode (:785, :848-853)
    one = list(sonata_b200.SpeechStreamer(m.infer_encoder(workload.synthetic_ids(8, utt=1)), 72, 3))
    assert len(one) == 1
    m.close()


def test_concurrent_calls_are_reentrant(models):
    """The reference calls `speak_one_sentence` concurrently from rayon workers on ONE model
    (synth/src/lib.rs:316-320): every call must own its stream / workspace."""
    import threading
    m = models("medium"); _det(m)
    sents = [workload.synthetic_ids(n, utt=200 + i) for i, n in enumerate((20, 33, 9, 41, 15, 28, 37, 12))]
    expect = [m.infer_with_values(s).samples.as_slice().copy() for s in sents]
    got = [None] * len(sents)
    errs = []

    def work(i):
        try:
            for _ in range(3):
                got[i] = m.infer_with_values(sents[i]).samples.as_slice().copy()
        except Exception as e:      # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=work, args=(i,)) for i in range(len(sents))]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errs, errs
    for e, g in zip(expect, got):
        assert g is not None and np.array_equal(e, g)


def test_smoke_entry():
    import __graft_entry__ as ge
    ge.smoke()


def test_handles_may_be_freed_in_any_order(voice_paths):
    """A job hands its context back to the voice's pool and a latent belongs to a voice: both share ownership of the
    voice, so a garbage-collected caller that drops the model first does not touch freed memory (seen as
    `std::system_error: Invalid argument` from the pool mutex at interpreter exit)."""
    m = sonata_b200.from_config_path(voice_paths["medium"], device=0)
    _det(m)
    ids = workload.synthetic_ids(64, utt=3)
    job = SynthesisJob(m, [ids]); job.run()
    n = job.lengths()[1][0]
    m.close()                                     # voice handle first ...
    out = job.fetch()[0].samples.as_slice()       # ... the job still owns the weights it reads
    assert out.shape[0] == n and np.isfinite(out).all()
    job.close()
