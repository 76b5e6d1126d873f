"""GPU (-m gpu): the text encoder stage by stage against float64 (tests/enc_reference.py), each stage recomputed from the
kernel's own captured input so that errors do not compound:
    ids -> enc.emb -> enc.{l}.qkv -> .att -> .o -> .ln1 -> .ffn1 -> .ffn2 -> .ln2 (l = 0 .. 5) -> stats,
on the medium, high and x_low voices, on backend 1 (3xTF32 contractions, tensor-core attention), backend 1 with the fp32
attention (SB200_ATT_SIMT=1) and backend 0 (fp32 CUDA cores); backend 2 runs the encoder on backend 0's kernels and must
give its captures bit for bit.  x and stats are also held end to end to the float64 encoder chained from the ids.  Run
with -s to print the per-stage tables: max |got - ref|, the yardstick's max error, the largest fraction of the bound and
where, and the same for the first and last id of every utterance."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import enc_reference as er  # noqa: E402
import sonata_b200  # noqa: E402
from sonata_b200 import PiperSynthesisConfig, voicegen, workload  # noqa: E402
from sonata_b200.job import SynthesisJob  # noqa: E402

pytestmark = pytest.mark.gpu

# One job per batch.  T <= w and T = 2w + 1: the clipped relative band; 31 / 32 / 33: the softmax's 32-key zero fill;
# 48: n + HX lands on the 64-id granule; 63 / 64 / 65: granule edges; 127 .. 257: conv_tf's 128-row tiles; 639 .. 1280:
# both softmax register regimes and the tensor-core limit; 1281: the whole job on the fp32 attention.
EDGE_BATCHES = {
    "short": (1, 2, 4, 5, 9, 10, 31, 32, 33, 48, 63, 64, 65),
    "tiles": (127, 128, 129, 255, 257, 3),
    "softmax": (639, 640, 641, 1280, 2),
    "fallback": (1281, 33),
}
VOICES = ("medium", "high", "x_low")
# name -> (backend, fp32 attention forced)
CONFIGS = {"b1": (1, False), "b1_fp32att": (1, True), "b0": (0, False)}
TABLE, EDGE, E2E, CAL = {}, {}, {}, {}


@pytest.fixture(scope="module")
def models(lib_built):
    d = voicegen.default_voice_dir()
    ms = {}

    def get(q):
        if q not in ms:
            ms[q] = sonata_b200.from_config_path(voicegen.write_voice(d, q), device=0)
        return ms[q]
    yield get
    for m in ms.values():
        m.close()


_TENSORS = {}


def _tensors(q):
    if q not in _TENSORS:
        _TENSORS[q] = voicegen.make_tensors(q)
    return _TENSORS[q]


def _ids(n, utt):
    return workload.synthetic_ids(n // 2 + 1, utt=utt)[:n]


def _run(m, ids, backend, simt, monkeypatch, debug=True):
    if simt:
        monkeypatch.setenv("SB200_ATT_SIMT", "1")
    else:
        monkeypatch.delenv("SB200_ATT_SIMT", raising=False)
    m.set_backend(backend)
    try:
        job = SynthesisJob(m, ids, debug=debug, configs=[PiperSynthesisConfig(None, 0.0, 1.0, 0.0)] * len(ids))
        job.run()
    finally:
        m.set_backend(1)
        monkeypatch.delenv("SB200_ATT_SIMT", raising=False)
    return job


def _captures(job, t, utts, ids):
    """Per utterance: every enc.* capture, x, stats and the ids.  On the tensor-core attention path V reaches only the
    transposed capture enc.{l}.vt, which takes the place of qkv's V columns."""
    a = er.arch(t)
    H = a["hidden"]
    names = [s[0] for s in er.stages(t)]
    out = []
    for b in utts:
        c = {n: job.debug_fetch(n, b) for n in names}
        c["x"] = job.debug_fetch("x", b)
        c["ids"] = np.asarray(ids[b])
        for l in range(a["layers"]):
            try:
                vt = job.debug_fetch(f"enc.{l}.vt", b)
            except sonata_b200.OperationError:
                continue
            c[f"enc.{l}.qkv"] = c[f"enc.{l}.qkv"].copy()
            c[f"enc.{l}.qkv"][:, 2 * H:] = vt.T
            c[f"enc.{l}.vt"] = vt
        out.append(c)
    return out


def _stacked(fn, xs, ar_):
    """fn over every utterance's input at once: conv and LayerNorm stages are row-local (k = 3 reads one row each
    side), so the inputs go one zero row apart and the output is cut back into utterances."""
    tup = isinstance(xs[0], tuple)
    parts = list(zip(*xs)) if tup else [xs]
    lens = [np.asarray(x[0] if tup else x).shape[0] for x in xs]
    cat = []
    for p in parts:
        rows = []
        for x in p:
            x = er._np(x)
            rows += [x, np.zeros((1, x.shape[1]))]
        cat.append(np.concatenate(rows))
    y = er._np(fn(tuple(cat) if tup else cat[0], ar_))
    out, r = [], 0
    for n in lens:
        out.append(y[r:r + n])
        r += n + 1
    return out


def _eval(t, stage, xs, mode):
    name, src, kind, fn = stage
    if kind == "att":
        return [er._np(fn(x, er.Arith(mode))) for x in xs]
    if kind == "emb":
        return [er._np(fn(x, er.Arith(mode))) for x in xs]
    return _stacked(fn, xs, er.Arith(mode))


def _chain(t, ids_list, mode):
    """The whole encoder from the ids of every utterance, in `mode`'s arithmetic (no captures)."""
    res = [{"ids": np.asarray(i)} for i in ids_list]
    for st in er.stages(t):
        outs = _eval(t, st, [er.inputs(st[1], r) for r in res], mode)
        for r, o in zip(res, outs):
            r[st[0]] = o
    for r in res:
        r["x"] = r[f"enc.{er.arch(t)['layers'] - 1}.ln2"]
    return res


def _record(key, name, e, ey, r, where, edge_r, edge_where):
    row = TABLE.setdefault(key + (name,), [0.0, 0.0, 0.0, ""])
    if r >= row[2]:
        row[2], row[3] = r, where
    row[0], row[1] = max(row[0], e), max(row[1], ey)
    erow = EDGE.setdefault(key + (name,), [0.0, ""])
    if edge_r >= erow[0]:
        erow[:] = [edge_r, edge_where]


def _check_stages(voice, cfg, backend, caps, fails):
    """Every stage of every captured utterance within its bound."""
    t = _tensors(voice)
    stages = er.stages(t)
    for c in caps:
        assert np.array_equal(c["x"], c[stages[-2][0]]), (voice, cfg)          # x is the last layer's ln2
        emb = t["enc_p.emb.weight"].astype(np.float32)[c["ids"]] * np.sqrt(np.float32(emb_h(t)))
        assert np.array_equal(c["enc.emb"], emb), (voice, cfg, len(c["ids"]))   # bit for bit
    for st in stages[1:]:
        name, src, kind, fn = st
        xs = [er.inputs(src, c) for c in caps]
        refs = _eval(t, st, xs, "f64")
        yards = _eval(t, st, xs, er.yardstick(kind, backend))
        for c, ref, yard in zip(caps, refs, yards):
            got = c[name]
            n = len(c["ids"])
            assert got.shape == ref.shape, (voice, cfg, name, got.shape, ref.shape)
            assert np.isfinite(got).all(), (voice, cfg, name, n)
            rb = er.row_bounds(kind, ref, yard, backend)
            err = np.abs(got - ref).max(axis=1)
            r = err / rb
            k = int(np.argmax(r))
            ke = 0 if r[0] >= r[-1] else n - 1
            where = (f"T {n} row {k}" + (f" tile {k // er.TILE}" if kind == "conv" and backend == 1 else "") +
                     f" |ref| {float(np.abs(ref).max()):.2f}")
            _record((voice, cfg), name, float(err.max()), float(np.abs(yard - ref).max()), float(r[k]), where,
                    float(r[ke]), f"T {n} row {ke}")
            if r[k] > 1.0:
                fails.append((voice, cfg, n, name, where, float(r[k])))


def emb_h(t):
    return np.asarray(t["enc_p.emb.weight"]).shape[1]


def _check_e2e(voice, cfg, backend, caps, fails):
    """x and stats against the float64 encoder chained from the ids, within E2E_MULT x the host chain's own error."""
    t = _tensors(voice)
    ids = [c["ids"] for c in caps]
    key = (voice, tuple(len(i) for i in ids))
    if key + ("f64",) not in _CHAINS:
        _CHAINS[key + ("f64",)] = _chain(t, ids, "f64")
    mode = "emu" if backend == 1 else "f32"
    if key + (mode,) not in _CHAINS:
        _CHAINS[key + (mode,)] = _chain(t, ids, mode)
    for c, ref, yard in zip(caps, _CHAINS[key + ("f64",)], _CHAINS[key + (mode,)]):
        for name in ("x", "stats"):
            e, ec, r = er.e2e_check(c[name], ref[name], yard[name])
            row = E2E.setdefault((voice, cfg, name), [0.0, 0.0, 0.0, ""])
            if r >= row[2]:
                row[2], row[3] = r, f"T {len(c['ids'])}"
            row[0], row[1] = max(row[0], e), max(row[1], ec)
            if r > 1.0:
                fails.append((voice, cfg, len(c["ids"]), "e2e " + name, float(r)))


_CHAINS = {}


def _print(title):
    print(f"\n{title}\n{'voice':7s} {'config':10s} {'stage':12s} {'max|err|':>9s} {'yardstick':>9s} {'of bound':>8s}  "
          f"{'worst':36s} {'edge rows':>9s}  worst edge")
    for key, (e, ey, r, where) in sorted(TABLE.items()):
        er_, ew = EDGE[key]
        print(f"{key[0]:7s} {key[1]:10s} {key[2]:12s} {e:9.2e} {ey:9.2e} {r:8.3f}  {where:36s} {er_:9.3f}  {ew}")
    print(f"end to end\n{'voice':7s} {'config':10s} {'out':6s} {'max|err|':>9s} {'chain':>9s} {'of bound':>8s}  worst")
    for (v, c, n), (e, ec, r, where) in sorted(E2E.items()):
        print(f"{v:7s} {c:10s} {n:6s} {e:9.2e} {ec:9.2e} {r:8.3f}  {where}")
    for v, (ek, ee, f, where) in sorted(CAL.items()):
        print(f"layer-0 fp32 attention {v}: kernel {ek:.2e}, host emulation {ee:.2e}, factor {f:.2f} ({where})")
    TABLE.clear(); EDGE.clear(); E2E.clear(); CAL.clear()


@pytest.mark.parametrize("batch", list(EDGE_BATCHES))
@pytest.mark.parametrize("voice", VOICES)
def test_encoder_stages_at_edge_lengths(models, voice, batch, monkeypatch):
    """One job of EDGE_BATCHES[batch] per configuration: every stage of every utterance within its bound, x and stats
    within the end-to-end bound; backend 2's captures bit for bit backend 0's; and at layer 0, where the fp32 attention
    kernel sees the tensor-core run's Q / K / V bit for bit, its error within ATT_CAL of the host float32 emulation's."""
    m = models(voice)
    t = _tensors(voice)
    a = er.arch(t)
    H = a["hidden"]
    lens = EDGE_BATCHES[batch]
    ids = [_ids(n, 500 + i) for i, n in enumerate(lens)]
    fails, caps = [], {}
    for cfg, (backend, simt) in CONFIGS.items():
        job = _run(m, ids, backend, simt, monkeypatch)
        caps[cfg] = _captures(job, t, range(len(ids)), ids)
        job.close()
        _check_stages(voice, cfg, backend, caps[cfg], fails)
        _check_e2e(voice, cfg, backend, caps[cfg], fails)
    # layer 0: same Q / K / V on both backend-1 runs, so the fp32 kernel's real error calibrates the emulation
    stage = next(s for s in er.stages(t) if s[0] == "enc.0.att")
    for ct, cs in zip(caps["b1"], caps["b1_fp32att"]):
        assert np.array_equal(ct["enc.0.qkv"], cs["enc.0.qkv"]), (voice, len(ct["ids"]))
        ref = er._np(stage[3](cs["enc.0.qkv"], er.Arith("f64")))
        emu = er._np(stage[3](cs["enc.0.qkv"], er.Arith("f32")))
        ulp = 2.0 ** -24 * float(np.abs(ref).max())
        e_k, e_e = float(np.abs(cs["enc.0.att"] - ref).max()), float(np.abs(emu - ref).max())
        f = max((e_k + ulp) / (e_e + ulp), (e_e + ulp) / (e_k + ulp))
        row = CAL.setdefault(voice, [0.0, 0.0, 0.0, ""])
        if f >= row[2]:
            row[:] = [e_k, e_e, f, f"T {len(ct['ids'])}"]
        if f > er.ATT_CAL:
            fails.append((voice, "att0 calibration", len(ct["ids"]), e_k, e_e))
    # backend 2: the encoder on backend 0's kernels, bit for bit
    job = _run(m, ids, 2, False, monkeypatch)
    c2 = _captures(job, t, range(len(ids)), ids)
    job.close()
    for u0, u2 in zip(caps["b0"], c2):
        for k, v in u0.items():
            assert np.array_equal(v, u2[k]), (voice, "backend 2", len(u0["ids"]), k)
    _print(f"{voice}, batch {lens}")
    assert not fails, fails


@pytest.mark.parametrize("voice,batch,phonemes", [("medium", 32, 256), ("high", 1, 512)])
def test_encoder_stages_full_size(models, voice, batch, phonemes, monkeypatch):
    """The production launch sizes on backend 1: every stage of utterances 0, 1, the middle one and the last within its
    bound, and x / stats end to end."""
    m = models(voice)
    t = _tensors(voice)
    ids = [workload.synthetic_ids(phonemes, utt=200 + i) for i in range(batch)]
    job = _run(m, ids, 1, False, monkeypatch)
    utts = sorted({0, 1 % batch, batch // 2, batch - 1})
    caps = _captures(job, t, utts, ids)
    job.close()
    torch.cuda.empty_cache()
    fails = []
    _check_stages(voice, "b1", 1, caps, fails)
    _check_e2e(voice, "b1", 1, caps, fails)
    _print(f"{voice} {batch} x {phonemes} phonemes, utterances {utts}")
    assert not fails, fails


@pytest.mark.parametrize("backend", [1, 0])
def test_captures_change_nothing(models, backend, monkeypatch):
    """A debug job and a plain job of the same batch give the same durations and waveforms, bit for bit."""
    m = models("medium")
    ids = [_ids(n, 600 + i) for i, n in enumerate(EDGE_BATCHES["short"] + (257,))]
    out = []
    for debug in (True, False):
        job = _run(m, ids, backend, False, monkeypatch, debug=debug)
        out.append(([job.durations(b) for b in range(len(ids))], [w.samples.as_slice().copy() for w in job.fetch()]))
        job.close()
    for b in range(len(ids)):
        assert np.array_equal(out[0][0][b], out[1][0][b]), b
        assert np.array_equal(out[0][1][b], out[1][1][b]), b
