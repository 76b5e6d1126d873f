"""GPU (-m gpu): streaming decoder chunk passes (decode_chunks: the chunk layout, the latent gather, each chunk's speaker
slot, then the decoder) stage by stage against float64 (tests/dec_reference.py), through the debug chunk pass
(sb200_debug_decode_chunks), which captures every decoder stage of every chunk:
    z (the gathered latent rows) -> dec.pre -> dec.up{i} -> dec.mrf{i} -> wav.
Each stage is recomputed from the chunk's own captured input, zero-padded at the chunk's edges as decoder.onnx pads a
frame slice, and held to the Job bounds: dec_reference.tc_bound per 128-row tile on backends 1 and 2, f32_bound per chunk
on backend 0 and on the waveform.  Bit for bit, the gathered rows are the latent's, a whole-latent chunk is a debug Job
of the same utterance, and every row whose receptive field (dec_reference.chunk_halo) lies inside its chunk equals the
whole-latent chunk's row.  Run with -s to print the per-stage tables."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import dec_reference as dr  # noqa: E402
from sonata_b200 import PiperSynthesisConfig, VitsStreamingModel, voicegen, workload  # noqa: E402
from sonata_b200 import _native as N  # noqa: E402
from sonata_b200.job import SynthesisJob  # noqa: E402
from sonata_b200.piper import _check  # noqa: E402

pytestmark = pytest.mark.gpu

# name -> (quality, speakers)
VOICES = {"medium": ("medium", 1), "high": ("high", 1), "x_low": ("x_low", 1), "medium_spk4": ("medium", 4)}
EDGE_CASES = [("medium", 1), ("medium", 0), ("medium", 2), ("high", 1), ("high", 0), ("x_low", 1), ("medium_spk4", 1)]
# the edge pass's latents (frames forced per id, zero noise): about 300 frames, more than 1024, about 300; and their
# speakers on the 4-speaker voice
LATENT_FRAMES = (300, 1030, 290)
LATENT_SPEAKERS = (3, 1, 2)
IDS = 24
# the production-size pass: chunks of 45 frames and 3 of overlap each side from 8 latents of 256 phonemes (the C2
# utterance length), 4 chunks each
STEP, PAD, PROD_LATENTS, PROD_CHUNKS = 45, 3, 8, 4


@pytest.fixture(scope="module")
def models(lib_built):
    d = voicegen.default_voice_dir()
    ms = {}

    def get(voice):
        if voice not in ms:
            quality, nspk = VOICES[voice]
            ms[voice] = VitsStreamingModel(voicegen.write_voice(d, quality, n_speakers=nspk), device=0)
        return ms[voice]
    yield get
    for m in ms.values():
        m.close()


_TENSORS = {}


def _tensors(voice):
    if voice not in _TENSORS:
        quality, nspk = VOICES[voice]
        _TENSORS[voice] = voicegen.make_tensors(quality, n_speakers=nspk)
    return _TENSORS[voice]


def _frames(n_ids, y_len):
    """Per-id frame counts summing to y_len."""
    return np.diff(np.rint(np.linspace(0, y_len, n_ids + 1))).astype(np.int32)


def _edge_inputs(voice):
    """ids, configs and per-id frames of the edge pass's latents."""
    multi = VOICES[voice][1] > 1
    batches = [workload.synthetic_ids(IDS // 2, utt=70 + i)[:IDS] for i in range(len(LATENT_FRAMES))]
    cfgs = [PiperSynthesisConfig(LATENT_SPEAKERS[b] if multi else None, 0.0, 1.0, 0.0) for b in range(len(batches))]
    return batches, cfgs, [_frames(IDS, f) for f in LATENT_FRAMES]


def _edge_chunks(encs):
    """The edge pass, speakers side by side: each latent whole, chunks of 1 and 2 frames at frame 0 and of 1 at the last
    frame, (1, 128) and (5, 134), 127 / 128 / 129 frames starting mid-latent and mid-granule, and two overlapping chunks
    of the long latent, the second ending at its last frame."""
    a, b, c = encs
    fa, fb, fc = (e.num_frames for e in encs)
    return [(a, 0, fa), (b, 0, fb), (c, 0, fc), (a, 0, 1), (b, 0, 2), (a, fa - 1, fa), (c, 1, 128), (a, 5, 134),
            (b, 301, 428), (c, 150, 278), (b, 450, 579), (b, 700, 900), (b, 850, fb)]


def _debug_pass(m, chunks):
    """One debug chunk pass: per chunk {stage name: captured rows}, and the kernels it launched."""
    lib = m._lib
    n = len(chunks)
    hs = (C.c_void_p * n)(*[e._h.value for e, _, _ in chunks])
    lo = np.array([c[1] for c in chunks], np.int64)
    hi = np.array([c[2] for c in chunks], np.int64)
    caps, count, err = C.POINTER(N.sb200_chunk_capture)(), C.c_size_t(), N.sb200_error()
    l0 = lib.sb200_launch_count()
    _check(lib.sb200_debug_decode_chunks(m._h, hs, lo.ctypes.data_as(C.POINTER(C.c_int64)),
                                         hi.ctypes.data_as(C.POINTER(C.c_int64)), n, C.byref(caps), C.byref(count),
                                         C.byref(err)), err)
    launches = lib.sb200_launch_count() - l0
    out = [{} for _ in range(n)]
    try:
        for i in range(count.value):
            r = caps[i]
            out[r.chunk][r.name.decode()] = np.ctypeslib.as_array(r.data, shape=(r.rows, r.cols)).copy()
    finally:
        lib.sb200_bytes_free(C.cast(caps, C.POINTER(C.c_uint8)))
    return out, launches


def _check_chunk(voice, backend, u, sid, where, table):
    """Every decoder stage of one chunk's captures u against float64; returns the failures."""
    t = _tensors(voice)
    fails = []
    for name, src, fn in dr.stages(t, sid):
        if name.startswith("flow."):
            continue
        x, got = u[src], u[name]
        ref = fn(x, dr.Arith("f64"))
        assert got.shape == tuple(ref.shape), (voice, where, name, got.shape, tuple(ref.shape))
        assert np.isfinite(got).all(), (voice, where, name)
        if name == "wav" or backend == 0:
            e, e_yard, r = dr.f32_check(got, ref, fn(x, dr.Arith("f32")))
            tile = -1
        else:
            e, e_yard, r, tile = dr.tc_check(got, ref, fn(x, dr.Arith("emu")), dr.tc_mult(t, name))
        row = table.setdefault((voice, backend, name), [0.0, 0.0, 0.0, ""])
        if r >= row[2]:
            row[2], row[3] = r, f"{where} tile {tile}"
        row[0], row[1] = max(row[0], e), max(row[1], e_yard)
        if r > 1.0:
            fails.append((voice, backend, where, name, tile, r))
    return fails


def _interior_fails(t, chunks, caps, whole):
    """Rows of every stage whose receptive field lies inside their chunk against the same rows of the latent's whole
    chunk (caps[whole[latent]]), bit for bit; an edge that is the latent's own edge has no halo."""
    halo = dr.chunk_halo(t)
    fails = []
    for k, (e, lo, hi) in enumerate(chunks):
        w = caps[whole[id(e)]]
        for name, (left, right) in halo.items():
            got = caps[k][name]
            U = got.shape[0] // (hi - lo)
            i0 = 0 if lo == 0 else left
            i1 = got.shape[0] - (0 if hi == e.num_frames else right)
            if i0 >= i1:
                continue
            ref = w[name][lo * U + i0:lo * U + i1]
            if not np.array_equal(got[i0:i1], ref):
                bad = np.flatnonzero((got[i0:i1] != ref).any(axis=1)) + i0
                fails.append((k, lo, hi, name, int(bad[0]), int(bad[-1]), len(bad)))
    return fails


def _print(table, title):
    print(f"\n{title}\n{'voice':12s} be {'stage':9s} {'max|err|':>9s} {'emu/fp32':>9s} {'of bound':>8s}  worst")
    for (voice, backend, name), (e, ey, r, where) in table.items():
        print(f"{voice:12s} {backend:2d} {name:9s} {e:9.2e} {ey:9.2e} {r:8.3f}  {where}")


def _same(a, b):
    return len(a) == len(b) and all(x.keys() == y.keys() and all(np.array_equal(x[s], y[s]) for s in x)
                                    for x, y in zip(a, b))


@pytest.mark.parametrize("voice,backend", EDGE_CASES)
def test_chunk_pass_stages_at_chunk_edges(models, voice, backend):
    """The edge pass: every stage of every chunk within its bound (the latent's own speaker on the 4-speaker voice); each
    chunk's z is its rows of the latent; each whole-latent chunk is a debug Job of the same ids and config, stage for
    stage; interior rows are the whole-latent chunk's; and the waveforms and launch count are the plain pass's."""
    m = models(voice)
    multi = VOICES[voice][1] > 1
    m.set_backend(backend)
    try:
        batches, cfgs, frames = _edge_inputs(voice)
        encs = m.infer_encoder_batch(batches, cfgs, durations=frames)
        assert [e.num_frames for e in encs] == list(LATENT_FRAMES)
        chunks = _edge_chunks(encs)
        caps, launches = _debug_pass(m, chunks)
        l0 = m._lib.sb200_launch_count()
        plain = m.infer_decoder_batch(chunks)
        assert launches == m._lib.sb200_launch_count() - l0
        job = SynthesisJob(m, batches, debug=True, configs=cfgs)
        job.set_durations(None, frames)
        job.run()
        jwav = [w.samples.as_slice() for w in job.fetch()]
        jcaps = [{name: job.debug_fetch(name, b) for name in caps[b] if name != "wav"} for b in range(len(encs))]
        job.close()
    finally:
        m.set_backend(1)

    whole = {id(e): b for b, e in enumerate(encs)}
    table, fails = {}, []
    for k, (e, lo, hi) in enumerate(chunks):
        u = caps[k]
        assert np.array_equal(u["wav"][:, 0], plain[k].as_slice()), (voice, k, lo, hi)
        assert np.array_equal(u["z"], caps[whole[id(e)]]["z"][lo:hi]), (voice, k, lo, hi)
        sid = LATENT_SPEAKERS[whole[id(e)]] if multi else None
        fails += _check_chunk(voice, backend, u, sid, f"chunk {k} [{lo}, {hi})", table)
    for b in range(len(encs)):
        assert np.array_equal(caps[b]["wav"][:, 0], jwav[b]), (voice, b)
        for name, x in jcaps[b].items():
            assert np.array_equal(caps[b][name], x), (voice, b, name)
    interior = _interior_fails(_tensors(voice), chunks, caps, whole)
    _print(table, f"{voice} backend {backend}, chunks {[(lo, hi) for _, lo, hi in chunks]}")
    assert not fails, fails
    assert not interior, interior


def test_chunk_pass_stages_at_production_size(models):
    """A realtime step's shape on medium, backend 1: 32 chunks of 51 frames from 8 latents of 256 phonemes; every stage
    of the first, a middle and the last chunk within its bound.  Around it, the edge pass runs before and after on the
    same context and gives the same bits: no stale rows survive in a reused workspace."""
    m = models("medium")
    batches, cfgs, frames = _edge_inputs("medium")
    encs = m.infer_encoder_batch(batches, cfgs, durations=frames)
    edge = _edge_chunks(encs)
    first, _ = _debug_pass(m, edge)

    lat = m.infer_encoder_batch([workload.synthetic_ids(256, utt=200 + i) for i in range(PROD_LATENTS)])
    chunks = [(e, STEP * j - PAD, STEP * (j + 1) + PAD) for e in lat for j in range(1, PROD_CHUNKS + 1)]
    assert all(hi <= e.num_frames for e, _, hi in chunks)
    caps, _ = _debug_pass(m, chunks)
    table, fails = {}, []
    for k in (0, len(chunks) // 2, len(chunks) - 1):
        _, lo, hi = chunks[k]
        fails += _check_chunk("medium", 1, caps[k], None, f"chunk {k} [{lo}, {hi})", table)
    del caps
    torch.cuda.empty_cache()

    again, _ = _debug_pass(m, edge)
    _print(table, f"medium backend 1, {len(chunks)} chunks of {STEP + 2 * PAD} frames")
    assert not fails, fails
    assert _same(first, again)
