"""CPU: the pitch-contour specification (tests/prosody_contour_reference.py) against the library's no-device plan hook,
against the utterance-ratio plan it reduces to, on a tone, and the argument checks."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import prosody_contour_reference as pc
import prosody_reference as pr
from sonata_b200 import OperationError
from sonata_b200 import _native as N
from sonata_b200.piper import _alignment, _contour_arrays, _prosody_arrays

RATES = (22050, 16000)
NAN = float("nan")


def _lib_plan(rate, n, ends, ratios, tempo):
    ends = np.ascontiguousarray(ends, np.int64)
    ratios = np.ascontiguousarray(ratios, np.float32)
    shape = (C.c_int64 * 6)()
    pos = np.zeros(8 * n // (rate // 100) + 8, np.int64)
    bounds = np.zeros(len(ends), np.int64)
    rc = N.lib().sb200_debug_prosody_contour_plan(
        rate, n, ends.ctypes.data_as(C.POINTER(C.c_int64)), ratios.ctypes.data_as(C.POINTER(C.c_float)), len(ends),
        NAN if tempo is None else tempo, shape, pos.ctypes.data_as(C.POINTER(C.c_int64)), pos.size,
        bounds.ctypes.data_as(C.POINTER(C.c_int64)))
    return rc, list(shape), pos, bounds


def _contours(rng, n_ids):
    """(frames per id, ratios) cases: zero-frame ids, adjacent equal ratios, NaN / 1, many short pieces."""
    f = rng.integers(0, 12, n_ids)
    f[rng.random(n_ids) < 0.2] = 0
    yield f, rng.choice([0.8, 1.0, 1.25, NAN, 0.5, 2.0], n_ids)
    yield f, np.repeat(rng.choice([0.7, 1.3], (n_ids + 2) // 3), 3)[:n_ids]          # runs of equal ratios
    yield np.ones(n_ids, np.int64), rng.uniform(0.5, 2.0, n_ids)                      # one frame each, all distinct
    f2 = f.copy()
    f2[:n_ids // 2] = 0
    yield f2, np.where(np.arange(n_ids) < n_ids // 2, 1.9, rng.choice([0.6, 1.1], n_ids))   # leading empty ids


@pytest.mark.parametrize("rate", RATES)
def test_plan_equals_the_library(lib_built, rate):
    rng = np.random.default_rng(rate)
    checked = 0
    for n_ids in (2, 7, 31):
        for frames, ratios in _contours(rng, n_ids):
            cum = np.cumsum(frames)
            n = 256 * max(int(cum[-1]), 1)
            ends = 256 * cum
            for tempo in (None, 0.5, 2.5, 1.25):
                pl = pc.plan(rate, n, ends, ratios, tempo)
                rc, shape, pos, bounds = _lib_plan(rate, n, ends, ratios, tempo)
                assert rc == 0
                assert shape == [pl["Hs"], pl["N"], pl["D"], pl["n1"], pl["n2"], pl["F"]], (n_ids, tempo)
                np.testing.assert_array_equal(pos[:pl["F"]], pl["a"])
                np.testing.assert_array_equal(bounds, pl["bounds"])
                assert np.all(np.diff(bounds) >= 0) and bounds[-1] == pl["n2"]
                checked += pl["m"] > 1
    assert checked > 20
    # sample-level ends: pieces shorter than a synthesis hop
    ends = np.cumsum([0, 50, 3, 0, 400, 90, 1000, 7])
    ratios = [1.5, 0.6, 2.0, 1.1, 0.5, 1.5, 0.9, 1.2]
    for tempo in (None, 0.5, 2.5):
        pl = pc.plan(rate, int(ends[-1]), ends, ratios, tempo)
        rc, shape, pos, bounds = _lib_plan(rate, int(ends[-1]), ends, ratios, tempo)
        assert rc == 0 and shape[3:] == [pl["n1"], pl["n2"], pl["F"]] and pl["m"] == 6
        np.testing.assert_array_equal(pos[:pl["F"]], pl["a"])
        np.testing.assert_array_equal(bounds, pl["bounds"])


@pytest.mark.parametrize("rate", RATES)
def test_one_piece_is_the_utterance_ratio(lib_built, rate):
    shape_u = (C.c_int64 * 6)()
    for p in (0.5, 0.8, 1.25, 2.0, 1.0):
        for tempo in (None, 0.5, 2.5):
            for frames in ([3, 0, 5, 2], [0, 0, 0]):
                cum = np.cumsum(frames)
                n = 256 * max(int(cum[-1]), 1)
                # NaN and 1 mean 1, and ids without frames do not split the piece
                ratios = [p, NAN if p == 1.0 else p, p, 1.0 if p == 1.0 else p][:len(frames)]
                if frames[1] == 0:
                    ratios[1] = 1.7
                rc, shape, pos, bounds = _lib_plan(rate, n, 256 * cum, ratios, tempo)
                t = NAN if tempo is None else tempo
                pos_u = np.zeros(pos.size, np.int64)
                u = p if cum[-1] else NAN           # an utterance whose ids all have 0 frames is one piece of ratio 1
                assert N.lib().sb200_debug_prosody_plan(rate, n, u, t, shape_u,
                                                        pos_u.ctypes.data_as(C.POINTER(C.c_int64)), pos_u.size) == 0
                assert rc == 0 and shape == list(shape_u), (p, tempo, frames)
                np.testing.assert_array_equal(pos, pos_u)
                pl = pc.plan(rate, n, 256 * cum, ratios, tempo)
                if frames[-1]:
                    assert pl["m"] == 1 and pl["one"] is not None
                    assert (pl["n1"], pl["n2"], pl["F"]) == (pl["one"]["n1"], pl["one"]["n2"], pl["one"]["F"])
                    np.testing.assert_array_equal(pl["a"], pl["one"]["a"])


@pytest.mark.parametrize("rate", RATES)
def test_no_tempo_keeps_the_boundaries(lib_built, rate):
    rng = np.random.default_rng(7 + rate)
    for _ in range(40):
        n_ids = int(rng.integers(2, 40))
        frames = rng.integers(0, 15, n_ids)
        frames[-1] = max(frames[-1], 1)
        ratios = rng.choice([0.5, 0.8, 1.0, 1.25, 1.6, 2.0, NAN], n_ids)
        cum = np.cumsum(frames)
        n = 256 * int(cum[-1])
        rc, shape, _, bounds = _lib_plan(rate, n, 256 * cum, ratios, None)
        assert rc == 0
        np.testing.assert_array_equal(bounds[:-1], 256 * cum[:-1])
        assert bounds[-1] == shape[4] and abs(bounds[-1] - n) <= 1


@pytest.mark.parametrize("rate", RATES)
def test_two_pieces_move_each_tone_and_keep_each_length(rate):
    f, half = 300.0, rate // 2
    x = pr.tone(rate, f, 1.0)[:2 * half]
    ends = np.array([half, 2 * half])
    for tempo in (None, 1.5):
        r = pc.process(x, rate, ends, [1.0, 1.5], tempo)
        pl = r["plan"]
        t = 1.0 if tempo is None else tempo
        b = int(pl["bounds"][0])
        assert abs(b - half / t) <= 1 and abs(pl["n2"] - b - half / t) <= 1
        y = r["y"]
        for seg, p in ((y[:b], 1.0), (y[b:], 1.5)):
            seg = seg[len(seg) // 8: -len(seg) // 8]        # away from the knot and the edges
            peak, res = pr.spectral_peak_hz(seg, rate)
            assert abs(peak - f * p) <= res + 1e-9, (tempo, p, peak)


def test_argument_checks(lib_built):
    ends = np.array([256, 512, 768], np.int64)
    for bad in (0.4, 2.5, float("inf"), -1.0):
        assert _lib_plan(22050, 768, ends, [1.0, bad, 1.0], None)[0] == 19
    assert _lib_plan(22050, 768, ends, [1.0, 1.25, 1.0], 9.0)[0] == 19
    assert _lib_plan(22050, 768, [256, 100, 768], [1.0, 1.25, 1.0], None)[0] == 19          # decreasing ends
    assert _lib_plan(22050, 1024, ends, [1.0, 1.25, 1.0], None)[0] == 19                    # last end short of n
    assert _lib_plan(500, 768, ends, [1.0, 1.25, 1.0], None)[0] == 19
    # Python: the same checks, each naming the utterance and the id
    assert _contour_arrays([3, 2], None) is None
    assert _contour_arrays([3, 2], [None, [1.0, float("nan")]]) is None
    got = _contour_arrays([3, 2], [[1.25, None, 1.0], None])
    assert got.dtype == np.float32 and got[0] == np.float32(1.25) and np.isnan(got[1:]).sum() == 3
    for bad, what in ((2.5, "2.5"), (0.1, "0.1"), (float("inf"), "inf"), ("x", "'x'")):
        for seq in ([1.0, bad], np.array([1.0, bad]) if not isinstance(bad, str) else (1.0, bad)):
            with pytest.raises(OperationError, match=f"utterance 1, id 1: pitch ratio {what}"):
                _contour_arrays([2, 2], [None, seq])
    with pytest.raises(OperationError, match="utterance 0: 2 pitch ratios for 3 ids"):
        _contour_arrays([3], [[1.0, 1.25]])
    with pytest.raises(OperationError, match="2 entries for 1"):
        _contour_arrays([3], [None, None])
    pit, _ = _prosody_arrays([None, 1.25], None, 2)
    with pytest.raises(OperationError, match="utterance 1: a pitch contour and a pitch ratio together"):
        _contour_arrays([2, 2], [None, [1.0, 0.8]], pit)
    assert _contour_arrays([2, 2], [[0.8, 1.0], [1.0, None]], pit) is not None     # utterance 1's contour is neutral


def test_alignment_from_delivered_ends():
    frames, src = [2, 3, 0, 5, 1], [-1, 0, 0, 1, -1]
    bounds = [500, 1290, 1290, 2555, 2800]
    al = _alignment("ab", src, frames, 2800, bounds=bounds)
    assert [(a.start_sample, a.num_samples) for a in al] == [(0, 500), (500, 790), (1290, 1265), (2555, 245)]
    al = _alignment("ab", src, frames, 2 * 2800 + 1, up=2, down=1, bounds=bounds)
    assert [a.start_sample for a in al] == [0, 1000, 2580, 5110] and sum(a.num_samples for a in al) == 5601
