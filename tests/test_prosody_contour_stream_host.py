"""CPU: the emission rule of streams with a pitch contour (prosody_contour_stream_reference) against the library's
no-device plan hook, its reduction to the ratio stream for one piece, its history bounds, and the Python-side
refusals."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import prosody_contour_reference as pcr
import prosody_contour_stream_reference as pcs
import prosody_stream_reference as psr
from sonata_b200 import OperationError
from sonata_b200 import _native as N
from sonata_b200.piper import ProsodyStream, StreamBatch, VitsModel, VitsStreamingModel, _contour_arrays

RATES = (16000, 22050)
TEMPOS = (None, 0.25, 0.8, 4.0)
NAN = float("nan")
FIELDS = ("emitted", "frames", "stretched", "h_in", "h_s")


def question(k):
    """1 on the first 75 % of ids, then rising in five steps to 1.3 (the README's question contour)."""
    c = [1.0] * k
    rise = k - int(0.75 * k)
    for i in range(int(0.75 * k), k):
        c[i] = 1.0 + 0.06 * (1 + (i - int(0.75 * k)) * 5 // rise)
    return c


def contours(seed=0):
    """name -> (frames per id, ratios)."""
    rng = np.random.default_rng(seed)
    f = rng.integers(1, 14, 40)
    zero = f.copy()
    zero[rng.random(40) < 0.3] = 0
    zero[-1] = 3
    return {
        "uniform": (f, [1.25] * 40),
        "question": (f, question(40)),
        "alternating": (np.ones(60, np.int64), [0.5 if i % 2 else 2.0 for i in range(60)]),
        "zero_frames": (zero, rng.choice([0.8, 1.0, 1.25, NAN, 0.5, 2.0], 40)),
        "all_zero": (np.zeros(12, np.int64), rng.choice([0.8, 1.25], 12)),
    }


def _ends(frames):
    """(n, ends): 256 samples per frame; a sentence of only empty ids still has one frame."""
    cum = np.cumsum(frames)
    return 256 * max(int(cum[-1]), 1), 256 * cum


def _lib_plan(rate, n, ends, ratios, tempo, lens):
    ends = np.ascontiguousarray(ends, np.int64)
    ratios = np.ascontiguousarray(ratios, np.float32)
    lens = np.ascontiguousarray(lens, np.int64)
    out = np.zeros(5 * len(lens), np.int64)
    p64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))
    rc = N.lib().sb200_debug_prosody_contour_stream_plan(
        rate, n, p64(ends), ratios.ctypes.data_as(C.POINTER(C.c_float)), len(ends), NAN if tempo is None else tempo,
        p64(lens), len(lens), p64(out))
    return rc, out.reshape(-1, 5)


@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("tempo", TEMPOS)
@pytest.mark.parametrize("name", list(contours()))
def test_plan_hook_equals_the_rule(lib_built, rate, tempo, name):
    frames, ratios = contours()[name]
    n, ends = _ends(frames)
    pl = pcr.plan(rate, n, ends, ratios, tempo)
    for cname, lens in psr.chunkings(n, rate).items():
        rc, got = _lib_plan(rate, n, ends, ratios, tempo, lens)
        if name == "all_zero" and tempo is None:
            assert rc == 19, cname          # one piece of ratio 1 and no tempo: nothing to do
            continue
        ref = pcs.stream(rate, n, ends, ratios, tempo, lens)
        assert rc == 0, cname
        np.testing.assert_array_equal(got, [[r[f] for f in FIELDS] for r in ref], err_msg=f"{name} {cname}")
        assert int(got[:, 0].sum()) == pl["n2"], cname
        if pl["one"] is None:
            cap_in, cap_s = pcs.caps(pl)
        else:
            p = float(pl["p"][0])
            cap_in, cap_s = psr.caps(rate, None if p == 1.0 else p, tempo)
        assert got[:, 3].max() <= cap_in and got[:, 4].max() <= cap_s, cname
        assert cap_s <= 68


@pytest.mark.parametrize("rate", RATES)
def test_zero_length_chunks(lib_built, rate):
    frames, ratios = contours(1)["zero_frames"]
    n, ends = _ends(frames)
    lens = [0, 300, 0, 0, 5000, 0] + [1000] * ((n - 5300) // 1000) + [(n - 5300) % 1000, 0]
    for tempo in TEMPOS:
        rc, got = _lib_plan(rate, n, ends, ratios, tempo, lens)
        assert rc == 0
        ref = pcs.stream(rate, n, ends, ratios, tempo, lens)
        np.testing.assert_array_equal(got, [[r[f] for f in FIELDS] for r in ref])


@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("tempo", TEMPOS)
@pytest.mark.parametrize("p", [0.5, 0.8, 1.25, 2.0])
def test_one_piece_is_the_ratio_stream(lib_built, rate, tempo, p):
    frames = np.random.default_rng(3).integers(0, 9, 30)
    frames[-1] = 2
    n, ends = _ends(frames)
    for cname, lens in psr.chunkings(n, rate).items():
        rc, got = _lib_plan(rate, n, ends, [p] * 30, tempo, lens)
        assert rc == 0
        l64 = np.ascontiguousarray(lens, np.int64)
        want = np.zeros(len(lens), np.int64)
        assert N.lib().sb200_debug_prosody_stream_plan(rate, p, NAN if tempo is None else tempo,
                                                       l64.ctypes.data_as(C.POINTER(C.c_int64)), len(lens),
                                                       want.ctypes.data_as(C.POINTER(C.c_int64))) == 0
        np.testing.assert_array_equal(got[:, 0], want, err_msg=cname)


@pytest.mark.parametrize("rate", RATES)
def test_total_must_be_n(lib_built, rate):
    frames, ratios = contours()["question"]
    n, ends = _ends(frames)
    for lens in ([n - 1], [n + 1], [n // 2, n // 2 - 256], [n, 256], [n + 256, 0], [n, 256, 0]):
        rc, _ = _lib_plan(rate, n, ends, ratios, None, lens)
        assert rc == 19, lens
        with pytest.raises(ValueError):
            pcs.stream(rate, n, ends, ratios, None, lens)
    rc, _ = _lib_plan(rate, n, ends, [1.0] * len(frames), None, [n])       # neutral: refused
    assert rc == 19


def test_bad_ratio_and_ends_refused(lib_built):
    frames, ratios = contours()["question"]
    n, ends = _ends(frames)
    bad = list(ratios)
    bad[7] = 2.5
    assert _lib_plan(22050, n, ends, bad, None, [n])[0] == 19
    assert _lib_plan(22050, n, ends, ratios, 5.0, [n])[0] == 19
    assert _lib_plan(22050, n + 256, ends, ratios, None, [n + 256])[0] == 19      # the last id does not end at n


# ---- Python-side refusals (no device: the checks run before any model work)
class _Fake:
    """Stands in for a loaded model where the checks need no device."""
    def __init__(self, cls):
        self.__class__ = type("Fake" + cls.__name__, (cls,), {})


def test_contour_values_checked():
    with pytest.raises(OperationError, match="utterance 0, id 2: pitch ratio 3.0"):
        _contour_arrays([4], [[1.0, 1.2, 3.0, 1.0]])
    with pytest.raises(OperationError, match="4 pitch ratios for 5 ids"):
        _contour_arrays([5], [[1.0, 1.2, 1.1, 1.0]])
    with pytest.raises(OperationError, match="a pitch contour and a pitch ratio together"):
        _contour_arrays([2], [[1.2, 1.1]], np.array([1.5], np.float32))


def test_prosody_stream_needs_its_encoder_outputs():
    with pytest.raises(OperationError, match="needs the EncoderOutputs"):
        ProsodyStream(object(), pitch_contour=[1.2, 1.1])
    with pytest.raises(OperationError, match="^stream: a pitch contour and a pitch ratio together"):
        ProsodyStream(object(), pitch=1.5, pitch_contour=[1.2, 1.1])


def test_non_streaming_models_refuse_a_contour():
    m = _Fake(VitsModel)
    with pytest.raises(OperationError, match="StreamBatch cannot apply a pitch contour"):
        sb = StreamBatch.__new__(StreamBatch)
        sb.model = m
        sb.add([1, 2, 3], pitch_contour=[1.2, 1.2, 1.2])
    with pytest.raises(OperationError, match="stream_synthesis cannot apply a pitch contour"):
        VitsStreamingModel.stream_synthesis(m, "abc", 10, 2, pitch_contour=[1.2] * 3)


def test_stream_batch_checks_the_contour_at_add():
    m = _Fake(VitsStreamingModel)
    sb = StreamBatch(m, 10, 2)
    with pytest.raises(OperationError, match="2 pitch ratios for 3 ids"):
        sb.add([1, 2, 3], pitch_contour=[1.2, 1.2])
    with pytest.raises(OperationError, match="id 1: pitch ratio 0.2"):
        sb.add([1, 2, 3], pitch_contour=[1.2, 0.2, 1.0])
    with pytest.raises(OperationError, match="a pitch contour and a pitch ratio together"):
        sb.add([1, 2, 3], pitch=1.5, pitch_contour=[1.2, 1.1, 1.0])
    assert len(sb) == 0
    key = sb.add([1, 2, 3], pitch_contour=[1.2, 1.1, 1.0], tempo=1.5)
    with pytest.raises(KeyError):
        sb.bounds(key)
    # errors name the stream being added, not an utterance of a batch
    with pytest.raises(OperationError, match="^stream 1, id 2: pitch ratio 3.0"):
        sb.add([1, 2, 3], pitch_contour=[1.2, 1.1, 3.0])
    with pytest.raises(OperationError, match="^stream 1: 2 pitch ratios for 3 ids"):
        sb.add([1, 2, 3], pitch_contour=[1.2, 1.1])
