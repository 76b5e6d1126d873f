"""CPU: the output-rate resampler's host side -- the filter design against scipy's, the up/down reduction, argument
checks at the C and Python layers, the formula against resample_poly, and phoneme alignment at the output rate."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import resample_reference as rr
from sonata_b200 import _native as N
from sonata_b200.core import OperationError
from sonata_b200.piper import OUTPUT_RATES, _alignment, _rate_array, rate_ratio

PAIRS = [(i, o) for i in rr.VOICE_RATES for o in rr.TARGETS if o != i]


def _filter(in_rate, out_rate):
    up, down = C.c_int32(), C.c_int32()
    assert N.lib().sb200_debug_resample_filter(in_rate, out_rate, None, 0, C.byref(up), C.byref(down)) == 0
    taps = np.zeros(20 * max(up.value, down.value) + 1, np.float32)
    assert N.lib().sb200_debug_resample_filter(in_rate, out_rate, taps.ctypes.data_as(C.POINTER(C.c_float)), taps.size,
                                               C.byref(up), C.byref(down)) == 0
    return up.value, down.value, taps


@pytest.mark.parametrize("in_rate,out_rate", PAIRS)
def test_filter_matches_scipy(lib_built, in_rate, out_rate):
    up, down, taps = _filter(in_rate, out_rate)
    assert (up, down) == rr.ratio(in_rate, out_rate)
    assert max(up, down) <= 640
    ref = rr.taps64(up, down).astype(np.float32)
    ulp = np.spacing(np.abs(ref))
    assert np.all(np.abs(taps.astype(np.float64) - ref) <= ulp), float(np.max(np.abs(taps - ref) / ulp))


def test_ratio_examples(lib_built):
    assert _filter(22050, 48000)[:2] == (320, 147)
    assert _filter(22050, 8000)[:2] == (160, 441)
    assert _filter(16000, 11025)[:2] == (441, 640)
    assert _filter(16000, 48000)[:2] == (3, 1)
    for i, o in PAIRS:
        assert rate_ratio(i, o) == rr.ratio(i, o)
    assert rate_ratio(22050, None) == rate_ratio(22050, 0) == rate_ratio(22050, 22050) == (1, 1)


@pytest.mark.parametrize("out_rate", [0, 22050, 1, 7999, 96000, -8000])
def test_filter_refuses_unsupported_or_equal_rates(lib_built, out_rate):
    up, down = C.c_int32(), C.c_int32()
    assert N.lib().sb200_debug_resample_filter(22050, out_rate, None, 0, C.byref(up), C.byref(down)) == 19


def test_debug_resample_checks_rate_before_the_device(lib_built):
    x = np.zeros(16, np.float32)
    y = np.zeros(64, np.float32)
    err = N.sb200_error()
    rc = N.lib().sb200_debug_resample(0, x.ctypes.data_as(C.POINTER(C.c_float)), x.size, 22050, 12345,
                                      y.ctypes.data_as(C.POINTER(C.c_float)), C.byref(err))
    assert rc == 19 and err.code == 19
    msg = C.string_at(err.message).decode()
    N.lib().sb200_string_free(err.message)
    assert "12345" in msg and "not supported" in msg


def test_python_rate_checks_name_the_utterance():
    assert _rate_array(None, 2) is None
    assert list(_rate_array([None, 0, 48000], 3)) == [0, 0, 48000]
    for bad in (12345, 8000.0, True, "8000"):
        with pytest.raises(OperationError, match="utterance 1"):
            _rate_array([8000, bad], 2)
    with pytest.raises(OperationError, match="2 entries for 3"):
        _rate_array([8000, 8000], 3)
    assert set(OUTPUT_RATES) == set(rr.TARGETS)


@pytest.mark.parametrize("up,down", [(320, 147), (160, 441), (3, 1), (1, 2), (441, 640), (2, 1)])
def test_reference_formula_is_resample_poly(up, down):
    """The documented sum, restated in float64 here (not the library's kernel), is resample_poly's output exactly."""
    rng = np.random.default_rng(up * 1000 + down)
    x = rng.standard_normal(997)
    h = rr.taps64(up, down)
    H = (len(h) - 1) // 2
    y = np.zeros(rr.n_out(len(x), up, down))
    for j in range(len(y)):
        t = j * down + H
        i = np.arange(max(0, -((-(t - 2 * H)) // up)), min(t // up, len(x) - 1) + 1)
        y[j] = np.sum(x[i] * h[t - i * up])
        assert len(i) <= 56
    ref = rr.resample64(x, up, down)
    assert y.shape == ref.shape
    np.testing.assert_allclose(y, ref, rtol=0, atol=1e-12)


@pytest.mark.parametrize("frames", [[3, 0, 5, 7, 2], [0, 0, 0], [1], [12, 40, 1, 0, 9, 100]])
@pytest.mark.parametrize("rates", [(22050, 48000), (22050, 8000), (16000, 11025), (16000, 48000), (22050, 22050)])
def test_alignment_at_output_rate_is_contiguous(frames, rates):
    up, down = rate_ratio(*rates)
    total = max(sum(frames), 1)
    n = rr.n_out(total * 256, up, down)
    src = [-1] + list(range(len(frames) - 2)) + [-1] if len(frames) >= 2 else [-1]
    al = _alignment("abcdefgh", src, frames, n, up, down)
    assert al[0].start_sample == 0
    for a, b in zip(al, al[1:]):
        assert a.start_sample + a.num_samples == b.start_sample
        assert a.num_samples >= 0
    assert al[-1].start_sample + al[-1].num_samples == n
    cum = 0
    for a, f in zip(al[:-1], frames):
        cum += f
        assert a.start_sample + a.num_samples == -((-cum * 256 * up) // down)


def test_c_layer_rate_errors_name_the_utterance(voice_paths):
    import sonata_b200
    m = sonata_b200.VitsModel(voice_paths["medium"], device=-1)      # config only: the rates are checked first
    ids = np.array([1, 5, 0, 2, 1, 6, 0, 2], np.int64)
    offs = np.array([0, 4, 8], np.uint64)
    rates = np.array([48000, 12345], np.uint32)
    outs = (N.sb200_audio * 2)()
    err = N.sb200_error()
    rc = m._lib.sb200_speak_batch_ids_rates(m._h, ids.ctypes.data_as(C.POINTER(C.c_int64)),
                                            offs.ctypes.data_as(C.POINTER(C.c_size_t)), 2, None, None, None, None,
                                            None, rates.ctypes.data_as(C.POINTER(C.c_uint32)), outs, None,
                                            C.byref(err))
    assert rc == 19 and err.code == 19
    msg = C.string_at(err.message).decode()
    N.lib().sb200_string_free(err.message)
    assert msg.startswith("utterance 1: ") and "12345" in msg
    with pytest.raises(OperationError, match="utterance 1"):
        m.infer_batch_with_values([[1, 5, 0, 2], [1, 6, 0, 2]], output_rates=[8000, 12345])
    m.close()


def _emit(in_rate, out_rate, lens):
    lens = np.asarray(lens, np.int64)
    out = np.zeros(len(lens), np.int64)
    assert N.lib().sb200_debug_resample_emit(in_rate, out_rate, lens.ctypes.data_as(C.POINTER(C.c_int64)), len(lens),
                                             out.ctypes.data_as(C.POINTER(C.c_int64))) == 0
    return out


@pytest.mark.parametrize("frames,chunk", [(100, 72), (151, 55), (774, 45), (1, 72), (300, 10)])
@pytest.mark.parametrize("in_rate,out_rate", [(22050, 48000), (22050, 8000), (16000, 11025), (16000, 48000),
                                              (22050, 44100), (16000, 8000)])
def test_stream_emit_sums_to_n_out(lib_built, frames, chunk, in_rate, out_rate):
    from sonata_b200.piper import AdaptiveMelChunker
    pad = 3
    ch = AdaptiveMelChunker(frames, chunk, pad)
    lens = []
    if frames <= chunk * 2 + pad * 2:
        lens = [frames * 256]                                   # one-shot stream
    else:
        for (m0, m1), (a0, a1) in ch:
            hi = frames if m1 is None else m1
            lens.append((hi - m0) * 256 - (a0 or 0) + (a1 or 0))
    up, down = rr.ratio(in_rate, out_rate)
    em = _emit(in_rate, out_rate, lens)
    assert int(em.sum()) == rr.n_out(sum(lens), up, down)
    assert (em >= 0).all()
    H = 10 * max(up, down)
    consumed = np.cumsum(lens)
    for k in range(len(lens) - 1):                               # emitted only what its inputs allow, and all of that
        done = int(em[:k + 1].sum())
        assert (done - 1) * down + H < consumed[k] * up or done == 0
        assert done * down + H >= consumed[k] * up
    # a chunk too short to complete any output emits 0 samples
    e = _emit(in_rate, out_rate, [1, 1, 1, 1000])
    assert e[0] == 0 and int(e.sum()) == rr.n_out(1003, up, down)
