"""CPU: loudness normalisation's host side -- the K-weighting design against BS.1770-4's tables and the float64
reference, known answers of the reference meter, and target checks at the C, Python and CLI layers."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import loudness_reference as lr
from sonata_b200 import _native as N
from sonata_b200.core import AudioSamples, OperationError
from sonata_b200.piper import _loudness_array


def _filter(rate):
    c = np.zeros(10, np.float64)
    rc = N.lib().sb200_debug_loudness_filter(rate, c.ctypes.data_as(C.POINTER(C.c_double)))
    return rc, c


def test_filter_matches_bs1770_tables_at_48k(lib_built):
    rc, c = _filter(48000)
    assert rc == 0
    np.testing.assert_allclose(c, lr.TABLE_48K, rtol=0, atol=1e-12)


@pytest.mark.parametrize("rate", lr.RATES)
def test_filter_matches_reference_design(lib_built, rate):
    rc, c = _filter(rate)
    assert rc == 0
    np.testing.assert_allclose(c, lr.coeffs(rate), rtol=1e-14, atol=1e-15)


@pytest.mark.parametrize("rate", [0, -48000, 7999, 384001])
def test_filter_refuses_unsupported_rates(lib_built, rate):
    assert _filter(rate)[0] == 19


@pytest.mark.parametrize("rate", lr.RATES)
def test_reference_sine_is_minus_23(rate):
    """A 997 Hz sine of peak 0.1 (-20 dBFS) is -23 LUFS, to within the filter's gain at 997 Hz at each rate."""
    assert abs(lr.integrated(lr.sine(rate, 5.0), rate) + 23.01) <= 0.1


def test_reference_gates():
    rate = 48000
    S = lr.step(rate)
    assert lr.integrated(np.zeros(rate * 2, np.float32), rate) == -math.inf
    assert lr.integrated(lr.sine(rate, 1.0)[:4 * S - 1], rate) == -math.inf
    assert lr.integrated(lr.sine(rate, 1.0, peak=1e-4), rate) == -math.inf          # about -83 LUFS
    assert lr.integrated(lr.sine(rate, 1.0)[:4 * S], rate) > -24
    # the relative gate drops the quiet half: -20 then -40 LUFS measures about -20
    loud, quiet = lr.sine(rate, 2.0, peak=0.1 * 10 ** 0.15), lr.sine(rate, 2.0, peak=0.1 * 10 ** -0.85)
    both = lr.integrated(np.concatenate([loud, quiet]), rate)
    assert abs(both - lr.integrated(loud, rate)) < 0.5
    # without the relative gate the mean would be well below
    z = lr.block_energies(np.concatenate([loud, quiet]), rate)
    assert -0.691 + 10 * math.log10(z.mean()) < both - 2.0


def test_reference_gain_never_exceeds_full_scale():
    x = lr.sine(48000, 2.0, peak=0.5)
    L = lr.integrated(x, 48000)
    g = lr.gain(x, 0.0, L)                 # the peak limit binds
    assert float(np.max(np.abs(x * g))) <= 1.0 + 2e-7
    assert lr.gain(x, -40.0, L) < 1.0
    assert lr.gain(np.zeros(10, np.float32), -23.0, -math.inf) == 1.0


def test_python_targets_name_the_utterance():
    assert _loudness_array(None, 2) is None
    assert _loudness_array([None, float("nan")], 2) is None          # NaN is "none", like None
    t = _loudness_array([-23, None, 0, -70.0], 4)
    assert t.dtype == np.float32 and np.isnan(t[1]) and list(t[[0, 2, 3]]) == [-23, 0, -70]
    for bad in (float("inf"), -float("inf"), 0.5, -70.01, "x", True):
        with pytest.raises(OperationError, match="utterance 1"):
            _loudness_array([-23, bad], 2)
    with pytest.raises(OperationError, match="1 entries for 2"):
        _loudness_array([-23], 2)


def test_fixed_scale_pcm():
    v = np.array([0.0, 0.5, -0.5, 1.0, -1.0, 1.5, -1.5, 1e-5], np.float32)
    ref = np.trunc(np.clip(v * np.float32(32767), -32768, 32767)).astype(np.int16)
    np.testing.assert_array_equal(AudioSamples(v).to_i16_fixed(), ref)
    assert AudioSamples(v).as_wave_bytes(fixed_scale=True) == ref.astype("<i2").tobytes()
    assert AudioSamples(v).as_wave_bytes() == AudioSamples(v).to_i16_vec().astype("<i2").tobytes()


def test_c_layer_target_errors_name_the_utterance(voice_paths):
    import sonata_b200
    m = sonata_b200.VitsModel(voice_paths["medium"], device=-1)      # config only: the targets are checked first
    ids = np.array([1, 5, 0, 2, 1, 6, 0, 2], np.int64)
    offs = np.array([0, 4, 8], np.uint64)
    for bad in (np.inf, -np.inf, 1.0, -71.0):
        t = np.array([np.nan, bad], np.float32)
        outs = (N.sb200_audio * 2)()
        err = N.sb200_error()
        rc = m._lib.sb200_speak_batch_ids_loudness(m._h, ids.ctypes.data_as(C.POINTER(C.c_int64)),
                                                   offs.ctypes.data_as(C.POINTER(C.c_size_t)), 2, None, None, None,
                                                   None, None, None, t.ctypes.data_as(C.POINTER(C.c_float)), outs,
                                                   None, None, None, C.byref(err))
        assert rc == 19 and err.code == 19
        msg = C.string_at(err.message).decode()
        N.lib().sb200_string_free(err.message)
        assert msg.startswith("utterance 1: ") and "loudness target" in msg, msg
    with pytest.raises(OperationError, match="utterance 1"):
        m.infer_batch_with_values([[1, 5, 0, 2], [1, 6, 0, 2]], loudness=[-23, 3])
    with pytest.raises(OperationError, match="utterance 0"):
        m.speak_batch(["ab"], loudness=[float("inf")])
    m.close()


def test_cli_refuses_bad_targets_and_realtime(voice_paths, tmp_path):
    from sonata_b200 import cli
    (tmp_path / "in.txt").write_text("hɛloʊ\n", encoding="utf-8")
    base = [voice_paths["medium"], "-f", str(tmp_path / "in.txt"), "--device", "-1"]
    for bad in ("1", "-80", "inf"):
        with pytest.raises(OperationError, match="utterance 0"):
            cli.main(base + ["--loudness", bad])
    with pytest.raises(OperationError, match="realtime"):
        cli.main(base + ["--mode", "realtime", "--loudness", "-23"])
