"""Host tests of volume contours (include/sonata_b200.h, sb200_speak_batch_ids_volume): the numpy contract, the checks
and their messages in Python and in the library, the per-character mapping, and the stream emission rule simulated
over random chunkings."""
import ctypes as C
import math
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import volume_reference as vr
import sonata_b200
from sonata_b200 import _native as N, voicegen
from sonata_b200.core import Audio, OperationError
from sonata_b200.piper import (_VitsCommons, _batch_options, _check, _stream_options, _volume_arrays,
                               VitsStreamingModel)

NAN, INF = float("nan"), float("inf")


# ---------------------------------------------------------------------------------------------------- the contract
def test_pieces_drop_empty_ids_and_merge_equal_levels():
    ends = [0, 300, 300, 500, 900, 1000]
    levels = [6.0, NAN, -6.0, 0.0, 0.0, -INF]
    starts, gains = vr.pieces(ends, levels, 1000)
    # id 0 and id 2 are empty; ids 1 (NaN -> 0) and 3, 4 (0) merge across the dropped id 2
    np.testing.assert_array_equal(starts, [0, 900])
    np.testing.assert_array_equal(gains, [1.0, 0.0])
    assert vr.asks(ends, levels, 1000)
    assert not vr.asks(ends, [NAN, 0.0, 3.0, 0.0, 0.0, 0.0], 1000)      # the level is on an empty id
    with pytest.raises(ValueError):
        vr.pieces([10, 5], [1.0, 2.0], 5)
    with pytest.raises(ValueError):
        vr.pieces([10, 20], [1.0, 2.0], 30)


def test_gains_are_rounded_from_double():
    assert vr.gain_of(NAN) == 1 and vr.gain_of(-INF) == 0 and vr.gain_of(0.0) == 1
    for v in (-60.0, -6.0, 0.5, 6.0, 20.0):
        assert vr.gain_of(v) == np.float32(10.0 ** (float(np.float32(v)) / 20.0))
    assert vr.gain_of(20.0) == np.float32(10.0)


@pytest.mark.parametrize("rate", (22050, 16000))
def test_curve_matches_the_header_sample_by_sample(rate):
    rng = np.random.default_rng(rate)
    half = rate // 200
    # short pieces (shorter than a ramp) make overlapping ramps; long ones hold their gain
    lens = [1, 3, half, 2 * half + 1, 40, 5000, 7, half // 2, 900]
    ends = np.cumsum(lens)
    levels = [6.0, -6.0, -INF, 3.0, 12.0, -20.0, 0.0, 20.0, -60.0]
    n2 = int(ends[-1])
    starts, gains = vr.pieces(ends, levels, n2)
    j = np.arange(n2)
    G = vr.gain_curve(starts, gains, rate, j)
    for jj in list(range(0, 2 * half + 60)) + list(rng.integers(0, n2, 300)):
        assert G[jj].tobytes() == vr.gain_scalar(starts, gains, rate, int(jj)).tobytes(), jj
    # away from any boundary each sample has its piece's gain exactly
    mid = int(starts[5]) + 2500
    assert G[mid] == gains[5]
    # an isolated boundary: a monotone smoothstep between the two gains, symmetric about its centre
    st2, g2 = vr.pieces([3000, 6000], [-6.0, 6.0], 6000)
    ramp = vr.gain_curve(st2, g2, rate, np.arange(3000 - half - 1, 3000 + half + 1))
    assert ramp[0] == g2[0] and ramp[-1] == g2[1] and np.all(np.diff(ramp) > 0)
    mid_gain = (float(g2[0]) + float(g2[1])) / 2
    np.testing.assert_allclose(ramp[1:-1] + ramp[1:-1][::-1], 2 * mid_gain, rtol=1e-6)


def test_one_piece_is_the_signal_times_its_gain():
    rng = np.random.default_rng(3)
    x = rng.standard_normal(4000).astype(np.float32)
    ends = [0, 1000, 2500, 4000]
    for level in (6.0, -12.5, -INF, 20.0):
        y = vr.apply(x, ends, [level] * 4, 22050)
        assert y.tobytes() == (x * vr.gain_of(level)).tobytes()
    # a neutral contour keeps every bit
    assert vr.apply(x, ends, [NAN, 0.0, NAN, 0.0], 22050).tobytes() == x.tobytes()


def test_muting_one_word():
    rate = 16000
    x = np.ones(6000, np.float32)
    y = vr.apply(x, [2000, 4000, 6000], [NAN, -INF, NAN], rate)
    half = rate // 200
    assert np.all(y[:2000 - half] == 1) and np.all(y[2000 + half:4000 - half] == 0) and np.all(y[4000 + half:] == 1)
    assert np.all((y[2000 - half:2000 + half] > 0) & (y[2000 - half:2000 + half] < 1))


# ---------------------------------------------------------------------------------------------------- emission rule
@pytest.mark.parametrize("seed", range(6))
def test_stream_emission_over_random_chunkings(seed):
    """The stage holds nothing back: each chunk of the stages before it, scaled at its delivered positions, joins to
    the whole signal scaled at once."""
    rng = np.random.default_rng(seed)
    rate = (22050, 16000)[seed % 2]
    n_ids = int(rng.integers(1, 40))
    frames = rng.integers(0, 6, n_ids)
    ends = 256 * np.cumsum(frames)
    n2 = int(ends[-1]) if ends[-1] else 256
    ends[-1] = n2
    levels = rng.choice([NAN, 0.0, -6.0, 6.0, -INF, 3.5], n_ids)
    x = rng.standard_normal(n2).astype(np.float32)
    whole = vr.apply(x, ends, levels, rate)
    cuts = np.sort(rng.choice(np.arange(1, n2), size=min(n2 - 1, int(rng.integers(1, 30))), replace=False))
    parts, j0 = [], 0
    for a, b in zip(np.r_[0, cuts], np.r_[cuts, n2]):
        parts.append(vr.apply(x[a:b], ends, levels, rate, j0=int(a)))
        j0 = b
    assert np.concatenate(parts).tobytes() == whole.tobytes()


# ---------------------------------------------------------------------------------------------------- Python checks
def test_python_checks_name_the_utterance_and_the_id():
    assert _volume_arrays([3], None) is None
    assert _volume_arrays([3, 2], [[NAN, 0.0, None], None]) is None
    img = _volume_arrays([3, 2], [[6.0, None, -INF], [0, -60]])
    assert img.dtype == np.float32 and img[0] == 6 and np.isnan(img[1]) and img[2] == -INF and img[4] == -60
    cases = [([[0.0, 21.0, 0.0]], "utterance 0, id 1: volume level 21.0 dB is not a finite value in"),
             ([[0.0, 0.0, INF]], "utterance 0, id 2: volume level inf dB"),
             ([[-61.0, 0.0, 0.0]], "utterance 0, id 0: volume level -61.0 dB"),
             ([[0.0, "loud", 0.0]], "utterance 0, id 1: volume level 'loud' is not a number"),
             ([[0.0, 0.0]], "utterance 0: 2 volume levels for 3 ids")]
    for contour, msg in cases:
        with pytest.raises(OperationError, match=re.escape(msg)):
            _volume_arrays([3], contour)
    with pytest.raises(OperationError, match=re.escape("stream 4, id 0: volume level 30.0 dB")):
        _volume_arrays([1], [[30.0]], ["stream 4"])


def test_batch_options_check_volume_last():
    # per id on an id surface, the utterance and id named
    o = _batch_options(None, 2, [2, 1], volume_contours=[[6.0, NAN], None])
    assert o.volume is not None and o.volume[0] == 6
    with pytest.raises(OperationError, match="utterance 1, id 0"):
        _batch_options(None, 2, [2, 1], volume_contours=[None, [99.0]])


class FakeModel:
    """Ids: bos 1, (ord(ch) % 50 + 3, pad 0) per character except '~' (dropped), eos 2; the f32 route records the
    options it is given."""

    def __init__(self):
        self.calls = []

    def phonemes_to_input_ids_map(self, ph):
        ids, src = [1], [-1]
        for c, ch in enumerate(ph):
            if ch != "~":
                ids += [ord(ch) % 50 + 3, 0]
                src += [c, c]
        return ids + [2], src + [-1]

    def _speak_ids(self, batches, o, frames=False):
        self.calls.append((batches, o))
        return [(Audio(np.zeros(256 * len(ids), np.float32), 22050), np.ones(len(ids), np.int32), None)
                for ids in batches]


def test_per_character_levels_map_to_each_id_and_its_pad():
    fake = FakeModel()
    _VitsCommons.speak_batch(fake, ["ab~c", "xy"], volume_contours=[[6.0, None, 99.0, -INF], None])
    batches, o = fake.calls[0]
    v = o.volume[:len(batches[0])]
    # bos and eos keep their level (0 dB), a None character is NaN, and the dropped character's bad level is ignored
    want = np.array([0.0, 6.0, 6.0, NAN, NAN, -INF, -INF, 0.0], np.float32)
    assert v.tobytes() == want.tobytes()
    assert np.isnan(o.volume[len(batches[0]):]).all()
    with pytest.raises(OperationError, match=re.escape("utterance 1: 1 volume levels for 2 characters")):
        _VitsCommons.speak_batch(fake, ["ab", "xy"], volume_contours=[None, [1.0]])
    with pytest.raises(OperationError, match=re.escape("utterance 0, character 1: volume level 25.0 dB")):
        _VitsCommons.speak_batch(fake, ["ab"], volume_contours=[[0.0, 25.0]])
    _VitsCommons.speak_batch_with_alignment(fake, ["ab"], volume_contours=[[-6.0, 0.0]])
    assert fake.calls[-1][1].volume is not None


# ---------------------------------------------------------------------------------------------------- library checks
@pytest.fixture(scope="module")
def config_only(lib_built):
    p = voicegen.write_voice(voicegen.default_voice_dir(), "medium")
    m = sonata_b200.VitsStreamingModel(p, device=-1)       # config only: any device call fails differently
    yield m
    m.close()


def test_the_c_entry_points_refuse_before_any_device_work(config_only):
    lib = N.lib()
    ids = np.array([1, 5, 2, 1, 6, 7, 2], np.int64)
    offs = np.array([0, 3, 7], np.uint64)
    i64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))
    f32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    sz = lambda a: a.ctypes.data_as(C.POINTER(C.c_size_t))
    outs = (N.sb200_audio * 2)()
    for bad, msg in ((25.0, "utterance 1, id 2: volume level 25.000000 dB is not a finite value in [-60, 20] or -inf"),
                     (INF, "utterance 1, id 2: volume level inf dB"), (-60.5, "utterance 1, id 2: volume level -60.5")):
        vol = np.array([6, NAN, 0, 0, -INF, bad, 0], np.float32)
        err = N.sb200_error()
        rc = lib.sb200_speak_batch_ids_volume(config_only._h, i64(ids), sz(offs), 2, None, None, None, None, None,
                                              None, None, None, None, None, None, None, None, None, f32(vol), outs,
                                              None, None, None, None, C.byref(err))
        with pytest.raises(OperationError) as e:
            _check(rc, err)
        assert re.escape(msg) and msg in str(e.value), str(e.value)
    # a good contour passes the checks and reaches the job, which a config-only voice cannot run
    vol = np.array([6, NAN, 0, 0, -INF, -3, 0], np.float32)
    err = N.sb200_error()
    rc = lib.sb200_speak_batch_ids_volume(config_only._h, i64(ids), sz(offs), 2, None, None, None, None, None, None,
                                          None, None, None, None, None, None, None, None, f32(vol), outs, None, None,
                                          None, None, C.byref(err))
    with pytest.raises(OperationError) as e:
        _check(rc, err)
    assert "volume" not in str(e.value)
    # the debug hook checks its levels before any device work
    x = np.zeros(10, np.float32)
    err = N.sb200_error()
    rc = lib.sb200_debug_volume(0, f32(x), 10, i64(np.array([10], np.int64)), f32(np.array([21.0], np.float32)), 1,
                                22050, f32(x), C.byref(err))
    with pytest.raises(OperationError, match=re.escape("id 0: volume level 21.000000 dB")):
        _check(rc, err)


def test_stream_options_name_the_stream(config_only):
    with pytest.raises(OperationError, match=re.escape("stream 2, id 1: volume level 40.0 dB")):
        _stream_options(config_only, "StreamBatch", 2, [1, 5, 2], volume_contour=[0.0, 40.0, 0.0])
    with pytest.raises(OperationError, match=re.escape("stream: 2 volume levels for 3 ids")):
        _stream_options(config_only, "stream_synthesis", None, [1, 5, 2], volume_contour=[0.0, 4.0])
    o = _stream_options(config_only, "stream_synthesis", None, [1, 5, 2], volume_contour=[0.0, 4.0, None])
    assert o.volume == [0.0, 4.0, None]


def test_models_without_streaming_voices_refuse_by_name():
    class Other:
        pass
    with pytest.raises(OperationError, match="stream_synthesis cannot apply a volume contour"):
        VitsStreamingModel.stream_synthesis(Other(), "ab", 10, 3, volume_contour=[0.0, 0.0])
