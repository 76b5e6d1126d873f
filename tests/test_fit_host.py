"""Target durations without a GPU: the numpy contract (tests/fit_reference.py) on crafted w, the Python and library
checks and their messages, the tempo refusal, the character-to-id span mapping and the C images."""
import ctypes as C
import math
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import fit_reference as fr
import sonata_b200
from sonata_b200 import _native as N, voicegen
from sonata_b200.core import OperationError
from sonata_b200.piper import (VitsStreamingModel, _batch_options, _char_targets_to_ids, _check, _stream_options,
                               _target_arrays)

NAN = float("nan")


def _next(u):
    return np.nextafter(np.float32(u), np.float32(np.inf))


def _holds(w, fixed, bud, u, f):
    """u is the contract's answer: it fits (or is 0.5 over the budget) and the next f32 does not fit."""
    assert f == fr.frames(w, fixed, u)
    if f > bud:
        assert u == fr.LO
    elif u < fr.HI:
        assert fr.frames(w, fixed, _next(u)) > bud


# ---------------------------------------------------------------------------------------------------- the contract
def test_plateaus_and_the_largest_u():
    w = np.array([3.0, 2.0, 5.0], np.float32)
    fixed = np.full(3, -1)
    for bud in range(5, 21):
        u, f = fr.solve(w, fixed, bud)
        _holds(w, fixed, bud, u, f)
        # the whole plateau below u* down to the previous step gives the same frames
        lower = [v for v in np.linspace(0.5, float(u), 50, dtype=np.float32) if fr.frames(w, fixed, v) == f]
        assert lower and fr.frames(w, fixed, lower[0]) == f


def test_a_jump_of_several_frames_at_one_u():
    # ten equal ids: at u = 0.7 every id steps together, so the sum jumps by 10 frames
    w = np.full(10, 10.0, np.float32)
    fixed = np.full(10, -1)
    u, f = fr.solve(w, fixed, 75)
    _holds(w, fixed, 75, u, f)
    assert f == 70 and fr.frames(w, fixed, _next(u)) == 80


def test_over_and_under_the_range():
    w = np.array([40.0, 60.0], np.float32)
    fixed = np.full(2, -1)
    u, f = fr.solve(w, fixed, 10)             # even 0.5 overruns: over its target
    assert u == np.float32(0.5) and f == 50
    u, f = fr.solve(w, fixed, 10**6)          # even 2 fits: the longest delivery
    assert u == np.float32(2.0) and f == 200


def test_fixed_and_zero_count_ids():
    w = np.array([0.0, 4.0, 1e-30, 7.0], np.float32)
    fixed = np.array([-1, 9, -1, -1])
    u, f = fr.solve(w, fixed, 20)
    _holds(w, fixed, 20, u, f)
    assert fr.counts(w[[0]], u)[0] == 0 and fr.counts(w[[2]], u)[0] == 1
    # a span of fixed ids only asks for nothing
    assert fr.solve(w[1:2], fixed[1:2], 3) == (np.float32(1.0), 9)


def test_saturation():
    w = np.array([np.inf, np.nan, 3e9], np.float32)
    assert fr.counts(w, 1.0).tolist() == [fr.INT_MAX] * 3
    u, f = fr.solve(w, np.full(3, -1), 10)
    assert u == np.float32(0.5) and f == 2 * fr.INT_MAX + 1500000000     # 3e9 * 0.5 fits an int again


def test_breaks_inside_a_span_count_in_P():
    rate = 22050
    w = np.array([5.0, 5.0, 5.0, 5.0], np.float32)
    fixed = np.full(4, -1)
    brk = np.array([NAN, 100.0, 0.0, 10.0], np.float32)
    (got,), factor, c = fr.fit(w, fixed, [(0, 4, 400.0)], rate, brk)
    P = int(math.floor(100.0 * rate / 1000 + 0.5)) + int(math.floor(10.0 * rate / 1000 + 0.5))
    T = fr.target_samples(400.0, rate)
    u, L = got
    assert L <= T and L == 256 * int(c.sum()) + P
    assert u < fr.HI and fr.frames(w, fixed, _next(u)) * 256 + P > T
    # the same span without breaks takes longer
    (nob,), _, _ = fr.fit(w, fixed, [(0, 4, 400.0)], rate)
    assert nob[0] > u


def test_ids_outside_the_spans_are_untouched():
    rng = np.random.default_rng(3)
    w = rng.uniform(0, 12, 30).astype(np.float32)
    fixed = np.full(30, -1)
    spans = [(2, 9, 800.0), (9, 12, NAN), (20, 30, 300.0)]
    res, factor, c = fr.fit(w, fixed, spans, 22050)
    assert (factor[:2] == 1).all() and (factor[9:20] == 1).all()
    assert (c[:2] == np.ceil(w[:2])).all() and (c[9:20] == np.ceil(w[9:20])).all()
    assert math.isnan(res[1][0]) and res[1][1] == -1
    for (a, e, ms), (u, L) in zip(spans, res):
        if not math.isnan(ms):
            bud = fr.budget(fr.target_samples(ms, 22050), 0)
            _holds(w[a:e], fixed[a:e], bud, u, L // 256)


@pytest.mark.parametrize("seed", range(6))
def test_random_spans_hold_the_contract(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 80))
    w = rng.choice([0.0, 0.3, 1.0, 2.5, 7.0, 19.0], n).astype(np.float32) * rng.uniform(0.5, 1.5, n).astype(np.float32)
    fixed = np.where(rng.random(n) < 0.15, rng.integers(0, 9, n), -1)
    bud = int(rng.integers(-3, 400))
    u, f = fr.solve(w, fixed, bud)
    if (fixed < 0).any():
        _holds(w, fixed, bud, u, f)


# ---------------------------------------------------------------------------------------------------- Python checks
@pytest.mark.parametrize("targets,msg", [
    ([None, 0.0], "utterance 1: target duration 0.0 ms is not a finite value in (0.0, 600000.0]"),
    ([None, 600001], "utterance 1: target duration 600001.0 ms"),
    ([math.inf, None], "utterance 0: target duration inf ms"),
    ([-5.0, None], "utterance 0: target duration -5.0 ms"),
    (["2s", None], "utterance 0: target durations '2s' are neither"),
    ([[(0, 1, 500.0), (1, 2, 300.0)], None], "utterance 0, span 1: ids 1 .. 2 overlap or precede the span before it"),
    ([[(2, 3, 500.0), (0, 1, 300.0)], None], "utterance 0, span 1: ids 0 .. 1 overlap or precede"),
    ([None, [(0, 4, 500.0)]], "utterance 1, span 0: ids 0 .. 4 are not a range of the 4 ids"),
    ([None, [(2, 1, 500.0)]], "utterance 1, span 0: ids 2 .. 1 are not a range"),
    ([None, [(0, 1, 700000.0)]], "utterance 1, span 0: target duration 700000.0 ms"),
    ([None, [(0, 1)]], "utterance 1, span 0: (0, 1) is not a (first, last, ms) span"),
    ([None, [(0.5, 1, 100.0)]], "utterance 1, span 0: ids 0.5 .. 1 are not integers"),
    ([None], "Invalid target durations: 1 entries for 2 utterances"),
])
def test_python_checks_name_the_utterance_and_the_span(targets, msg):
    with pytest.raises(OperationError) as e:
        _batch_options(None, 2, [5, 4], target_durations=targets)
    assert msg in str(e.value), str(e.value)


def test_a_target_and_a_tempo_are_refused():
    with pytest.raises(OperationError, match="utterance 1: a target duration and a tempo ratio together"):
        _batch_options(None, 2, [5, 4], tempos=[None, 1.5], target_durations=[None, 900.0])
    # a target that asks for nothing, or a tempo of 1, goes
    _batch_options(None, 2, [5, 4], tempos=[None, 1.5], target_durations=[None, NAN])
    _batch_options(None, 2, [5, 4], tempos=[None, 1.0], target_durations=[None, 900.0])


def test_checks_come_after_breaks():
    with pytest.raises(OperationError, match="break"):
        _batch_options(None, 1, [3], breaks=[[0.0, -1.0, 0.0]], target_durations=[-1.0])


def test_the_c_images():
    t = _target_arrays([5, 4, 3], [[(0, 1, 300.0), (3, 4, NAN)], None, 700.0])
    first, end, ms, offs = t
    assert first.dtype == np.int64 and end.dtype == np.int64 and ms.dtype == np.float32 and offs.dtype == np.uint64
    assert first.tolist() == [0, 3, 0] and end.tolist() == [2, 5, 3] and offs.tolist() == [0, 2, 2, 3]
    assert ms[0] == 300.0 and math.isnan(ms[1]) and ms[2] == 700.0
    # nothing that asks: no table, so no launch and no copy
    assert _target_arrays([5], [NAN]) is None and _target_arrays([5], [None]) is None
    assert _batch_options(None, 2, [5, 4], target_durations=[None, [(0, 1, NAN)]]).targets is None


def test_character_spans_map_to_ids():
    # bos, 'a' (id, pad), 'b' dropped, 'c' (id, pad), eos
    src = [-1, 0, 0, 2, 2, -1]
    assert _char_targets_to_ids([(0, 2, 500.0)], "abc", src, 0) == [(1, 4, 500.0)]
    assert _char_targets_to_ids([(0, 0, 100.0), (2, 2, 200.0)], "abc", src, 0) == [(1, 2, 100.0), (3, 4, 200.0)]
    assert _char_targets_to_ids(800.0, "abc", src, 0) == 800.0
    with pytest.raises(OperationError, match=re.escape("utterance 3, span 0: characters 1 .. 1 map to no id")):
        _char_targets_to_ids([(1, 1, 100.0)], "abc", src, 3)
    with pytest.raises(OperationError, match=re.escape("span 0: characters 0 .. 3 are not a range of the 3 characters")):
        _char_targets_to_ids([(0, 3, 100.0)], "abc", src, 0)


def test_phoneme_surfaces_map_in_map_characters():
    o = _batch_options(None, 2, None, target_durations=[[(0, 1, 400.0)], 900.0])
    assert o.per_character and o.targets is None
    maps = [([1, 5, 0, 6, 0, 2], [-1, 0, 0, 1, 1, -1]), ([1, 7, 0, 2], [-1, 0, 0, -1])]
    o.map_characters(["ab", "c"], maps)
    assert o.targets[0].tolist() == [1, 0] and o.targets[1].tolist() == [5, 4] and o.targets[3].tolist() == [0, 1, 2]


# ---------------------------------------------------------------------------------------------------- library checks
@pytest.fixture(scope="module")
def config_only(lib_built):
    p = voicegen.write_voice(voicegen.default_voice_dir(), "medium")
    m = sonata_b200.VitsStreamingModel(p, device=-1)
    yield m
    m.close()


def test_the_c_entry_point_refuses_before_any_device_work(config_only):
    lib = N.lib()
    ids = np.array([1, 5, 2, 1, 6, 7, 2], np.int64)
    offs = np.array([0, 3, 7], np.uint64)
    i64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))
    f32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    sz = lambda a: a.ctypes.data_as(C.POINTER(C.c_size_t))
    outs = (N.sb200_audio * 2)()

    def speak(first, end, ms, fo, tempo=None):
        err = N.sb200_error()
        args = [np.array(first, np.int64), np.array(end, np.int64), np.array(ms, np.float32), np.array(fo, np.uint64)]
        rc = lib.sb200_speak_batch_ids_fit(config_only._h, i64(ids), sz(offs), 2, None, None, None, None, None, None,
                                           None, None, None if tempo is None else f32(tempo), None, None, None, None,
                                           None, None, None, i64(args[0]), i64(args[1]), f32(args[2]), sz(args[3]),
                                           outs, None, None, None, None, None, None, C.byref(err))
        with pytest.raises(OperationError) as e:
            _check(rc, err)
        return str(e.value)
    assert "utterance 1, span 0: ids [0, 5) are not a non-empty range of the 4 ids" in speak([0], [5], [100], [0, 0, 1])
    assert "utterance 0, span 1: ids [1, 2) overlap or precede" in speak([0, 1], [2, 2], [100, 100], [0, 2, 2])
    assert "utterance 0, span 0: target duration 0.000000 ms is not a finite value in (0, 600000]" in \
        speak([0], [3], [0.0], [0, 1, 1])
    assert "utterance 1: a target duration and a tempo ratio" in \
        speak([0], [4], [100.0], [0, 0, 1], np.array([NAN, 1.5], np.float32))
    # good targets pass the checks and reach the job, which a config-only voice cannot run
    assert "span" not in speak([0, 2], [2, 3], [100.0, NAN], [0, 2, 2])


def test_stream_options_name_the_stream(config_only):
    with pytest.raises(OperationError, match=re.escape("stream 2, span 0: ids 0 .. 3 are not a range of the 3 ids")):
        _stream_options(config_only, "StreamBatch", 2, [1, 5, 2], target_duration=[(0, 3, 100.0)])
    with pytest.raises(OperationError, match=re.escape("stream: a target duration and a tempo ratio")):
        _stream_options(config_only, "stream_synthesis", None, [1, 5, 2], tempo=1.2, target_duration=500.0)
    o = _stream_options(config_only, "stream_synthesis", None, [1, 5, 2], target_duration=[(1, 2, 300)])
    assert o.target == [(1, 2, 300.0)]


def test_models_without_streaming_voices_refuse_by_name():
    class Other:
        pass
    with pytest.raises(OperationError, match="stream_synthesis cannot fit a target duration"):
        VitsStreamingModel.stream_synthesis(Other(), "ab", 10, 3, target_duration=500.0)
