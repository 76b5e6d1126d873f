"""CPU: the emission rule of pitch / tempo streams (prosody_stream_reference) against the library's no-device plan hook,
and the rule's invariants: every stream emits exactly the whole-signal length, nothing before its end that a longer
input would not also produce, and never holds more history than its create-time buffers."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import prosody_reference as pr
import prosody_stream_reference as psr
from sonata_b200 import _native as N

RATES = (22050, 16000)
RATIOS = [(0.5, 0.25), (2.0, 4.0), (0.5, 4.0), (2.0, 0.25), (1.25, 1.25), (0.8, 0.8), (1.25, None), (None, 1.5),
          (0.8, 2.0), (None, 0.25), (2.0, None)]


def _lib_plan(rate, p, t, lens):
    lens = np.ascontiguousarray(lens, np.int64)
    out = np.zeros(len(lens), np.int64)
    f = lambda v: float("nan") if v is None else v
    rc = N.lib().sb200_debug_prosody_stream_plan(rate, f(p), f(t), lens.ctypes.data_as(C.POINTER(C.c_int64)),
                                                 len(lens), out.ctypes.data_as(C.POINTER(C.c_int64)))
    return rc, out


chunkings = psr.chunkings


@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("p,t", RATIOS)
def test_plan_hook_equals_the_rule(lib_built, rate, p, t):
    n = 2 * rate + 1234
    cap_in, cap_s = psr.caps(rate, p, t)
    whole = pr.plan(rate, n, p, t)
    for name, lens in chunkings(n, rate).items():
        ref = psr.stream(rate, p, t, lens)
        rc, got = _lib_plan(rate, p, t, lens)
        assert rc == 0, name
        np.testing.assert_array_equal(got, [r["emitted"] for r in ref], err_msg=name)
        assert int(got.sum()) == whole["n2"], name
        assert max(r["h_in"] for r in ref) <= cap_in and max(r["h_s"] for r in ref) <= cap_s, name


@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("p,t", [(0.5, 0.25), (2.0, 4.0), (0.5, 4.0), (1.25, 1.25), (0.8, 2.0)])
def test_single_samples(lib_built, rate, p, t):
    n = rate // 2 + 77
    lens = [1] * n
    ref = psr.stream(rate, p, t, lens)
    rc, got = _lib_plan(rate, p, t, lens)
    assert rc == 0
    np.testing.assert_array_equal(got, [r["emitted"] for r in ref])
    assert int(got.sum()) == pr.plan(rate, n, p, t)["n2"]
    cap_in, cap_s = psr.caps(rate, p, t)
    assert max(r["h_in"] for r in ref) <= cap_in and max(r["h_s"] for r in ref) <= cap_s


@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("p,t", RATIOS)
def test_library_emits_nothing_early(lib_built, rate, p, t):
    """The library's own plan: before its last chunk a stream has emitted no more than the whole-signal length of any
    longer input, whatever the chunking, and in total exactly that of its own."""
    n = rate + 4321
    for name, lens in chunkings(n, rate + 1).items():
        rc, got = _lib_plan(rate, p, t, lens)
        assert rc == 0, name
        emitted, consumed = np.cumsum(got), np.cumsum(lens)
        for i in range(len(lens) - 1):
            for extra in (0, 1, 7, 999):
                assert emitted[i] <= pr.plan(rate, int(consumed[i]) + extra, p, t)["n2"], (name, i, extra)
        assert emitted[-1] == pr.plan(rate, n, p, t)["n2"], name


@pytest.mark.parametrize("p,t", RATIOS)
def test_nothing_early_that_a_longer_input_would_not_produce(p, t):
    """Before its last chunk a stream has emitted no more than the whole-signal length of any longer input, and it
    has computed no frame or stretched sample past that input's own."""
    rate = 22050
    lens = [700] * 30
    ref = psr.stream(rate, p, t, lens[:-1] + [700, 1])    # never ends inside the prefix checked
    emitted = np.cumsum([r["emitted"] for r in ref])
    for i in range(len(lens) - 1):
        consumed = 700 * (i + 1)
        for extra in (0, 1, 5, 999):
            longer = pr.plan(rate, consumed + extra, p, t)
            assert emitted[i] <= longer["n2"], (i, extra)
            assert ref[i]["stretched"] <= longer["n1"], (i, extra)
            assert not longer["stretch"] or ref[i]["frames"] <= longer["F"], (i, extra)


def test_the_issue_example_keeps_the_length_bound():
    """p = 0.5, t = 4 at 22 050 Hz after 10 000 samples: 6 ready frames are 1 320 stretched samples, but n1 may be
    1 250; the stream computes 1 250."""
    r = psr.stream(22050, 0.5, 4.0, [10000, 1])[0]
    assert r["frames"] == 6 and r["stretched"] == 1250


class _Recorder:
    """A latent and model stand-in for SpeechStreamer: records each decoder call's keywords."""

    def __init__(self, frames):
        self.num_frames, self._m, self.calls = frames, self, []

    def infer_decoder_batch(self, chunks, **kw):
        self.calls.append((chunks, kw))
        return [b"" if kw.get("encoding") else None]


@pytest.mark.parametrize("frames", [150, 180, 206, 400])
@pytest.mark.parametrize("encoding", [None, "mulaw"])
@pytest.mark.parametrize("resampled", [False, True])
def test_streamer_flushes_its_last_chunk(frames, encoding, resampled):
    """Every route of SpeechStreamer that carries stream state flags exactly its last chunk as last, the one-shot
    chunk included (frames in (chunk + padding + 44, 2 chunk + 2 padding] are one-shot past the first window)."""
    from sonata_b200.piper import SpeechStreamer
    enc = _Recorder(frames)
    warp, rs = object(), (object() if resampled else None)
    list(SpeechStreamer(enc, 100, 3, resampler=rs, encoding=encoding, warp=warp))
    assert [kw["last"] for _, kw in enc.calls] == [[False]] * (len(enc.calls) - 1) + [[True]]
    assert all(kw["warps"] == [warp] and kw["resamplers"] == [rs] for _, kw in enc.calls)
    assert all(kw.get("encoding") == encoding for _, kw in enc.calls)
    if frames <= 206:
        assert len(enc.calls) == 1 and enc.calls[0][0][0][1:] == (0, frames, 0, 0)


def test_plan_hook_refuses_bad_arguments(lib_built):
    assert _lib_plan(22050, None, None, [100])[0] == 19
    assert _lib_plan(22050, 1.0, 1.0, [100])[0] == 19
    assert _lib_plan(22050, 2.5, None, [100])[0] == 19
    assert _lib_plan(22050, None, 0.2, [100])[0] == 19
    assert _lib_plan(500, 1.25, None, [100])[0] == 19
    assert _lib_plan(22050, 1.25, None, [100, -1])[0] == 19
