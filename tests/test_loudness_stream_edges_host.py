"""CPU: the float64 reference and case tables of the live loudness meter's edge tests -- readings_at against
loudness_stream_reference.readings at every boundary, and arithmetic on the tables showing that each GPU case reaches
the edge it is there for."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import loudness_reference as lr
import loudness_stream_edges as le
import loudness_stream_reference as lsr
from test_loudness_stream_host import _speechlike


@pytest.mark.parametrize("rate", (8000, 22050, 48000))
def test_readings_at_is_the_reference_at_every_boundary(rate):
    x = _speechlike(rate, 3.1, seed=rate)
    x[int(0.4 * rate):int(1.1 * rate)] = 0.0
    q = lsr._energies(x, rate)
    S = lr.step(rate)
    want = lsr.readings(x, rate)
    ms = list(range(1, len(q) + 1))
    assert np.array_equal(le.readings_at(q, S, ms), want)
    # any subset, in any order, and the provisional boundaries alone
    sub = [len(q), 4, 1, 17, 3, 2]
    assert np.array_equal(le.readings_at(q, S, sub), want[np.array(sub) - 1])
    assert np.array_equal(le.readings_at(q[:3], S, [1, 2, 3]), want[:3])


def test_readings_at_on_silence_and_a_quiet_start():
    rate = 16000
    S = lr.step(rate)
    x = np.zeros(8 * S, np.float32)
    q = lsr._energies(x, rate)
    assert np.all(le.readings_at(q, S, range(1, 9)) == -np.inf)
    x = np.concatenate([np.zeros(2 * S, np.float32), _speechlike(rate, 0.6, 3)])
    q = lsr._energies(x, rate)
    assert np.array_equal(le.readings_at(q, S, range(1, len(q) + 1)), lsr.readings(x, rate))


@pytest.mark.parametrize("rate,steps,tail", le.LONG_CASES)
def test_long_streams_gate_past_one_and_two_blocks_per_thread(rate, steps, tail):
    S = lr.step(rate)
    x = le.long_signal(rate, steps, tail, 1)
    assert len(x) == steps * S + tail and 0 <= tail < S
    blocks = set(range(1, steps - 3 + 1))                # m - 3 for m = 4 .. steps
    assert set(le.EDGE_BLOCKS) <= blocks
    # blocks per thread of ld_gates at the last reading: two or three
    assert -(-(steps - 3) // le.LD_THREADS) >= 2
    # the boundaries compared bit for bit with the batch meter cover both edges
    ms = le.check_ms(steps)
    assert {b + 3 for b in le.EDGE_BLOCKS} <= set(ms) and 4 in ms and steps in ms and len(ms) >= 20
    assert max(c for r, c, _ in le.LONG_CASES) > 1000


@pytest.mark.parametrize("rate,steps,tail", le.LONG_CASES)
def test_long_chunkings_reach_their_edges(rate, steps, tail):
    S = lr.step(rate)
    n = steps * S + tail
    ch = le.long_chunkings(n, rate, 7)
    for lens in ch.values():
        assert sum(lens) == n and min(lens) > 0
    # one chunk: every step in one launch, so steps (2) and (4) loop past the block's 256 threads
    assert le.steps_completed(ch["one"], S) == [steps] and steps > 2 * le.LD_THREADS
    # 1 s chunks: ten steps each
    assert set(le.steps_completed(ch["second"][:-1], S)) == {10}
    # every chunk but the last leaves S - 1 samples in the carry
    c = le.carries(ch["carry"], S)
    assert set(c[:-1]) == {S - 1} and len(c) > 20
    # the mix has 1-sample chunks, chunks that complete no step and chunks that complete several
    done = le.steps_completed(ch["mixed"], S)
    assert 1 in ch["mixed"] and 0 in done and max(done) >= 10


def test_capacity_totals_fall_either_side():
    S = le.CAP_S
    assert S == 800
    assert le.CAP_ACCEPTED // S == le.LS_MAX_STEPS and le.CAP_ACCEPTED % S == S - 1
    assert le.CAP_REFUSED // S == le.LS_MAX_STEPS + 1
    ms = le.cap_ms()
    assert {1, 2, 3, 4, le.LS_MAX_STEPS - 1, le.LS_MAX_STEPS} <= set(ms) and len(ms) >= 20
    # one chunk of the full meter completes 2^16 steps: 256 per thread in steps (2) and (4)
    assert le.steps_completed([le.CAP_ACCEPTED], S) == [le.LS_MAX_STEPS]


def test_decoder_streams_are_long_enough():
    for rate in le.OUT_RATES:
        S = lr.step(rate)
        total = sum(le.delivered(le.frames(p), rate) for p in le.REQUEST_PHONEMES)
        assert total > 30 * rate
        cs, pad = le.LONG_CHUNK
        f = le.frames(le.LONG_PHONEMES)
        assert f <= 2 * cs + 2 * pad                                 # one chunk
        assert le.delivered(f, rate) // S > le.LD_THREADS            # that completes more than 256 steps
        cs, pad = le.REQUEST_CHUNK
        assert all(le.frames(p) > 2 * cs + 2 * pad for p in le.REQUEST_PHONEMES)   # ordinary chunks
