"""GPU (-m gpu): the live loudness meter (loudness_stream_kernel) at its edges.

Every output bit follows from the kernel's own gains: y_i = clamp(f32(x_i G_i), -1, 1) with G_i the ramp of the header
evaluated in double with each operation rounded (loudness_stream_reference.sample_gains), and every gain from the
kernel's own reading.  The readings are held to the batch meter's bits and to float64 (1e-6 LU) on streams whose
readings gate more blocks than the kernel has threads, chunked so that one launch completes more steps than that or
every chunk carries S - 1 samples; at the meter's full capacity of 2^16 steps and one step past it; on silence, the
gates and the gain cap; and through the decoder on long requests."""
import ctypes as C
import os
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import loudness_reference as lr
import loudness_stream_edges as le
import loudness_stream_reference as lsr
from test_loudness_stream_gpu import DEFAULT, _message, _metered, _unmetered, batch_lufs, f32p, f64p, hook
from test_loudness_stream_host import _speechlike
from sonata_b200 import voicegen, workload
from sonata_b200 import _native as N
from sonata_b200.piper import LoudnessStream, VitsStreamingModel

pytestmark = pytest.mark.gpu
STEPS_PER_SLICE = 1 << 12       # the output check rebuilds G this many steps at a time


@pytest.fixture(scope="module")
def voices(lib_built):
    d = voicegen.default_voice_dir()
    ms = {}

    def get(q):
        if q not in ms:
            ms[q] = VitsStreamingModel(voicegen.write_voice(d, q), device=0)
            ms[q].set_fallback_synthesis_config(DEFAULT)
        return ms[q]
    yield get
    for m in ms.values():
        m.close()


def check_bits(x, run, rate, target, max_gain_db=20.0):
    """The hook's (y, L, a, clipped) over x against its own readings: a_m = a_{m-1} bit for bit where L_m = -inf, else
    within 1 f32 ulp of f32(min(10^((T - L_m)/20), 10^(M/20))); y = clamp(f32(x G), -1, 1) bit for bit with G rebuilt
    from a_0 = 1, a_1 .. a_M; the clamp count exact.  Returns how many gains are not bit-equal to that expression."""
    y, L, a, clipped = run
    S = lr.step(rate)
    M = len(x) // S
    assert len(y) == len(x) and len(L) == len(a) == M
    a_all = np.concatenate([[np.float32(1)], a]).astype(np.float32)
    held = L == -np.inf
    assert a[held].tobytes() == a_all[:-1][held].tobytes()
    want = np.minimum(10.0 ** ((target - L[~held]) / 20.0), 10.0 ** (max_gain_db / 20.0)).astype(np.float32)
    ulps = np.abs(a[~held].view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    assert ulps.max(initial=0) <= 1
    clip = 0
    for k0 in range(0, M + 1, STEPS_PER_SLICE):
        i0, i1 = k0 * S, min(len(x), (k0 + STEPS_PER_SLICE) * S)
        if i0 >= i1:
            break
        # a slice from boundary k0 > 0 ramps from a_{k0 - 1}: rebuild it one step early and drop that step
        G = lsr.sample_gains(i1, a_all, S) if k0 == 0 else lsr.sample_gains(i1 - i0 + S, a_all[k0 - 1:], S)[S:]
        v = x[i0:i1] * G
        assert np.clip(v, -1.0, 1.0).tobytes() == y[i0:i1].tobytes(), (i0, i1)
        clip += int(np.count_nonzero(np.abs(v) > 1.0))
    assert clip == clipped
    return int(np.count_nonzero(ulps))


def against_float64(x, L, rate, ms=None, what=""):
    """The hook's readings at ms (default: every m) against the float64 reference: the same finite set, within 1e-6 LU.
    Prints and returns the worst error."""
    S = lr.step(rate)
    ms = list(range(1, len(L) + 1)) if ms is None else list(ms)
    want = le.readings_at(lsr._energies(x, rate), S, ms)
    got = L[np.array(ms) - 1]
    fin = np.isfinite(want)
    assert np.array_equal(np.isfinite(got), fin)
    err = float(np.max(np.abs(got[fin] - want[fin]), initial=0.0))
    print(f"\nL against float64 at {rate} Hz ({what}): worst {err:.3e} LU over {int(fin.sum())} finite readings")
    assert err <= 1e-6
    return err


def against_batch(x, L, rate, ms):
    S = lr.step(rate)
    for m in ms:
        assert L[m - 1] == batch_lufs(x[:m * S], rate), m


def same_runs(runs):
    y, L, a, clipped = runs[0]
    for r in runs[1:]:
        assert r[0].tobytes() == y.tobytes()
        assert r[1].tobytes() == L.tobytes() and r[2].tobytes() == a.tobytes() and r[3] == clipped


# ---------------------------------------------------------------- every rate


@pytest.mark.parametrize("rate", lr.RATES)
def test_output_bits_follow_the_kernels_gains_at_every_rate(rate):
    S = lr.step(rate)
    x = le.long_signal(rate, 262, S // 2, rate)
    ch = le.long_chunkings(len(x), rate, rate)
    runs = [hook(x, ch[k], rate, -16.0) for k in ("one", "mixed")]
    same_runs(runs)
    off = check_bits(x, runs[0], rate, -16.0)
    print(f"\n{rate} Hz: {off} of {len(runs[0][2])} gains one ulp from f32(min(10^((T - L)/20), 10^(M/20)))")
    assert runs[0][3] > 0
    against_float64(x, runs[0][1], rate, what="every rate")
    against_batch(x, runs[0][1], rate, (4, 258, 259, 260, 262))


# ---------------------------------------------------------------- long streams


@pytest.mark.parametrize("rate,steps,tail", le.LONG_CASES)
def test_long_streams_in_any_chunking(rate, steps, tail):
    x = le.long_signal(rate, steps, tail, 11 + rate)
    ch = le.long_chunkings(len(x), rate, rate)
    runs = []
    for name in ("one", "second", "carry", "mixed"):
        t = time.perf_counter()
        runs.append(hook(x, ch[name], rate, -16.0))
        print(f"\n{rate} Hz, {steps} steps, {name} ({len(ch[name])} chunks): {time.perf_counter() - t:.2f} s")
    same_runs(runs)
    y, L, a, clipped = runs[0]
    assert len(L) == steps and clipped > 0
    off = check_bits(x, runs[0], rate, -16.0)
    print(f"{off} of {steps} gains one ulp from the expression")
    against_batch(x, L, rate, le.check_ms(steps))
    against_float64(x, L, rate, what=f"{steps} steps")


# ---------------------------------------------------------------- capacity


def test_a_full_meter():
    rate, S, n = le.CAP_RATE, le.CAP_S, le.CAP_ACCEPTED
    x = _speechlike(rate, (n + 1) / rate, 77)[:n]
    x[1000 * S:1020 * S] = 0.0
    x[(le.LS_MAX_STEPS - 7) * S:(le.LS_MAX_STEPS - 6) * S] *= 6.0
    t = time.perf_counter()
    run = hook(x, [n], rate, -16.0)
    print(f"\nthe full meter ({le.LS_MAX_STEPS} steps at {rate} Hz) in one chunk: {time.perf_counter() - t:.2f} s")
    y, L, a, clipped = run
    assert len(L) == le.LS_MAX_STEPS
    against_batch(x, L, rate, (4, 260, 1 << 15, le.LS_MAX_STEPS))
    against_float64(x, L, rate, le.cap_ms(), what="full meter")
    off = check_bits(x, run, rate, -16.0)
    print(f"{off} of {len(a)} gains one ulp from the expression")


def test_one_step_past_capacity_is_refused_and_nothing_is_written():
    rate, S, n = le.CAP_RATE, le.CAP_S, le.CAP_REFUSED
    x = np.full(n, 0.25, np.float32)
    M = n // S
    y = np.full(n, 7.0, np.float32)
    L, a = np.full(M, 7.0), np.full(M, 7.0, np.float32)
    clipped, err = C.c_int64(-7), N.sb200_error()
    lens = np.array([n], np.uint64)
    rc = N.lib().sb200_debug_loudness_stream(0, f32p(x), lens.ctypes.data_as(C.POINTER(C.c_size_t)), 1, rate, -16.0,
                                             20.0, f32p(y), f64p(L), f32p(a), C.byref(clipped), C.byref(err))
    assert rc != 0 and "capacity of 65536 steps" in _message(err)
    assert np.all(y == 7.0) and np.all(L == 7.0) and np.all(a == 7.0) and clipped.value == -7


# ---------------------------------------------------------------- gates and gain


def test_a_stream_under_the_absolute_gate_is_untouched():
    rate = 16000
    x = _speechlike(rate, 30.0, 5) * np.float32(3e-4)
    ch = le.long_chunkings(len(x), rate, 5)
    runs = [hook(x, ch[k], rate, -16.0) for k in ("one", "mixed")]
    same_runs(runs)
    y, L, a, clipped = runs[0]
    assert np.all(le.readings_at(lsr._energies(x, rate), lr.step(rate), range(1, len(L) + 1)) == -np.inf)
    assert np.all(L == -np.inf) and np.all(a == 1.0) and clipped == 0
    assert y.tobytes() == x.tobytes()
    check_bits(x, runs[0], rate, -16.0)


def test_silence_then_speech_holds_the_gain_until_a_block_passes():
    rate = 16000
    S = lr.step(rate)
    x = np.concatenate([np.zeros(10 * rate, np.float32), _speechlike(rate, 10.0, 6)])
    ch = le.long_chunkings(len(x), rate, 6)
    runs = [hook(x, ch[k], rate, -16.0) for k in ("one", "second")]
    same_runs(runs)
    y, L, a, clipped = runs[0]
    first = int(np.argmax(np.isfinite(L))) + 1        # the first boundary with a reading
    assert first == 101                               # block 97 (steps 97 .. 100) holds the first speech step
    assert np.all(L[:first - 1] == -np.inf) and np.all(a[:first - 1] == 1.0) and a[first - 1] != 1.0
    assert not y[:10 * rate].view(np.uint32).any()
    # the first speech step still plays at a_99 = a_100 = 1
    assert y[10 * rate:(first - 1) * S].tobytes() == x[10 * rate:(first - 1) * S].tobytes()
    check_bits(x, runs[0], rate, -16.0)
    against_batch(x, L, rate, (100, 101, 102, len(L)))
    against_float64(x, L, rate, what="silence, then speech")


def test_speech_then_silence_freezes_the_reading():
    rate = 16000
    S = lr.step(rate)
    speech = _speechlike(rate, 10.0, 8)
    speech[-S:] *= 4.0                                 # loud up to the last sample, so the filter rings on
    x = np.concatenate([speech, np.zeros(60 * rate, np.float32)])
    ch = le.long_chunkings(len(x), rate, 8)
    runs = [hook(x, ch[k], rate, -16.0) for k in ("one", "second")]
    same_runs(runs)
    y, L, a, clipped = runs[0]
    # in float64 the K-weighting rings on into the silence, but from some block on none passes the absolute gate
    q = lsr._energies(x, rate)
    z = (q[:-3] + q[1:-2] + q[2:-1] + q[3:]) / (4 * S)
    assert q[100] > 0.0 and q[101] > 0.0
    with np.errstate(divide="ignore"):
        passing = np.nonzero(-0.691 + 10.0 * np.log10(z) > -70.0)[0]
    stop = int(passing[-1]) + 4                        # the first reading that includes the last passing block
    assert 100 <= stop <= 106
    assert np.all(L[stop - 1:] == L[stop - 1]) and np.isfinite(L[stop - 1])
    assert np.all(a[stop - 1:] == a[stop - 1])
    assert L[stop - 1:].tobytes() == np.full(len(L) - stop + 1, L[stop - 1]).tobytes()
    assert a[stop - 1:].tobytes() == np.full(len(a) - stop + 1, a[stop - 1]).tobytes()
    against_batch(x, L, rate, (stop, stop + 1, 400, len(L)))
    assert not y[len(speech):].view(np.uint32).any()   # exact +0.0
    check_bits(x, runs[0], rate, -16.0)
    against_float64(x, L, rate, what="speech, then silence")


def test_the_relative_gate_drops_a_quiet_section_and_keeps_a_louder_one():
    rate = 16000
    seg = 20 * rate                                    # 200 steps each
    tone = lr.sine(rate, 60.0, peak=0.5)
    level = np.concatenate([np.full(seg, 1.0), np.full(seg, 10 ** (-15 / 20)), np.full(seg, 10 ** (-5 / 20))])
    x = (tone * level.astype(np.float32)).astype(np.float32)
    ch = le.long_chunkings(len(x), rate, 9)
    runs = [hook(x, ch[k], rate, -23.0) for k in ("one", "carry")]
    same_runs(runs)
    y, L, a, clipped = runs[0]
    # blocks 200 .. 396 lie in the section 15 LU down: each reading that adds one adds nothing that passes both gates
    assert L[203 - 1:400].tobytes() == np.full(400 - 203 + 1, L[202]).tobytes()
    # blocks from 400 on lie 5 LU down: kept, each one lowers the reading
    assert np.all(np.diff(L[404 - 1:]) < 0)
    assert L[-1] < L[399] - 0.5
    check_bits(x, runs[0], rate, -23.0)
    against_batch(x, L, rate, (203, 300, 400, 404, len(L)))
    against_float64(x, L, rate, what="relative gate")


@pytest.mark.parametrize("target,max_gain_db,scale", ((-16.0, 0.0, 0.007), (-16.0, 40.0, 0.007), (0.0, 20.0, 1.0),
                                                      (-70.0, 20.0, 1.0)))
def test_gain_cap_and_target_edges(target, max_gain_db, scale):
    rate = 16000
    x = _speechlike(rate, 12.0, 10) * np.float32(scale)
    ch = le.long_chunkings(len(x), rate, 10)
    runs = [hook(x, ch[k], rate, target, max_gain_db) for k in ("one", "mixed")]
    same_runs(runs)
    y, L, a, clipped = runs[0]
    fin = np.isfinite(L)
    assert fin.sum() > 50
    if max_gain_db == 0.0:                             # no gain above 1: the stream passes unchanged
        assert np.all(a == 1.0) and y.tobytes() == x.tobytes()
    elif max_gain_db == 40.0:                          # 43 .. 51 dB asked: the cap of exactly 100 holds
        assert np.all(a[fin] == np.float32(100.0))
    elif target == 0.0:
        assert np.all(a[fin] > 4.0) and clipped > 0
    else:
        assert np.all(a[fin] < 0.01) and clipped == 0
    check_bits(x, runs[0], rate, target, max_gain_db)
    against_float64(x, L, rate, what=f"T {target}, M {max_gain_db}")


# ---------------------------------------------------------------- the decoder at long length


def _encode(m, phonemes, utt0):
    ids = [list(workload.synthetic_ids(p, utt=utt0 + i)) for i, p in enumerate(phonemes)]
    encs = m.infer_encoder_batch(ids, seeds=[utt0 + i for i in range(len(ids))],
                                 durations=[[le.FRAMES_PER_ID] * len(s) for s in ids])
    for enc, p in zip(encs, phonemes):
        assert enc.num_frames == le.frames(p)
    return encs


def _stream_and_hook(m, encs, cs, pad, out_rate):
    """The encs as one request's sentences, through one meter: (joined metered chunks, the unmetered chunks, the hook
    over them, the meter's state)."""
    meter = LoudnessStream(m, -16.0, output_rate=out_rate)
    plain, got = [], []
    for enc in encs:
        plain += _unmetered(m, enc, cs, pad, out_rate)
        got += [c.as_slice() for c in _metered(m, enc, cs, pad, out_rate, meter)]
    assert [len(c) for c in got] == [len(c) for c in plain]
    x = np.concatenate(plain)
    run = hook(x, [len(c) for c in plain], out_rate, -16.0)
    return np.concatenate(got), plain, x, run, meter.state()


@pytest.mark.parametrize("out_rate", le.OUT_RATES)
def test_a_long_request_in_ordinary_chunks(voices, out_rate):
    m = voices("medium")
    got, plain, x, run, st = _stream_and_hook(m, _encode(m, le.REQUEST_PHONEMES, 40), *le.REQUEST_CHUNK, out_rate)
    assert len(x) > 30 * out_rate and len(plain) > 3 * len(le.REQUEST_PHONEMES)
    assert got.tobytes() == run[0].tobytes()
    check_bits(x, run, out_rate, -16.0)
    assert st["samples"] == len(x) and st["clipped"] == run[3]
    assert st["gain"] == run[2][-1] and st["lufs"] == run[1][-1]


@pytest.mark.parametrize("out_rate", le.OUT_RATES)
def test_one_chunk_past_256_steps(voices, out_rate):
    m = voices("medium")
    got, plain, x, run, st = _stream_and_hook(m, _encode(m, (le.LONG_PHONEMES,), 50), *le.LONG_CHUNK, out_rate)
    assert len(plain) == 1 and len(x) // lr.step(out_rate) > le.LD_THREADS
    assert got.tobytes() == run[0].tobytes()
    check_bits(x, run, out_rate, -16.0)
    assert st["samples"] == len(x) and st["clipped"] == run[3]
    assert st["gain"] == run[2][-1] and st["lufs"] == run[1][-1]
