"""The volume-contour contract (include/sonata_b200.h, sb200_speak_batch_ids_volume) as numpy.

A signal of n2 delivered samples at `rate`, whose id i ends at ends[i] (the last at n2) with levels[i] in dB (NaN or 0:
none, -inf: silence), is scaled sample by sample by a gain curve: one gain per piece (a run of ids with equal levels),
with a smoothstep ramp of L = 2 (rate // 200) samples centred on each boundary.  Every float64 operation below is one
rounded operation, as the kernel computes it."""
import math

import numpy as np


def gain_of(level) -> np.float32:
    """g = f32(10^(level / 20)) in double; 1 for NaN, 0 for -inf."""
    v = float(np.float32(level))
    if math.isnan(v):
        return np.float32(1.0)
    if v == -math.inf:
        return np.float32(0.0)
    return np.float32(math.pow(10.0, v / 20.0))


def pieces(ends, levels, n2):
    """(B, g): each piece's first delivered sample and gain, after dropping empty ids and merging runs of equal f32
    levels (NaN -> 0).  Raises ValueError for ends that go back, pass n2 or do not end at n2."""
    starts, gains = [], []
    prev, level = 0, None
    for e, v in zip(ends, levels):
        e = int(e)
        if e < prev or e > n2:
            raise ValueError(f"id ends at {e}")
        v = np.float32(0.0) if np.isnan(np.float32(v)) else np.float32(v)
        if e > prev and (level is None or v != level):
            starts.append(prev)
            gains.append(gain_of(v))
            level = v
        prev = e
    if len(ends) and prev != n2:
        raise ValueError(f"the last id ends at {prev}, not at {n2}")
    return np.array(starts, np.int64), np.array(gains, np.float32)


def asks(ends, levels, n2) -> bool:
    """Whether the stage runs: some piece's gain is not 1."""
    _, g = pieces(ends, levels, n2)
    return bool(np.any(g != np.float32(1.0)))


def gain_curve(starts, gains, rate, j):
    """G_j (f32) at the delivered positions j (int64 array)."""
    j = np.asarray(j, np.int64)
    m, half = len(starts), rate // 200
    L = float(2 * half)
    if m == 0:
        return np.ones(j.shape, np.float32)
    # the first boundary r >= 1 whose ramp B_r - half <= j < B_r + half could cover j: B_r > j - half
    lo = np.searchsorted(starts[1:], j - half, side="right") + 1
    acc = gains[lo - 1].astype(np.float64)
    for r in range(1, m):
        cover = (starts[r] - half <= j) & (j < starts[r] + half)
        if not cover.any():
            continue
        jj = j[cover]
        t = ((jj - starts[r] + half).astype(np.float64) + 0.5) / L
        s = (t * t) * (3.0 - 2.0 * t)
        acc[cover] = acc[cover] + (np.float64(gains[r]) - np.float64(gains[r - 1])) * s
    return acc.astype(np.float32)


def apply(x, ends, levels, rate, j0=0):
    """y = x G over delivered samples [j0, j0 + len(x)) of a signal of n2 = ends[-1] samples; x itself (a copy) when
    the contour asks for nothing."""
    x = np.asarray(x, np.float32)
    n2 = int(ends[-1]) if len(ends) else len(x)
    starts, gains = pieces(ends, levels, n2)
    if not np.any(gains != np.float32(1.0)):
        return x.copy()
    return x * gain_curve(starts, gains, rate, np.arange(j0, j0 + len(x), dtype=np.int64))


def gain_scalar(starts, gains, rate, j) -> np.float32:
    """G_j for one sample, written as the header states it (a cross-check of gain_curve)."""
    half = rate // 200
    L = 2 * half
    covering = [r for r in range(1, len(starts)) if starts[r] - half <= j < starts[r] + half]
    if not covering:
        a = max(r for r in range(len(starts)) if starts[r] <= j)
        return np.float32(gains[a])
    acc = float(gains[covering[0] - 1])
    for r in covering:
        t = (float(j - starts[r] + half) + 0.5) / float(L)
        acc = acc + (float(gains[r]) - float(gains[r - 1])) * ((t * t) * (3.0 - 2.0 * t))
    return np.float32(acc)
