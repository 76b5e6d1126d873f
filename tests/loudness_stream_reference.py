"""Float64 restatement of a live loudness stream (include/sonata_b200.h, sb200_loudness_stream_create): the causal
BS.1770 meter of everything delivered so far, its readings at each 100 ms step boundary, the gains they give and the
ramp, scale and clamp of every sample.  Built on loudness_reference's design, step and gates."""
import math

import numpy as np

import loudness_reference as lr


def _energies(x, rate):
    """q_c of every complete step of x: the sum of y^2 over samples [cS, (c + 1)S) of the K-weighted signal."""
    from scipy.signal import lfilter
    (bs, as_), (bh, ah) = lr.design(rate)
    y = lfilter(bh, ah, lfilter(bs, as_, np.asarray(x, np.float64)))
    S = lr.step(rate)
    return np.array([np.sum(y[c * S:(c + 1) * S] ** 2) for c in range(len(y) // S)])


def _gated(z):
    """integrated()'s gates over block energies z."""
    with np.errstate(divide="ignore"):
        l = -0.691 + 10.0 * np.log10(z)
    keep = l > -70.0
    if not keep.any():
        return -math.inf
    rel = -0.691 + 10.0 * math.log10(np.mean(z[keep])) - 10.0
    keep &= l > rel
    if not keep.any():
        return -math.inf
    return -0.691 + 10.0 * math.log10(np.mean(z[keep]))


def readings(x, rate):
    """L_m, m = 1 .. floor(len(x) / S): the gated loudness of x[0, mS) from m = 4 on (integrated(x[:mS]), computed from
    the step energies, which a causal filter makes the same), the provisional mean square before it."""
    q = _energies(x, rate)
    S = lr.step(rate)
    out = []
    for m in range(1, len(q) + 1):
        if m >= 4:
            nb = m - 3
            z = (q[:nb] + q[1:nb + 1] + q[2:nb + 2] + q[3:nb + 3]) / (4 * S)
            out.append(_gated(z))
        else:
            s = 0.0
            for c in range(m):
                s += q[c]
            L = -0.691 + 10.0 * math.log10(s / (m * S)) if s > 0.0 else -math.inf
            out.append(-math.inf if L <= -70.0 else L)
    return np.array(out, np.float64)


def gains(L, target, max_gain_db=20.0, a0=1.0):
    """a_0 .. a_M for readings L_1 .. L_M: a_m keeps a_{m-1} without a reading, else
    f32(min(10^((T - L_m)/20), 10^(M/20)))."""
    a = [np.float32(a0)]
    cap = 10.0 ** (max_gain_db / 20.0)
    for l in L:
        a.append(a[-1] if l == -math.inf else np.float32(min(10.0 ** ((target - l) / 20.0), cap)))
    return np.array(a, np.float32)


def sample_gains(n, a, S):
    """G_i of samples 0 .. n: a_0 in step 0, then the ramp a_{m-1} + (a_m - a_{m-1}) (i - mS + 1) / S in float64 with
    each operation rounded, to f32."""
    i = np.arange(n, dtype=np.int64)
    m = i // S
    lo = np.asarray(a, np.float64)[np.maximum(m - 1, 0)]
    hi = np.asarray(a, np.float64)[m]
    g = lo + ((hi - lo) * (i - m * S + 1).astype(np.float64)) / float(S)
    g[m == 0] = a[0]
    return g.astype(np.float32)


def meter(x, rate, target, max_gain_db=20.0):
    """(y, L, a, clipped) of a fresh meter over the whole of x: the metered f32 samples, readings L_1 .. L_M, gains
    a_1 .. a_M and the samples clamped."""
    x = np.asarray(x, np.float32)
    S = lr.step(rate)
    L = readings(x, rate)
    a = gains(L, target, max_gain_db)
    v = x * sample_gains(len(x), a, S)
    clipped = int(np.count_nonzero(np.abs(v) > 1.0))
    return np.clip(v, -1.0, 1.0).astype(np.float32), L, a[1:], clipped


class Meter:
    """The same meter fed chunk by chunk: push(chunk) returns the metered chunk, computed from everything pushed so
    far only (the signal before the boundary of the step each sample is in)."""

    def __init__(self, rate, target, max_gain_db=20.0):
        self.rate, self.target, self.max_gain_db = rate, target, max_gain_db
        self.x = np.zeros(0, np.float32)

    def push(self, chunk):
        n0 = len(self.x)
        self.x = np.concatenate([self.x, np.asarray(chunk, np.float32)])
        S = lr.step(self.rate)
        # samples [n0, n) need the gains up to the boundary of the step of sample n - 1, which x[0, n) determines
        L = readings(self.x, self.rate)
        a = gains(L, self.target, self.max_gain_db)
        v = self.x[n0:] * sample_gains(len(self.x), a, S)[n0:]
        return np.clip(v, -1.0, 1.0).astype(np.float32)
