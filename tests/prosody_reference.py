"""The specification of the pitch / tempo stage (include/sonata_b200.h, sb200_speak_batch_ids_prosody) in numpy:
integer offsets in int64, the overlap-add and the windowed-sinc sum in float64.  The kernels are held to it: offsets
exactly, waveforms within the bounds `ola_bound` and `pitch_bound` return."""
import math

import numpy as np

PITCH_RANGE = (0.5, 2.0)
TEMPO_RANGE = (0.25, 4.0)


def ratios(pitch, tempo):
    """(p, t) as the library holds them: float32 values, 1 for None / NaN."""
    f = lambda v: np.float32(1.0) if v is None or math.isnan(float(v)) else np.float32(v)
    return f(pitch), f(tempo)


def plan(rate, n, pitch=None, tempo=None):
    """dict(Hs, N, D, n1, n2, F, a (analysis positions, int64[F]), alpha, p, stretch, pitch)."""
    p, t = ratios(pitch, tempo)
    Hs, D = rate // 100, rate // 160
    alpha = float(p) / float(t)
    stretch, pit = bool(p != t), bool(p != 1)
    n1 = int(math.floor(n * alpha + 0.5)) if stretch else n
    n2 = int(math.floor(n1 / float(p) + 0.5)) if pit else n1
    F = -(-n1 // Hs) if stretch else 0
    a = np.floor(np.arange(F, dtype=np.float64) * Hs / alpha + 0.5).astype(np.int64)
    return dict(Hs=Hs, N=2 * Hs, D=D, n1=n1, n2=n2, F=F, a=a, alpha=alpha, p=float(p), stretch=stretch, pitch=pit)


def quantise(x):
    x = np.asarray(x, np.float32)
    return np.trunc(np.clip(x, np.float32(-1), np.float32(1)) * np.float32(32767)).astype(np.int64)


def _padded(v, lo, hi):
    """v[lo:hi] with zeros outside v."""
    out = np.zeros(hi - lo, v.dtype)
    a, b = max(lo, 0), min(hi, len(v))
    if b > a:
        out[a - lo:b - lo] = v[a:b]
    return out


def offsets(x, pl):
    """delta_k, k < F: the argmax of the exact integer scores, ties to the smaller |delta|, then to the negative one."""
    q = quantise(x)
    Hs, N, D, a = pl["Hs"], pl["N"], pl["D"], pl["a"]
    d = np.zeros(pl["F"], np.int64)
    lags = np.arange(-D, D + 1)
    order = np.lexsort((lags, np.abs(lags)))          # by |delta|, the negative one first
    for k in range(1, pl["F"]):
        c = int(a[k - 1] + d[k - 1] + Hs)
        ref = _padded(q, c, c + N)
        cand = _padded(q, int(a[k]) - D, int(a[k]) + D + N)
        scores = np.correlate(cand, ref, mode="valid")      # scores[l] = sum_i ref[i] cand[l + i], int64
        best = scores.max()
        d[k] = next(lags[l] for l in order if scores[l] == best)
    return d


def window(N):
    return 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(N) / N)


def overlap_add(x, pl, d):
    """(s float64[n1], bound float64[n1]): the two-term sum and the per-sample bound the f32 kernel is held to."""
    x = np.asarray(x, np.float64)
    Hs, N, a = pl["Hs"], pl["N"], pl["a"]
    m = np.arange(pl["n1"])
    k, r = m // Hs, m % Hs
    w = window(N)
    pos1 = a[k] + d[k] + r
    prev = np.where(k > 0, a[np.maximum(k - 1, 0)] + d[np.maximum(k - 1, 0)], -Hs)
    pos0 = prev + r + Hs
    take = lambda pos: np.where((pos >= 0) & (pos < len(x)), x[np.clip(pos, 0, len(x) - 1)], 0.0)
    t1, t0 = w[r] * take(pos1), w[r + Hs] * take(pos0)
    return t1 + t0, 4 * 2.0 ** -24 * (np.abs(t1) + np.abs(t0))


def kernel_h(u, p):
    c = min(1.0, 1.0 / p)
    W = 16.0 / c
    h = c * np.sinc(c * u) * (0.42 + 0.5 * np.cos(np.pi * u / W) + 0.08 * np.cos(2 * np.pi * u / W))
    return np.where(np.abs(u) < W, h, 0.0)


def pitch_resample(s, pl):
    """(y float64[n2], bound float64[n2]) of the float64 signal s (length n1)."""
    s = np.asarray(s, np.float64)
    p, n1, n2 = pl["p"], pl["n1"], pl["n2"]
    W = 16.0 * max(1.0, p)
    taps = int(2 * W) + 1
    pos = np.arange(n2, dtype=np.float64) * p
    i0 = np.floor(pos - W).astype(np.int64)
    y, mag = np.zeros(n2), np.zeros(n2)
    for q in range(taps + 2):
        i = i0 + q
        h = kernel_h(pos - i, p)
        v = np.where((i >= 0) & (i < n1), s[np.clip(i, 0, max(n1 - 1, 0))] if n1 else 0.0, 0.0)
        y += v * h
        mag += np.abs(v * h)
    return y, (taps + 2) * 2.0 ** -24 * mag + 2e-6


def process(x, rate, pitch=None, tempo=None):
    """dict(plan, offsets, s (float64 or None), s_bound, y float64, y_bound): the whole stage in float64."""
    pl = plan(rate, len(x), pitch, tempo)
    out = dict(plan=pl, offsets=np.zeros(0, np.int64), s=None, s_bound=None)
    cur = np.asarray(x, np.float64)
    bound = np.zeros(len(cur))
    if pl["stretch"]:
        out["offsets"] = offsets(x, pl)
        cur, bound = overlap_add(x, pl, out["offsets"])
        out["s"], out["s_bound"] = cur, bound
    if pl["pitch"]:
        cur, bound = pitch_resample(cur, pl)
    out["y"], out["y_bound"] = cur, bound
    return out


def tone(rate, freq, seconds, peak=0.5):
    t = np.arange(int(rate * seconds)) / rate
    return (peak * np.sin(2 * np.pi * freq * t)).astype(np.float32)


def spectral_peak_hz(x, rate):
    x = np.asarray(x, np.float64)
    spec = np.abs(np.fft.rfft(x * np.hanning(len(x))))
    return np.argmax(spec) * rate / len(x), rate / len(x)
