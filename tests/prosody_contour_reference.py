"""The specification of pitch contours (include/sonata_b200.h, sb200_speak_batch_ids_contour) in numpy: the pieces,
their knots, the analysis positions and the delivered ends in float64 with every operation rounded as written; the
offsets and the overlap-add are those of tests/prosody_reference.py fed these positions, and the pitch stage a
windowed-sinc sum whose position and kernel follow the piece of each output."""
import math

import numpy as np

import prosody_reference as pr


def _ratio(v):
    v = np.float32(v)
    return np.float32(1.0) if np.isnan(v) else v


def pieces(n, ends, ratios):
    """(B int64[m + 1], p float64[m]): ids with 0 samples dropped, runs of equal f32 ratios merged; one piece of ratio 1
    when every id is empty."""
    B, P = [0], []
    prev = 0
    for e, r in zip(ends, ratios):
        e, r = int(e), _ratio(r)
        assert prev <= e <= n
        if e > prev:
            if P and P[-1] == r:
                B[-1] = e
            else:
                B.append(e)
                P.append(r)
        prev = e
    if not P:
        return np.array([0, n], np.int64), np.array([1.0])
    assert prev == n
    return np.array(B, np.int64), np.array([float(p) for p in P])


def plan(rate, n, ends, ratios, tempo=None):
    """dict(Hs, N, D, n1, n2, F, a (int64[F]), bounds (int64, one per id), B, S, Q, alpha, p, m, stretch, pitch, one):
    `one` is the single-piece plan of prosody_reference when the ids make one piece (the ratio it equals)."""
    B, p = pieces(n, ends, ratios)
    _, t = pr.ratios(None, tempo)
    t = float(t)
    m = len(p)
    Hs, D = rate // 100, rate // 160
    alpha = p / t
    S = np.zeros(m + 1)
    for r in range(m):
        S[r + 1] = S[r] + float(B[r + 1] - B[r]) * alpha[r]
    Q = np.zeros(m)
    for r in range(m - 1):
        Q[r + 1] = Q[r] + (S[r + 1] - S[r]) / p[r]
    stretch = not (m == 1 and p[0] == t)
    pitch = not (m == 1 and p[0] == 1.0)
    n1 = int(math.floor(S[m] + 0.5)) if stretch else n
    n2 = int(math.floor(Q[m - 1] + (n1 - S[m - 1]) / p[m - 1] + 0.5)) if pitch else n1
    F = -(-n1 // Hs) if stretch else 0
    a = np.zeros(F, np.int64)
    r = 0
    for k in range(F):
        kh = float(k * Hs)
        while r + 1 < m and kh >= S[r + 1]:
            r += 1
        a[k] = math.floor(float(B[r]) + (kh - S[r]) / alpha[r] + 0.5)
    bounds = np.zeros(len(ends), np.int64)
    r = 0
    for i, b in enumerate(ends):
        b = int(b)
        while b > B[r + 1]:
            r += 1
        bounds[i] = math.floor(Q[r] + (float(b - B[r]) * alpha[r]) / p[r] + 0.5)
    if len(ends):
        bounds[-1] = n2
    one = pr.plan(rate, n, float(p[0]), tempo) if m == 1 else None
    return dict(Hs=Hs, N=2 * Hs, D=D, n1=n1, n2=n2, F=F, a=a, bounds=bounds, B=B, S=S, Q=Q, alpha=alpha, p=p, m=m,
                stretch=stretch, pitch=pitch, one=one)


def positions(pl):
    """Output j's piece index and position pos (float64[n2])."""
    j = np.arange(pl["n2"], dtype=np.float64)
    r = np.searchsorted(pl["Q"], j, side="right") - 1
    return r, pl["S"][r] + (j - pl["Q"][r]) * pl["p"][r]


def pitch_resample(s, pl):
    """(y float64[n2], bound float64[n2]) of the float64 stretched signal s (length n1)."""
    s = np.asarray(s, np.float64)
    n1 = pl["n1"]
    r, pos = positions(pl)
    pj = pl["p"][r]
    W = 16.0 * np.maximum(1.0, pj)
    i0 = np.floor(pos - W).astype(np.int64)
    y, mag = np.zeros(pl["n2"]), np.zeros(pl["n2"])
    taps = int(2 * W.max()) + 1
    for q in range(taps + 2):
        i = i0 + q
        u = pos - i
        c = np.minimum(1.0, 1.0 / pj)
        h = c * np.sinc(c * u) * (0.42 + 0.5 * np.cos(np.pi * u / W) + 0.08 * np.cos(2 * np.pi * u / W))
        h = np.where(np.abs(u) < W, h, 0.0)
        v = np.where((i >= 0) & (i < n1), s[np.clip(i, 0, max(n1 - 1, 0))] if n1 else 0.0, 0.0)
        y += v * h
        mag += np.abs(v * h)
    return y, (taps + 2) * 2.0 ** -24 * mag + 2e-6


def process(x, rate, ends, ratios, tempo=None):
    """dict(plan, offsets, s (float64 or None), s_bound, y float64, y_bound): the whole stage in float64."""
    pl = plan(rate, len(x), ends, ratios, tempo)
    if pl["one"] is not None:
        out = pr.process(x, rate, None if pl["p"][0] == 1.0 else float(pl["p"][0]), tempo)
        out["plan"] = pl
        return out
    out = dict(plan=pl)
    out["offsets"] = pr.offsets(x, pl)
    out["s"], out["s_bound"] = pr.overlap_add(x, pl, out["offsets"])
    out["y"], out["y_bound"] = pitch_resample(out["s"], pl)
    return out
