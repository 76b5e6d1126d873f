"""Executable specification of target durations (include/sonata_b200.h, sb200_speak_batch_ids_fit): each span's
predicted ids get one f32 factor u, c_i(u) = ceil(w_i u), and u* is the largest f32 u in [0.5, 2] whose frames fit the
span's budget.  Given w, numpy's f32 multiply and ceil are exact, so the device agrees bit for bit."""
import numpy as np

HOP = 256
INT_MAX = 2**31 - 1
LO, HI = np.float32(0.5), np.float32(2.0)


def target_samples(ms, rate: int) -> int:
    """T = floor(ms R / 1000 + 0.5) in double, ms first rounded to f32 as the library receives it."""
    return int(np.floor(float(np.float32(ms)) * rate / 1000.0 + 0.5))


def counts(w, u) -> np.ndarray:
    """c_i(u) = ceil(w_i u) as int64, one f32 multiply, saturating at INT_MAX (NaN and inf too)."""
    c = np.ceil(np.asarray(w, np.float32) * np.float32(u))
    with np.errstate(invalid="ignore"):
        ok = c < np.float32(2.0**31)
    return np.where(ok, np.where(ok, c, 0).astype(np.int64), INT_MAX)


def frames(w, fixed, u) -> int:
    """A span's frames at u: predicted ids (fixed < 0) take ceil(w u), the others their fixed count."""
    fixed = np.asarray(fixed, np.int64)
    pred = fixed < 0
    return int(counts(np.asarray(w, np.float32)[pred], u).sum() + fixed[~pred].sum())


def budget(T: int, P: int, hop: int = HOP) -> int:
    """The most frames a span may take: floor((T - P) / hop)."""
    return (T - P) // hop


def solve(w, fixed, bud: int):
    """(u*, frames at u*) of one span: the largest f32 u in [0.5, 2] with frames(u) <= bud, by bisection over the f32
    bit patterns; 0.5 when even that overruns; 1.0 for a span without a predicted id."""
    fixed = np.asarray(fixed, np.int64)
    if not (fixed < 0).any():
        return np.float32(1.0), int(fixed.sum())
    f = frames(w, fixed, LO)
    if f > bud:
        return LO, f
    lo, hi = int(LO.view(np.uint32)), int(HI.view(np.uint32))
    while lo < hi:
        mid = lo + (hi - lo + 1) // 2
        t = frames(w, fixed, np.uint32(mid).view(np.float32))
        if t <= bud:
            lo, f = mid, t
        else:
            hi = mid - 1
    return np.uint32(lo).view(np.float32), f


def fit(w, fixed, spans, rate: int, breaks_ms=None, hop: int = HOP):
    """One utterance: spans [(first, end, ms)] over ids with w (f32) and fixed counts (-1: predicted), breaks per id
    (None: none).  Returns (per span (u*, L) with L = hop frames + P, NaN / -1 for a span that asks nothing; the
    factor image; the fitted counts per id)."""
    w = np.asarray(w, np.float32)
    fixed = np.asarray(fixed, np.int64)
    factor = np.ones(w.size, np.float32)
    out = []
    for a, e, ms in spans:
        if np.isnan(ms):
            out.append((np.float32(np.nan), -1))
            continue
        P = 0
        if breaks_ms is not None:
            b = np.asarray(breaks_ms, np.float32)[a:e].astype(np.float64)
            asked = ~np.isnan(b) & (b != 0)
            P = int(np.floor(np.where(asked, b, 0.0) * rate / 1000.0 + 0.5)[asked].sum())
        u, f = solve(w[a:e], fixed[a:e], budget(target_samples(ms, rate), P, hop))
        if (fixed[a:e] < 0).any():
            factor[a:e] = u
        out.append((u, hop * f + P))
    c = np.where(fixed >= 0, fixed, counts(w * factor, 1.0))
    return out, factor, c
