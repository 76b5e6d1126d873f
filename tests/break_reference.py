"""Executable specification of breaks (include/sonata_b200.h, sb200_speak_batch_ids_breaks): a pause in ms after any
id, inserted into the delivered samples at the voice's rate.  Every operation is float64, each rounded as numpy rounds
it, in the header's order, so the device agrees bit for bit."""
import numpy as np


def samples(ms, rate: int) -> np.ndarray:
    """N_i = floor(ms_i R / 1000 + 0.5) per id, 0 for NaN / 0."""
    ms = np.asarray(ms, np.float32).astype(np.float64)
    asked = ~np.isnan(ms) & (ms != 0)
    n = np.floor(np.where(asked, ms, 0.0) * rate / 1000.0 + 0.5)
    return np.where(asked, n, 0).astype(np.int64)


def plan(ends, ms, rate: int):
    """(P, M): the merged breaks' positions (ascending) and lengths; breaks of 0 samples dropped, those at equal ends
    summed in id order."""
    P, M = [], []
    for e, n in zip(np.asarray(ends, np.int64).tolist(), samples(ms, rate).tolist()):
        if n == 0:
            continue
        if P and P[-1] == e:
            M[-1] += n
        else:
            P.append(e)
            M.append(n)
    return np.array(P, np.int64), np.array(M, np.int64)


def half(rate: int) -> int:
    return rate // 200


def step(t):
    return t * t * (3.0 - 2.0 * t)


def fades(n2: int, P, rate: int) -> np.ndarray:
    """h_j (f32) for j in [0, n2): 1.0 times the fade-out and fade-in of each break, in ascending k."""
    F = half(rate)
    h = np.ones(n2, np.float64)
    j = np.arange(n2, dtype=np.int64)
    for p in np.asarray(P, np.int64).tolist():
        out = (j >= p - F) & (j < p)
        h[out] = h[out] * step(((p - j[out]).astype(np.float64) - 0.5) / F)
        inn = (j >= p) & (j < p + F)
        h[inn] = h[inn] * step(((j[inn] - p).astype(np.float64) + 0.5) / F)
    return h.astype(np.float32)


def apply(x, ends, ms, rate: int) -> np.ndarray:
    """The paused signal of x (n2 samples) whose id i ends at ends[i] with a break of ms[i] after it."""
    x = np.asarray(x, np.float32)
    P, M = plan(ends, ms, rate)
    if P.size == 0:
        return x.copy()
    y = x * fades(x.size, P, rate)
    D = np.concatenate([[0], np.cumsum(M)])
    out = np.zeros(x.size + int(D[-1]), np.float32)
    k = np.searchsorted(P, np.arange(x.size), side="right")      # #{k : P_k <= j}
    out[np.arange(x.size) + D[k]] = y
    return out


def delivered_ends(ends, ms, rate: int) -> np.ndarray:
    """E'_i = E_i + sum of M_k over P_k <= E_i."""
    ends = np.asarray(ends, np.int64)
    P, M = plan(ends, ms, rate)
    D = np.concatenate([[0], np.cumsum(M)]).astype(np.int64)
    return ends + D[np.searchsorted(P, ends, side="right")]


def emitted(J, P, M) -> int:
    """O(J) = J + sum of M_k over P_k <= J: what a stream's stage has emitted once it has received J samples."""
    P, M = np.asarray(P, np.int64), np.asarray(M, np.int64)
    return int(J) + int(M[P <= J].sum())
