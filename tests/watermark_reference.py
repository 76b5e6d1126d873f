"""The watermark's specification (include/sonata_b200.h, sb200_voice_set_watermark and sb200_watermark_detect) in
numpy: chips from Philox4x32-10, block sums in int64, gains in float64 with one rounding per operation, the mark as
one float32 multiply and one float32 add; detection by an exact int64 fold, the phase transform and two circular
correlations in float64."""
import math

import numpy as np

from noise_reference import philox4x32_10
from prosody_reference import quantise

P = 4096
THRESHOLD = 6.5


def chips(key: int) -> np.ndarray:
    """int64 [2][P]: c_j[m] = +1 when bit 0 of word 0 of the block of counter (m, j, 0, 0) under key is 1, else -1."""
    m = np.arange(P, dtype=np.uint32)
    out = np.empty((2, P), np.int64)
    k = np.array([key & 0xFFFFFFFF, (key >> 32) & 0xFFFFFFFF], np.uint32)
    for j in range(2):
        ctr = np.stack([m, np.full(P, j, np.uint32), np.zeros(P, np.uint32), np.zeros(P, np.uint32)], axis=-1)
        out[j] = np.where(philox4x32_10(ctr, k)[:, 0] & 1, 1, -1)
    return out


def chip_total(c: np.ndarray, payload: int, n: np.ndarray) -> np.ndarray:
    """c[n] = c0[n mod P] + c1[(n - s) mod P] at positions n (int64)."""
    n = np.asarray(n, np.int64)
    return c[0][n % P] + c[1][(n - payload) % P]


def alpha(strength_db: float) -> float:
    return 10.0 ** (float(np.float32(strength_db)) / 20.0)


def gains(x: np.ndarray, rate: int, strength_db: float) -> np.ndarray:
    """a_k per block of B = rate // 100 samples, float32."""
    q = quantise(x)
    B = rate // 100
    K = -(-q.size // B)
    if K == 0:
        return np.zeros(0, np.float32)
    S = np.add.reduceat(q * q, np.arange(0, q.size, B))
    L = np.minimum(B, q.size - np.arange(K) * B).astype(np.float64)
    Sp, Lp = np.concatenate([S[:1], S[:-1]]), np.concatenate([L[:1], L[:-1]])
    E = np.minimum(Sp.astype(np.float64) / Lp, S.astype(np.float64) / L)
    return ((alpha(strength_db) * np.sqrt(E * 0.5)) / 32767.0).astype(np.float32)


def embed(x, rate: int, key: int, payload: int, strength_db: float, c=None) -> np.ndarray:
    """The marked signal, bit for bit what the stage delivers."""
    x = np.asarray(x, np.float32)
    c = chips(key) if c is None else c
    a = gains(x, rate, strength_db)
    n = np.arange(x.size, dtype=np.int64)
    mark = a[n // (rate // 100)] * chip_total(c, payload, n).astype(np.float32)
    return (x + mark).astype(np.float32)


def fold(clip) -> np.ndarray:
    """F[m] = sum of q[i] over i = m mod P, int64: q = the clip itself for int16, quantise(clip) for float32."""
    clip = np.asarray(clip)
    q = clip.astype(np.int64) if clip.dtype == np.int16 else quantise(clip)
    pad = np.zeros(-(-q.size // P) * P, np.int64)
    pad[:q.size] = q
    return pad.reshape(-1, P).sum(axis=0)


def score(r: np.ndarray):
    """(o, z) of one correlation: the first argmax and its z over the other P - 1 lags."""
    o = int(np.argmax(r))
    others = np.delete(r, o)
    sd = float(others.std())
    return o, 0.0 if sd == 0.0 else (float(r[o]) - float(others.mean())) / sd


def correlations(F: np.ndarray, c: np.ndarray):
    """r_j[o] = sum_m w[m] c_j[(m + o) mod P], w the phase transform of F: float64 [2][P]."""
    X = np.fft.fft(F.astype(np.float64))
    mag = np.abs(X)
    W = np.where(mag > 0, X / np.where(mag > 0, mag, 1.0), 0)
    return np.stack([np.real(np.fft.ifft(np.conj(W) * np.fft.fft(c[j].astype(np.float64)))) for j in range(2)])


def detect(clip, key: int, c=None) -> dict:
    c = chips(key) if c is None else c
    r = correlations(fold(clip), c)
    o0, z0 = score(r[0])
    o1, z1 = score(r[1])
    marked = z0 >= THRESHOLD
    return dict(marked=bool(marked), payload=(o0 - o1) % P if marked and z1 >= THRESHOLD else -1, offset=o0, z0=z0,
                z1=z1)


def standardised_lags(clip, key: int, c=None) -> np.ndarray:
    """Both correlations' lags other than their peaks, standardised: about N(0, 1) without a mark."""
    c = chips(key) if c is None else c
    r = correlations(fold(clip), c)
    out = []
    for j in range(2):
        o = int(np.argmax(r[j]))
        others = np.delete(r[j], o)
        out.append((others - others.mean()) / others.std())
    return np.concatenate(out)


def expected_z(strength_db: float, marked_samples: int) -> float:
    """z of a white host signal: (alpha / sqrt 2) sqrt(marked samples)."""
    return alpha(strength_db) / math.sqrt(2.0) * math.sqrt(marked_samples)


def stream(chunks, rate: int, key: int, payload: int, strength_db: float, c=None):
    """A stream's marked chunks, computed chunk by chunk as the stage does: after J samples received it has emitted
    floor(J / B) B of them, all on the last chunk; each block's gain uses the S carried from the block before it."""
    c = chips(key) if c is None else c
    B = rate // 100
    alpha_ = alpha(strength_db)
    held = np.zeros(0, np.float32)
    out, pos, s_prev = [], 0, None
    for i, x in enumerate(chunks):
        z = np.concatenate([held, np.asarray(x, np.float32)])
        last = i == len(chunks) - 1
        n = z.size if last else z.size // B * B
        e, held = z[:n], z[n:]
        K = -(-n // B)
        q = quantise(e)
        S = np.add.reduceat(q * q, np.arange(0, n, B)) if n else np.zeros(0, np.int64)
        L = np.minimum(B, n - np.arange(K) * B).astype(np.float64)
        if s_prev is None:
            Sp, Lp = np.concatenate([S[:1], S[:-1]]), np.concatenate([L[:1], L[:-1]])
        else:
            Sp, Lp = np.concatenate([[s_prev], S[:-1]]), np.concatenate([[float(B)], L[:-1]])
        E = np.minimum(Sp.astype(np.float64) / Lp, S.astype(np.float64) / L)
        a = ((alpha_ * np.sqrt(E * 0.5)) / 32767.0).astype(np.float32)
        m = np.arange(n, dtype=np.int64)
        out.append((e + a[m // B] * chip_total(c, payload, pos + m).astype(np.float32)).astype(np.float32))
        if K:
            s_prev = int(S[-1])
        pos += n
    return out
