"""The speaker-blend contract (include/sonata_b200.h, sb200_speak_batch_ids_blends) as numpy.

A blend is n >= 1 pairs (s_i, u_i): distinct speaker ids and finite f32 weights u_i >= 0, not all zero.
  1. Canonical form: drop the pairs with u_i = 0, sort the rest by s ascending, U = sum of (double) u_i in that order,
     w_i = (float)((double) u_i / U).
  2. Embedding: acc = 0.0f, then acc = fmaf(w_i, emb_g[s_i][k], acc) for each i in canonical order; g[k] = acc.
  3. Conditioning: the effective biases base[r] + sum_k W[r][k] g[k]."""
import numpy as np


def canonical(pairs):
    """(speakers int64, weights f32) of the canonical form of pairs [(s, u), ...]; ValueError for a blend the library
    refuses (ids are not checked against a voice here)."""
    if not pairs:
        raise ValueError("empty blend")
    seen = set()
    for s, u in pairs:
        if s in seen:
            raise ValueError(f"speaker {s} appears more than once")
        seen.add(s)
        u = np.float32(u)
        if not (np.isfinite(u) and u >= 0):
            raise ValueError(f"weight {u} of speaker {s}")
    kept = sorted((int(s), np.float32(u)) for s, u in pairs if np.float32(u) > 0)
    if not kept:
        raise ValueError("every weight is zero")
    U = 0.0
    for _, u in kept:
        U += float(u)
    return (np.array([s for s, _ in kept], np.int64),
            np.array([np.float32(float(u) / U) for _, u in kept], np.float32))


def _fmaf(a, b, c):
    """fmaf in f32: a * b + c rounded once.  a * b is exact in float64; the sum is taken in float64 with its rounding
    error (TwoSum) and made round-to-odd, which then rounds to f32 exactly as a single rounding would."""
    a, b, c = (np.asarray(x, np.float64) for x in (a, b, c))
    p = a * b                                   # exact: 24 + 24 bits
    s = p + c
    bp = s - c
    err = (p - bp) + (c - (s - bp))
    s_odd = s.copy()
    inexact = err != 0
    bits = s_odd.view(np.int64)
    fix = inexact & ((bits & 1) == 0)
    bits[fix & (np.sign(err) == np.sign(s_odd))] += 1
    bits[fix & (np.sign(err) != np.sign(s_odd)) & (s_odd != 0)] -= 1
    return s_odd.astype(np.float32)


def blend_g(emb_g, speakers, weights):
    """g [gin] of a canonical blend, bit for bit as the device forms it (f32 fused multiply-adds in canonical order)."""
    emb_g = np.asarray(emb_g, np.float32)
    acc = np.zeros(emb_g.shape[1], np.float32)
    for s, w in zip(speakers, weights):
        acc = _fmaf(np.float32(w), emb_g[int(s)], acc)
    return acc


def blend_g64(emb_g, speakers, weights):
    """The float64 weighted sum sum_i w_i E[s_i] (the exact value the f32 g approximates) and the bound
    n 2^-24 sum_i |w_i E[s_i][k]| per element."""
    E = np.asarray(emb_g, np.float64)
    terms = np.stack([float(w) * E[int(s)] for s, w in zip(speakers, weights)])
    return terms.sum(0), len(speakers) * 2.0 ** -24 * np.abs(terms).sum(0)
