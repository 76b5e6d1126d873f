"""The emission rule of a pitch / tempo stream (include/sonata_b200.h, sb200_decode_chunks_warped) in Python, built on
prosody_reference.plan: what each chunk of a stream emits, and how much history it holds between chunks."""
import math

import numpy as np

import prosody_reference as pr


def _analysis(Hs, alpha, k):
    return -Hs if k < 0 else int(math.floor(float(k * Hs) / alpha + 0.5))


def _radius(p):
    return 16.0 / (1.0 / p if p > 1.0 else 1.0)


def chunkings(n, seed=0):
    """Chunk lengths of n samples: one whole chunk, 256 and 14 080 samples at a time, and random lengths (0 included)."""
    rng = np.random.default_rng(seed)
    rand, left = [], n
    while left > 0:
        rand.append(min(left, int(rng.integers(0, 3000))))
        left -= rand[-1]
    split = lambda m: [m] * (n // m) + ([n % m] if n % m else [])
    return {"one": [n], "256": split(256), "14080": split(14080), "random": rand}


def caps(rate, pitch, tempo):
    """(input history, stretched history): the most samples a stream holds between chunks."""
    pl = pr.plan(rate, 0, pitch, tempo)
    tail = 2 * math.ceil(_radius(pl["p"])) + 4 if pl["pitch"] else 0
    if not pl["stretch"]:
        return tail, 0
    return max(math.ceil(2.0 * pl["Hs"] / pl["alpha"]), pl["Hs"]) + 2 * pl["D"] + pl["N"] + 4, tail


def stream(rate, pitch, tempo, chunk_lens):
    """[dict(emitted, frames, stretched, h_in, h_s)] per chunk, the last chunk ending the stream."""
    pl = pr.plan(rate, 0, pitch, tempo)
    Hs, N, D, alpha, p = pl["Hs"], pl["N"], pl["D"], pl["alpha"], pl["p"]
    a = lambda k: _analysis(Hs, alpha, k)
    W = _radius(p)
    C = K = S = J = 0
    out = []
    for i, n in enumerate(chunk_lens):
        last = i + 1 == len(chunk_lens)
        C += int(n)
        J0 = J
        if last:
            e = pr.plan(rate, C, pitch, tempo)
            K, S, J = e["F"], e["n1"], e["n2"]
            h_in = h_s = 0
        else:
            S = C
            if pl["stretch"]:
                while max(a(K - 1) + D + Hs + N, a(K) + D + N) <= C:
                    K += 1
                S = min(K * Hs, int(math.floor(C * alpha + 0.5)))
            J = S
            if pl["pitch"]:
                J = J0
                while math.ceil(J * p + W) <= S:
                    J += 1
            pitch_from = min(S, max(0, math.floor(J * p - W) + 1)) if pl["pitch"] else S
            if pl["stretch"]:
                in_from = 0 if K == 0 else max(0, min(a(K - 2) + Hs, a(K - 1)) - D)
                h_in, h_s = C - min(in_from, C), (S - pitch_from if pl["pitch"] else 0)
            else:
                h_in, h_s = C - pitch_from, 0
        out.append(dict(emitted=J - J0, frames=K, stretched=S, h_in=h_in, h_s=h_s))
    return out
