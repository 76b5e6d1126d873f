"""The emission rule of a stream with a pitch contour (include/sonata_b200.h, sb200_prosody_stream_create_contour) in
Python, built on prosody_contour_reference.plan: what each chunk of a contoured stream emits, and how much history it
holds between chunks.  A contour that makes one piece is the ratio stream of prosody_stream_reference."""
import math

import prosody_contour_reference as pcr
import prosody_stream_reference as psr


def _radius(p):
    return 16.0 / (1.0 / p if p > 1.0 else 1.0)


def caps(pl):
    """(input history, stretched history) of a plan of two or more pieces: the most samples it holds between chunks."""
    Hs, N, D = pl["Hs"], pl["N"], pl["D"]
    w_max = max(_radius(float(p)) for p in pl["p"])
    alpha_min = float(min(pl["alpha"]))
    return max(math.ceil(2.0 * Hs / alpha_min), Hs) + 2 * D + N + 4, 2 * math.ceil(w_max) + 4


def stream(rate, n, ends, ratios, tempo, chunk_lens):
    """[dict(emitted, frames, stretched, h_in, h_s)] per chunk, the last chunk ending the stream.  Raises ValueError
    when the contour and the tempo ask for nothing, or when the chunks do not add up to n."""
    if sum(int(c) for c in chunk_lens) != n:
        raise ValueError("the chunks do not add up to the stream's input")
    pl = pcr.plan(rate, n, ends, ratios, tempo)
    if pl["one"] is not None:
        p = float(pl["p"][0])
        if not pl["stretch"] and not pl["pitch"]:
            raise ValueError("a contour and tempo that ask for nothing")
        return psr.stream(rate, None if p == 1.0 else p, tempo, chunk_lens)
    Hs, N, D, m = pl["Hs"], pl["N"], pl["D"], pl["m"]
    B, S_, Q, alpha, P = pl["B"], pl["S"], pl["Q"], pl["alpha"], pl["p"]

    def a(k):
        if k < 0:
            return -Hs
        kh = float(k * Hs)
        r = max(q for q in range(m) if S_[q] <= kh)
        return math.floor(float(B[r]) + (kh - float(S_[r])) / float(alpha[r]) + 0.5)

    def sigma(x):
        r = max(q for q in range(m) if B[q] <= x)
        return float(S_[r]) + float(x - B[r]) * float(alpha[r])

    def piece(j):
        return max(q for q in range(m) if Q[q] <= j)

    def pos(j):
        r = piece(j)
        return float(S_[r]) + (float(j) - float(Q[r])) * float(P[r]), _radius(float(P[r]))

    w_max = max(_radius(float(p)) for p in P)
    C = K = S = J = 0
    out = []
    for i, c in enumerate(chunk_lens):
        last = i + 1 == len(chunk_lens)
        C += int(c)
        J0 = J
        if last:
            K, S, J = pl["F"], pl["n1"], pl["n2"]
            h_in = h_s = 0
        else:
            while max(a(K - 1) + D + Hs + N, a(K) + D + N) <= C:
                K += 1
            S = min(K * Hs, math.floor(sigma(C) + 0.5))
            while True:
                x, W = pos(J)
                if math.ceil(x + W) > S:
                    break
                J += 1
            pitch_from = min(S, max(0, math.floor(pos(J)[0] - w_max) + 1))
            in_from = 0 if K == 0 else max(0, min(a(K - 2) + Hs, a(K - 1)) - D)
            h_in, h_s = C - min(in_from, C), S - pitch_from
        out.append(dict(emitted=J - J0, frames=K, stretched=S, h_in=h_in, h_s=h_s))
    return out
