"""Case tables and helpers for the edge tests of the waveform stages after the decoder (formant, pitch / tempo,
output-rate resampling, loudness): the lengths, signals, ratios and contours where those kernels' runs, chains and
clamps change, and the library's device-free plan hooks that show each case reaches its edge.  Used by
tests/test_waveform_edges_host.py (the tables and the float64 specifications) and tests/test_waveform_edges_gpu.py (the
kernels against those specifications)."""
import ctypes as C
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import formant_reference as fr
import loudness_reference as lr
import prosody_contour_reference as pc
import prosody_reference as pr
import resample_reference as rr

NAN = float("nan")
RATES = (16000, 22050)
H = fr.H                     # the formant stage's hop
FM_HOPS = 32                 # hops of output per formant CTA
RS_OUTS = 1024               # outputs per resampler block run
PP_OUTS = 256                # outputs per pitch-resampler block run
LD_THREADS = 256             # threads of the loudness kernel's one block per utterance

f32p = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
i64p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))


def _nan(v):
    return NAN if v is None else float(v)


# ---------------------------------------------------------------- signals

def signals(n, rate, seed=0, loud=False, square_period=2):
    """name -> f32[n]: silence, impulses at the first sample, the last and a hop boundary, +-1 square, DC 1.0, noise,
    noise at 1e-20, an f32 denormal square (1e-40), the vowel; with `loud` also |x| > 1 (the quantiser's clamp) and
    the +-0.5 square of period 4 whose frames tie their lags."""
    rng = np.random.default_rng(seed * 100003 + n)
    out = {"silence": np.zeros(n, np.float32)}
    for name, at in (("impulse_first", 0), ("impulse_last", n - 1), ("impulse_hop", hop_boundary(n))):
        x = np.zeros(n, np.float32)
        x[at] = 1.0
        out[name] = x
    sq = np.where((np.arange(n) // (square_period // 2)) % 2 == 0, 1.0, -1.0).astype(np.float32)
    out["square"] = sq
    out["dc"] = np.ones(n, np.float32)
    out["noise"] = (0.3 * rng.standard_normal(n)).astype(np.float32)
    out["tiny"] = (1e-20 * rng.standard_normal(n)).astype(np.float32)
    out["denormal"] = (np.float32(1e-40) * sq).astype(np.float32)
    out["vowel"] = fr.vowel(rate, seconds=(n + 16) / rate)[:n]
    if loud:
        out["loud"] = np.clip(rng.standard_normal(n) * 2.0, -3, 3).astype(np.float32)
        out["tied"] = np.tile(np.array([0.5, 0.5, -0.5, -0.5], np.float32), n // 4 + 1)[:n]
    return out


def hop_boundary(n):
    """A sample that starts a hop of the formant stage: the last multiple of 256 (at most 32 hops in, the first hop of
    the second CTA) inside the signal, or its middle when it is shorter than a hop and a sample."""
    if n <= H:
        return n // 2
    return min(FM_HOPS, (n - 1) // H) * H


# ---------------------------------------------------------------- formant stage

FORMANT_LENGTHS = (1, 2, 3, 255, 256, 257, 767, 768, 769, 1023, 1024, 1025,
                   FM_HOPS * H - 1, FM_HOPS * H, FM_HOPS * H + 1, 2 * FM_HOPS * H + 1)

# (name, pitch, tempo, phi): pitch / formant corners, pitch NaN, and tempo ahead of the stage
FORMANT_RATIOS = (("p0.5_phi0.5", 0.5, None, 0.5), ("p0.5_phi2", 0.5, None, 2.0), ("p2_phi0.5", 2.0, None, 0.5),
                  ("p2_phi2", 2.0, None, 2.0), ("nan_phi0.5", None, None, 0.5), ("nan_phi2", None, None, 2.0),
                  ("t0.25_phi2", None, 0.25, 2.0), ("t4_phi0.5", None, 4.0, 0.5))


def formant_contours(n):
    """(name, ends, ratios, Q, m, d) contours over n input samples without tempo: the last piece starts at output Q,
    which lies d samples past the (clamped) centre of frame m: "at" 0, "before" 1 (frame m's centre is the last sample
    of the piece before), "after" -1.  Ratios 0.5 and 2 keep every knot exactly at its input sample."""
    cases = []
    if n >= 2:       # a last piece of one sample: it holds the centre of the frames clamped to n2 - 1, and nothing else
        cases.append(("last_clamped", [n - 1, n], [0.5, 2.0], n - 1, -(-n // H) - 1, 0))
    for m in (1, FM_HOPS):
        c = m * H + fr.N // 2
        for name, d in (("at", 0), ("before", 1), ("after", -1)):
            q = c + d
            if 0 < q and q + 1 < n:
                cases.append((f"knot_{name}_m{m}", [q, n], [0.5, 2.0], q, m, d))
    if n > 800:      # a middle piece of 100 samples, less than a hop, holding frame 1's centre 768
        cases.append(("short_piece", [700, 800, n], [2.0, 0.5, 2.0], 800, 1, 32))
    return cases


def formant_debug(lib, x, rate, phi, pitch=None, tempo=None, ends=None, ratios=None):
    """(pre, y) of sb200_debug_formant: the signal the stage reads and its output."""
    x = np.ascontiguousarray(x, np.float32)
    cap = 4 * len(x) + 4096
    pre, y = np.zeros(cap, np.float32), np.zeros(cap, np.float32)
    n2 = C.c_int64()
    from sonata_b200 import _native as N
    err = N.sb200_error()
    e = None if ends is None else np.ascontiguousarray(ends, np.int64)
    r = None if ratios is None else np.ascontiguousarray(ratios, np.float32)
    rc = lib.sb200_debug_formant(0, f32p(x), len(x), rate, _nan(pitch), _nan(tempo), None if e is None else i64p(e),
                                 None if r is None else f32p(r), 0 if e is None else len(e), _nan(phi), f32p(pre),
                                 f32p(y), cap, C.byref(n2), C.byref(err))
    assert rc == 0, C.string_at(err.message) if err.message else rc
    return pre[:n2.value].copy(), y[:n2.value].copy()


# The job path: (frames per id, pitch, tempo, contour (one ratio per id) or None, phi, n2).  Totals of 1, 2, 3, 4, 5 and
# 33 frames of 256 samples; tempos put n2 at and around 1024 and 32 * 256.  The ids' frames are forced, so n2 does not
# depend on the voice.
FORMANT_JOB = (
    ([0, 1, 0], 1.25, None, None, 1.0, 256),
    ([1, 1], None, None, None, 0.8, 512),
    ([1, 1, 1], None, None, [1.0, 1.3, 0.7], 1.0, 768),
    ([2, 0, 2], 0.8, None, None, 1.2, 1024),
    ([4], None, 1024 / 1023, None, 1.3, 1023),
    ([3, 2], 2.0, 1280 / 1025, None, 0.5, 1025),
    ([8, 8, 8, 9], 0.5, 1.03125, None, 2.0, 8192),
    ([11, 11, 11], None, 8448 / 8191, [1.2, 0.6, 1.9], 1.1, 8191),
    ([33], None, 8448 / 8193, None, 0.7, 8193),
    ([16, 17], 1.5, None, None, 1.0, 8448),
)


def job_ends(frames):
    return 256 * np.cumsum(frames)


# ---------------------------------------------------------------- pitch / tempo

# (name, pitch, tempo)
PROSODY_CORNERS = (("p0.5_t4", 0.5, 4.0), ("p2_t0.25", 2.0, 0.25), ("t4", None, 4.0), ("t0.25", None, 0.25),
                   ("p2", 2.0, None), ("p0.5", 0.5, None))
PROSODY_N2 = (255, 256, 257, 513)


def prosody_plan(lib, rate, n, pitch, tempo):
    """(Hs, N, D, n1, n2, F) from the library's plan hook."""
    shape = np.zeros(6, np.int64)
    assert lib.sb200_debug_prosody_plan(rate, n, _nan(pitch), _nan(tempo), i64p(shape), None, 0) == 0
    return tuple(int(v) for v in shape)


def n_for_n2(rate, pitch, tempo, target):
    """The smallest n whose n2 (prosody_reference.plan) is at least `target`: the target itself where the ratios reach
    it, else the next length they give (n2 is even at p = 0.5 and a multiple of 4 at t = 0.25 with p = 1 or 2)."""
    n = 1
    while pr.plan(rate, n, pitch, tempo)["n2"] < target:
        n += 1
    return n


def prosody_lengths(rate, pitch, tempo):
    """(name, n): 1, 2, Hs - 1 .. Hs + 1, N - 1 .. N + 1 and the n for each n2 in PROSODY_N2."""
    Hs = rate // 100
    out = [("1", 1), ("2", 2), ("Hs-1", Hs - 1), ("Hs", Hs), ("Hs+1", Hs + 1), ("N-1", 2 * Hs - 1), ("N", 2 * Hs),
           ("N+1", 2 * Hs + 1)]
    out += [(f"n2>={t}", n_for_n2(rate, pitch, tempo, t)) for t in PROSODY_N2]
    return out


def prosody_contours(n, rate):
    """(name, ends, ratios) contours over n >= 3 samples: a one-sample piece, a knot at sample 1, a knot at n - 1, and
    every piece shorter than Hs."""
    Hs = rate // 100
    cases = [("one_sample", [n // 2, n // 2 + 1, n], [2.0, 0.5, 2.0]),
             ("knot_1", [1, n], [0.5, 2.0]),
             ("knot_n-1", [n - 1, n], [2.0, 0.5])]
    step = max(1, Hs // 3)
    ends = list(range(step, n, step)) + [n]
    cases.append(("all_short", ends, [(0.5, 2.0, 0.7, 1.6)[i % 4] for i in range(len(ends))]))
    return cases


def contour_plan(lib, rate, n, ends, ratios, tempo):
    """((Hs, N, D, n1, n2, F), bounds) from the library's contour plan hook."""
    shape = np.zeros(6, np.int64)
    e = np.ascontiguousarray(ends, np.int64)
    r = np.ascontiguousarray(ratios, np.float32)
    bounds = np.zeros(len(e), np.int64)
    assert lib.sb200_debug_prosody_contour_plan(rate, n, i64p(e), f32p(r), len(e), _nan(tempo), i64p(shape), None, 0,
                                                i64p(bounds)) == 0
    return tuple(int(v) for v in shape), bounds


# ---------------------------------------------------------------- resampler

RS_PAIRS = tuple((i, o) for i in RATES for o in rr.TARGETS if o != i)
RS_N_OUT = (1023, 1024, 1025, 2049)


def taps_per_phase(in_rate, out_rate):
    """K, the taps per phase of resample_reference's filter: ceil((2 H + 1) / up), H = 10 max(up, down)."""
    up, down = rr.ratio(in_rate, out_rate)
    return -(-len(rr.taps64(up, down)) // up)


def n_for_n_out(up, down, target):
    """The smallest n whose n_out is at least `target` (the target itself when down >= up)."""
    n = max(1, (target * down) // up)
    while rr.n_out(n, up, down) < target:
        n += 1
    while n > 1 and rr.n_out(n - 1, up, down) >= target:
        n -= 1
    return n


def resample_lengths(in_rate, out_rate):
    """(name, n): 1, 2, K - 1, K, K + 1 and the n for each n_out in RS_N_OUT."""
    up, down = rr.ratio(in_rate, out_rate)
    K = taps_per_phase(in_rate, out_rate)
    out = [("1", 1), ("2", 2), ("K-1", K - 1), ("K", K), ("K+1", K + 1)]
    return out + [(f"n_out>={t}", n_for_n_out(up, down, t)) for t in RS_N_OUT]


def resample_signals(n, seed=0):
    s = signals(n, 22050, seed)
    return {k: s[k] for k in ("impulse_first", "impulse_last", "silence", "dc", "square", "noise")}


def resample_filter(lib, in_rate, out_rate):
    """(up, down, f32 taps) from the library's filter hook."""
    up, down = C.c_int32(), C.c_int32()
    assert lib.sb200_debug_resample_filter(in_rate, out_rate, None, 0, C.byref(up), C.byref(down)) == 0
    taps = np.zeros(20 * max(up.value, down.value) + 1, np.float32)
    assert lib.sb200_debug_resample_filter(in_rate, out_rate, f32p(taps), taps.size, C.byref(up), C.byref(down)) == 0
    return up.value, down.value, taps


def resample_emit(lib, in_rate, out_rate, lens):
    lens = np.ascontiguousarray(lens, np.int64)
    out = np.zeros(len(lens), np.int64)
    assert lib.sb200_debug_resample_emit(in_rate, out_rate, i64p(lens), len(lens), i64p(out)) == 0
    return out


# ---------------------------------------------------------------- loudness

def loudness_lengths(rate):
    """(name, n): 255, 256 and 257 chunks of S (the last with one sample of a 258th chunk) and about 70 s, more
    chunks and blocks than the kernel has threads."""
    S = lr.step(rate)
    return (("255S", 255 * S), ("256S", 256 * S), ("257S+1", 257 * S + 1), ("70s", 70 * rate + 3))


def block_loudness(x, rate):
    with np.errstate(divide="ignore"):
        return -0.691 + 10.0 * np.log10(lr.block_energies(x, rate))


def relative_gate(x, rate):
    """The relative gate of lr.integrated: -0.691 + 10 log10(mean z over the blocks above -70) - 10."""
    z = lr.block_energies(x, rate)
    l = block_loudness(x, rate)
    return -0.691 + 10.0 * math.log10(np.mean(z[l > -70.0])) - 10.0


def _sine(rate, n, peak, start=0, freq=997.0):
    return peak * np.sin(2 * np.pi * freq * (start + np.arange(n)) / rate)


def level_step(rate, n, margin=0.01):
    """A 997 Hz sine at 0.5 for the first 40 %, then two quiet stretches whose steady blocks lie `margin` LU above and
    `margin` LU below the relative gate of the whole signal (amplitudes found by a fixed-point iteration on the
    float64 specification)."""
    n0 = int(0.4 * n)
    n1 = (n - n0) // 2
    n2 = n - n0 - n1
    a_hi = a_lo = 0.5 * 10 ** (-0.5)      # about -10 LU below the loud part
    for _ in range(6):
        x = np.concatenate([_sine(rate, n0, 0.5), _sine(rate, n1, a_hi, n0), _sine(rate, n2, a_lo, n0 + n1)])
        x = x.astype(np.float32)
        g = relative_gate(x, rate)
        l = block_loudness(x, rate)
        hi, lo = steady_blocks(rate, n, "hi"), steady_blocks(rate, n, "lo")
        a_hi *= 10 ** ((g + margin - float(np.mean(l[hi]))) / 20)
        a_lo *= 10 ** ((g - margin - float(np.mean(l[lo]))) / 20)
    return x


def steady_blocks(rate, n, part):
    """Indices of the blocks lying wholly inside the "hi" or "lo" stretch of level_step (past a 20 ms settling)."""
    S = lr.step(rate)
    n0 = int(0.4 * n)
    n1 = (n - n0) // 2
    lo_s, hi_s = (n0, n0 + n1) if part == "hi" else (n0 + n1, n)
    lo_s += rate // 50
    nb = (n - 4 * S) // S + 1
    j = np.arange(nb)
    return j[(j * S >= lo_s) & (j * S + 4 * S <= hi_s)]


def at_absolute_gate(rate, n):
    """A 997 Hz sine whose blocks all lie within 0.01 LU of -70 LUFS (its level set from the specification's mean
    block loudness): some blocks pass the absolute gate and some do not."""
    x = _sine(rate, n, 1.0)
    l = block_loudness(x.astype(np.float32), rate)
    x = x * 10 ** ((-70.0 - float(np.mean(l))) / 20)
    return x.astype(np.float32)
