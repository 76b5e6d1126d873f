"""The specification of the formant stage (include/sonata_b200.h, sb200_speak_batch_ids_formants) in float64 numpy.
The kernels are held to it: each sample within `bound` of the value `apply` returns, computed from the device's own
input to the stage."""
import math

import numpy as np

N, H = 1024, 256
CLAMP = 24.0 / 20.0 * math.log(10.0)      # 24 dB as a natural-log amplitude
FORMANT_RANGE = (0.5, 2.0)


def window():
    return 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(N) / N)


def frame_ratios(n2, pitch=None, Q=None, P=None):
    """p_m of frames m = -3 .. ceil(n2 / H) - 1: the f32 pitch ratio (1 for None / NaN), or with a contour (Q, P: the
    pieces' first outputs and ratios, as prosody_contour_reference.plan gives them) the ratio of the piece holding
    each frame's clamped centre."""
    m = np.arange(-3, -(-n2 // H))
    c = np.clip(m * H + N // 2, 0, n2 - 1)
    if Q is not None and len(Q) > 1:
        r = np.searchsorted(np.asarray(Q, np.float64), c.astype(np.float64), side="right") - 1
        return m, np.asarray(P, np.float64)[r]
    p = 1.0 if pitch is None or math.isnan(float(pitch)) else float(np.float32(pitch))
    return m, np.full(len(m), p)


def asks(n2, phi, pitch=None, Q=None, P=None):
    """Whether the stage runs: phi is not None / NaN and some frame has p_m / phi != 1."""
    if phi is None or math.isnan(float(phi)) or n2 <= 0:
        return False
    _, p = frame_ratios(n2, pitch, Q, P)
    return bool(np.any(p / float(np.float32(phi)) != 1.0))


def apply(y, rate, phi, pitch=None, Q=None, P=None):
    """The stage's output in float64 (before its one rounding to f32) for the n2 samples y."""
    y = np.asarray(y, np.float64)
    n2 = len(y)
    m, p = frame_ratios(n2, pitch, Q, P)
    r = p / float(np.float32(phi))
    Q0 = rate // 250
    Qm = np.floor(Q0 / p + 0.5)
    w = window()
    idx = m[:, None] * H + np.arange(N)[None, :]
    frames = np.where((idx >= 0) & (idx < n2), y[np.clip(idx, 0, n2 - 1)], 0.0) * w
    X = np.fft.rfft(frames, axis=1)
    Pw = X.real ** 2 + X.imag ** 2
    eps = 1e-10 * Pw.mean(axis=1) + 1e-30
    lam = 0.5 * np.log(Pw + eps[:, None])
    c = np.fft.irfft(lam, n=N, axis=1)
    qq = np.minimum(np.arange(N), N - np.arange(N))[None, :]
    lift = np.where(qq == 0, 1.0, np.where(qq < Qm[:, None], 0.5 * (1 + np.cos(np.pi * qq / Qm[:, None])), 0.0))
    E = np.fft.rfft(c * lift, axis=1).real
    u = np.arange(N // 2 + 1)[None, :] * r[:, None]
    i = np.minimum(np.floor(u).astype(np.int64), N // 2 - 1)
    f = u - i
    rows = np.arange(len(m))[:, None]
    e0 = E[rows, i]
    Eh = np.where(u >= N // 2, E[:, N // 2][:, None], e0 + f * (E[rows, i + 1] - e0))
    g = np.clip(Eh - E, -CLAMP, CLAMP)
    z = np.fft.irfft(X * np.exp(g), n=N, axis=1)
    acc = np.zeros((len(m) + 3) * H + N)
    for k in range(len(m)):       # ascending m
        lo = k * H                # frame m = k - 3 starts at sample (k - 3) H: acc is offset by 3 H
        acc[lo:lo + N] += w * z[k]
    return acc[3 * H:3 * H + n2] / 1.5


def bound(ref):
    """Half an f32 ulp of the specification's value plus an absolute 1e-11."""
    return 0.5 * np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64) + 1e-11


# ---- measuring what the stage does, independently of it

def vowel(rate, seconds=1.0, f0=120.0, formants=(700.0, 1220.0, 2600.0), bandwidths=(80.0, 90.0, 120.0), peak=0.5):
    """A band-limited pulse train at f0 through two-pole resonators at `formants`, as float32."""
    from scipy.signal import lfilter
    t = np.arange(int(rate * seconds)) / rate
    x = np.zeros(len(t))
    for h in range(1, int((rate / 2) // f0) + 1):
        x += np.cos(2 * np.pi * h * f0 * t)
    for f, bw in zip(formants, bandwidths):
        rad = math.exp(-math.pi * bw / rate)
        a = [1.0, -2 * rad * math.cos(2 * math.pi * f / rate), rad * rad]
        x = lfilter([1.0 - rad], a, x)
    return (peak * x / np.max(np.abs(x))).astype(np.float32)


def lpc_formants(x, rate, order=12, count=3):
    """The `count` lowest formant frequencies of x by LPC (autocorrelation method, Levinson-Durbin) over its middle
    half: roots of the predictor above 90 Hz with bandwidths below 500 Hz.  Order 12: two poles per formant of a
    three-formant vowel and six for the source's tilt."""
    x = np.asarray(x, np.float64)
    n = len(x)
    seg = x[n // 4:3 * n // 4]
    seg = np.append(seg[0], seg[1:] - 0.63 * seg[:-1]) * np.hamming(len(seg))
    rr = np.correlate(seg, seg, "full")[len(seg) - 1:len(seg) + order]
    a = np.zeros(order + 1)
    a[0], err = 1.0, rr[0]
    for i in range(1, order + 1):
        k = -(rr[i] + np.dot(a[1:i], rr[i - 1:0:-1])) / err
        a[1:i + 1] = a[1:i + 1] + k * np.append(a[i - 1:0:-1], 1.0)
        err *= 1 - k * k
    roots = [z for z in np.roots(a) if z.imag > 0]
    f = np.array([math.atan2(z.imag, z.real) * rate / (2 * math.pi) for z in roots])
    bw = np.array([-math.log(abs(z)) * rate / math.pi for z in roots])
    keep = np.sort(f[(f > 90) & (bw < 500)])
    return keep[:count]


def f0_from_harmonics(x, rate, guess):
    """F0 within +-30 % of `guess` as the spacing that best fits the harmonic peaks of the middle half's spectrum."""
    x = np.asarray(x, np.float64)
    n = len(x)
    seg = x[n // 4:3 * n // 4] * np.hanning(n // 2)
    nfft = 1 << 18
    mag = np.log(np.abs(np.fft.rfft(seg, nfft)) + 1e-9)
    best, arg = -np.inf, guess
    for f in np.arange(0.7 * guess, 1.3 * guess, 0.02):
        ks = np.round(np.arange(1, 9) * f * nfft / rate).astype(np.int64)
        s = mag[ks].mean()
        if s > best:
            best, arg = s, f
    return arg
