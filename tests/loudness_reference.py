"""Float64 restatement of the library's loudness measurement and gain (ITU-R BS.1770-4, one channel, libebur128's
any-rate K-weighting design), for the loudness tests."""
import math

import numpy as np

RATES = (8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000)

# BS.1770-4 Tables 1 and 2 (48 kHz): shelf b0, b1, b2, a1, a2 and high-pass b0, b1, b2, a1, a2
TABLE_48K = (1.53512485958697, -2.69169618940638, 1.19839281085285, -1.69065929318241, 0.73248077421585,
             1.0, -2.0, 1.0, -1.99004745483398, 0.99007225036621)


def design(rate):
    """The cascade at `rate`: ((b, a) of the shelf, (b, a) of the high-pass), float64, a[0] = 1."""
    f0, G, Q = 1681.974450955533, 3.999843853973347, 0.7071752369554196
    K = math.tan(math.pi * f0 / rate)
    Vh = 10.0 ** (G / 20.0)
    Vb = Vh ** 0.4996667741545416
    a0 = 1.0 + K / Q + K * K
    shelf = ([(Vh + Vb * K / Q + K * K) / a0, 2.0 * (K * K - Vh) / a0, (Vh - Vb * K / Q + K * K) / a0],
             [1.0, 2.0 * (K * K - 1.0) / a0, (1.0 - K / Q + K * K) / a0])
    f0, Q = 38.13547087602444, 0.5003270373238773
    K = math.tan(math.pi * f0 / rate)
    a0 = 1.0 + K / Q + K * K
    hp = ([1.0, -2.0, 1.0], [1.0, 2.0 * (K * K - 1.0) / a0, (1.0 - K / Q + K * K) / a0])
    return shelf, hp


def coeffs(rate):
    """design(rate) flattened as the library's debug hook returns it."""
    (bs, as_), (bh, ah) = design(rate)
    return np.array(bs + as_[1:] + bh + ah[1:], np.float64)


def step(rate):
    return (rate + 5) // 10


def block_energies(x, rate):
    """z_j, the mean square of the K-weighted signal over block j = samples [jS, jS + 4S)."""
    from scipy.signal import lfilter
    (bs, as_), (bh, ah) = design(rate)
    y = lfilter(bh, ah, lfilter(bs, as_, np.asarray(x, np.float64)))
    S = step(rate)
    n = len(y)
    if n < 4 * S:
        return np.zeros(0)
    nb = (n - 4 * S) // S + 1
    q = np.array([np.sum(y[c * S:(c + 1) * S] ** 2) for c in range(nb + 3)])
    return (q[:nb] + q[1:nb + 1] + q[2:nb + 2] + q[3:nb + 3]) / (4 * S)


def integrated(x, rate):
    """Integrated loudness in LUFS, -inf when no block passes the gates."""
    z = block_energies(x, rate)
    with np.errstate(divide="ignore"):
        l = -0.691 + 10.0 * np.log10(z)
    keep = l > -70.0
    if not keep.any():
        return -math.inf
    rel = -0.691 + 10.0 * math.log10(np.mean(z[keep])) - 10.0
    keep &= l > rel
    if not keep.any():
        return -math.inf
    return -0.691 + 10.0 * math.log10(np.mean(z[keep]))


def gain(x, target, lufs):
    """g = min(10^((T - L)/20), 1/peak) in float64, rounded to f32 (1 when L = -inf or peak = 0)."""
    peak = float(np.max(np.abs(np.asarray(x, np.float32)))) if len(x) else 0.0
    if lufs == -math.inf or peak == 0.0:
        return np.float32(1.0)
    return np.float32(min(10.0 ** ((target - lufs) / 20.0), 1.0 / peak))


def sine(rate, seconds, freq=997.0, peak=0.1):
    n = int(round(rate * seconds))
    return (peak * np.sin(2 * np.pi * freq * np.arange(n) / rate)).astype(np.float32)
