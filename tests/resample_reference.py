"""Float64 restatement of the output-rate resampler (scipy.signal.resample_poly's default), for the resampling tests."""
from fractions import Fraction

import numpy as np

VOICE_RATES = (16000, 22050)
TARGETS = (8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000)


def ratio(in_rate, out_rate):
    f = Fraction(out_rate, in_rate)
    return f.numerator, f.denominator


def taps64(up, down):
    """resample_poly's filter in float64: firwin(2H + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up."""
    from scipy.signal import firwin
    m = max(up, down)
    return firwin(2 * 10 * m + 1, 1.0 / m, window=("kaiser", 5.0)) * up


def n_out(n, up, down):
    return -((-n * up) // down)


def bound(x, up, down):
    """Per output j: (terms_j + 2) * 2^-24 * sum_i |h * x| over the terms of output j, with terms_j their number."""
    from scipy.signal import resample_poly
    h = np.abs(taps64(up, down))
    ax = np.abs(np.asarray(x, np.float64))
    mag = resample_poly(ax, up, down, window=h / up)                 # resample_poly multiplies given taps by up
    terms = np.rint(resample_poly(np.ones_like(ax), up, down, window=np.ones_like(h) / up))
    return (terms + 2) * 2.0 ** -24 * mag


def resample64(x, up, down):
    from scipy.signal import resample_poly
    return resample_poly(np.asarray(x, np.float64), up, down)
