"""Case tables and a float64 reference that scales, for the edge tests of the live loudness meter
(include/sonata_b200.h, sb200_loudness_stream_create): the stream lengths whose readings gate more blocks than the
kernel has threads, the chunkings that complete more steps in one launch than it has threads or carry S - 1 samples
every time, the totals either side of the meter's capacity, and the long decoder streams.  Used by
tests/test_loudness_stream_edges_host.py (the tables and the reference) and tests/test_loudness_stream_edges_gpu.py
(the kernel against them)."""
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import loudness_reference as lr
import loudness_stream_reference as lsr
from test_loudness_stream_host import _speechlike

LD_THREADS = 256              # threads of loudness_stream_kernel's one block per chunk
LS_MAX_STEPS = 1 << 16        # steps of 100 ms a meter keeps q of (engine.h)

# ---------------------------------------------------------------- the float64 reference at any length


def readings_at(q, S, ms):
    """L_m at the boundaries ms from the step energies q (lsr._energies): lsr.readings' values, gating only the blocks of
    the requested m.  m <= 3 is the provisional mean square, summed left to right over at most three steps."""
    q = np.asarray(q, np.float64)
    z = (q[:-3] + q[1:-2] + q[2:-1] + q[3:]) / (4 * S) if len(q) >= 4 else np.zeros(0)
    out = np.empty(len(ms), np.float64)
    for k, m in enumerate(ms):
        if m >= 4:
            out[k] = lsr._gated(z[:m - 3])
        else:
            s = 0.0
            for c in range(m):
                s += q[c]
            L = -0.691 + 10.0 * math.log10(s / (m * S)) if s > 0.0 else -math.inf
            out[k] = -math.inf if L <= -70.0 else L
    return out


# ---------------------------------------------------------------- long streams

# (rate, complete steps, samples past the last boundary).  Readings gate m - 3 blocks for m = 4 .. steps, so every
# stream reaches 255 .. 257 and 511 .. 513 blocks, one or two per thread of ld_gates; the 8000 Hz stream passes 1000
# steps, the 22050 Hz one (S odd) ends with S - 1 samples in the carry and both end on 513 blocks.
LONG_CASES = ((8000, 1030, 399), (22050, 516, 2204), (48000, 516, 17))
EDGE_BLOCKS = (255, 256, 257, 511, 512, 513)


def long_signal(rate, steps, tail, seed):
    """Speech-like level changes over steps * S + tail samples, a 2 s silent gap and a burst the gain drives into the
    clamp."""
    n = steps * lr.step(rate) + tail
    x = _speechlike(rate, (n + 1) / rate, seed)[:n]
    assert len(x) == n
    x[int(0.3 * n):int(0.3 * n) + 2 * rate] = 0.0
    x[int(0.7 * n):int(0.7 * n) + rate // 10] *= 6.0
    return x


def long_chunkings(n, rate, seed):
    """name -> chunk lengths over n samples: one chunk; 1 s chunks; S - 1 samples, then whole steps, so every chunk
    but the last leaves S - 1 samples in the carry; a random mix with 1-sample chunks."""
    S = lr.step(rate)
    out = {"one": [n], "second": [rate] * (n // rate) + ([n % rate] if n % rate else [])}
    carry, k = [S - 1], 0
    while sum(carry) + (S, 3 * S, 10 * S)[k % 3] <= n:
        carry.append((S, 3 * S, 10 * S)[k % 3])
        k += 1
    if sum(carry) < n:
        carry.append(n - sum(carry))
    out["carry"] = carry
    rng = np.random.default_rng(seed)
    mixed = []
    while sum(mixed) < n:
        mixed.append(int(rng.choice([1, 1, 2, 7, S - 1, S + 1, 3 * S + 5, 10 * S, 30 * S])))
    mixed[-1] -= sum(mixed) - n
    out["mixed"] = [c for c in mixed if c > 0]
    return out


def carries(lens, S):
    """The samples each chunk leaves in the carry (past the last step boundary)."""
    return [int(c) % S for c in np.cumsum(lens)]


def steps_completed(lens, S):
    """The steps each chunk completes: the launch's nc."""
    b = np.concatenate([[0], np.cumsum(lens) // S])
    return np.diff(b).tolist()


def check_ms(M):
    """The boundaries at which a stream of M steps is compared with the batch meter bit for bit: m = 4, every m whose
    block count is within two of 256 or 512, 20 spread m and the last."""
    around = [b + 3 + d for b in (256, 512) for d in (-2, -1, 0, 1, 2)]
    spread = np.linspace(4, M, 20).round().astype(int).tolist()
    return sorted({m for m in [4] + around + spread + [M] if 4 <= m <= M})


# ---------------------------------------------------------------- capacity

CAP_RATE = 8000
CAP_S = lr.step(CAP_RATE)
CAP_ACCEPTED = LS_MAX_STEPS * CAP_S + CAP_S - 1      # 2^16 steps and an incomplete one in the carry
CAP_REFUSED = LS_MAX_STEPS * CAP_S + CAP_S           # one step past capacity


def cap_ms():
    """The boundaries of the full meter compared with float64: the provisional ones, both block edges, 20 spread and
    the last few, where q's last entries are written and read."""
    spread = np.linspace(4, LS_MAX_STEPS, 20).round().astype(int).tolist()
    return sorted({1, 2, 3, 4, 5, 258, 259, 260, 514, 515, 516, 1 << 15, LS_MAX_STEPS - 2, LS_MAX_STEPS - 1,
                   LS_MAX_STEPS} | set(spread))


# ---------------------------------------------------------------- the decoder at long length (the medium voice)

VOICE_RATE = 22050
HOP = 256
FRAMES_PER_ID = 5
REQUEST_PHONEMES = (70, 70, 70, 70)   # four sentences of 2 * 70 + 2 ids, FRAMES_PER_ID frames each
REQUEST_CHUNK = (55, 3)               # chunk size and padding, in frames
LONG_PHONEMES = 280                   # one utterance of 562 ids
LONG_CHUNK = (1500, 3)                # one-shot: frames <= 2 (chunk size + padding)
OUT_RATES = (8000, 48000)


def frames(n_phonemes):
    return (2 * n_phonemes + 2) * FRAMES_PER_ID


def delivered(n_frames, rate):
    """The samples n_frames decode to, delivered at `rate` (resampling rounds up)."""
    return -(-(n_frames * HOP * rate) // VOICE_RATE)
