"""Host tests of the watermark (include/sonata_b200.h, sb200_voice_set_watermark and sb200_watermark_detect): the numpy
specification against a literal per-sample reading of the header at every output rate, the Python and library checks
and their messages, and the detector in numpy on marked and unmarked synthetic signals."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import watermark_reference as wr
from noise_reference import philox4x32_10
from sonata_b200 import _native as N
from sonata_b200.core import OperationError, check_watermark

RATES = (8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000)
KEY = 0xC0FFEE_12345678


def literal(x, rate, key, payload, strength_db):
    """The header read one sample at a time."""
    x = [np.float32(v) for v in x]
    P, B = 4096, rate // 100

    def chip(j, m):
        w = philox4x32_10(np.array([m, j, 0, 0], np.uint32), np.array([key & 0xFFFFFFFF, key >> 32], np.uint32))
        return 1 if int(w[0]) & 1 else -1

    def q(v):
        return int(np.float32(min(max(v, np.float32(-1)), np.float32(1))) * np.float32(32767))

    n = len(x)
    K = -(-n // B)
    S = [sum(q(x[i]) ** 2 for i in range(k * B, min(k * B + B, n))) for k in range(K)]
    L = [min(B, n - k * B) for k in range(K)]
    alpha = 10.0 ** (float(np.float32(strength_db)) / 20.0)
    c0 = {m: chip(0, m) for m in range(P)} if n else {}
    c1 = {m: chip(1, m) for m in range(P)} if n else {}
    y = []
    for i in range(n):
        k = i // B
        kp = max(k - 1, 0)
        E = min(S[kp] / L[kp], S[k] / L[k])
        a = np.float32((alpha * math.sqrt(E * 0.5)) / 32767.0)
        c = c0[i % P] + c1[(i - payload) % P]
        y.append(np.float32(x[i] + np.float32(a * np.float32(c))))
    return np.array(y, np.float32)


@pytest.mark.parametrize("rate", RATES)
def test_spec_equals_the_literal_reading(rate):
    rng = np.random.default_rng(rate)
    B = rate // 100
    c = wr.chips(KEY)
    for n in (1, B - 1, B, B + 1, 3 * B + 7):
        x = (0.4 * rng.standard_normal(n)).astype(np.float32)
        x[::5] = 1.75                                 # beyond full scale: quantised at the clamp, never clamped
        x[1::7] = -3.0
        if n > B:
            x[:B] = 0.0                               # a silent block
        for payload, db in ((0, -40.0), (4095, -10.0), (77, -26.0)):
            want = literal(x, rate, KEY, payload, db)
            got = wr.embed(x, rate, KEY, payload, db, c)
            assert got.tobytes() == want.tobytes(), (n, payload, db)


def test_silence_gets_no_mark_and_the_mark_follows_the_envelope():
    rate, c = 16000, wr.chips(KEY)
    x = np.zeros(16000, np.float32)
    assert wr.embed(x, rate, KEY, 5, -10.0, c).tobytes() == x.tobytes()
    rng = np.random.default_rng(1)
    x[4000:8000] = (0.3 * rng.standard_normal(4000)).astype(np.float32)
    y = wr.embed(x, rate, KEY, 5, -20.0, c)
    d = (y - x).astype(np.float64)
    B = rate // 100
    assert not d[:4000].any() and not d[8000 + B:].any()      # before speech and 10 ms after it
    power = np.mean(d[4000 + B:8000] ** 2) / np.mean(x[4000 + B:8000].astype(np.float64) ** 2)
    assert abs(10 * math.log10(power) + 20.0) < 0.5


def test_chips_are_balanced_and_keyed():
    a, b = wr.chips(1), wr.chips(2)
    assert set(np.unique(a)) == {-1, 1} and abs(a.sum()) < 400
    assert (a != b).mean() > 0.4


def test_python_checks_and_messages():
    assert check_watermark(5, 0, -26) == (5, 0, -26.0)
    for args, msg in [((-1, 0, -26.0), "watermark: key -1 is not an integer in [0, 2^64)"),
                      ((1 << 64, 0, -26.0), "is not an integer in [0, 2^64)"),
                      ((1.5, 0, -26.0), "watermark: key 1.5 is not"),
                      ((1, 4096, -26.0), "watermark: payload 4096 is not in [0, 4096)"),
                      ((1, -1, -26.0), "watermark: payload -1 is not in [0, 4096)"),
                      ((1, True, -26.0), "watermark: payload True is not"),
                      ((1, 0, -9.0), "watermark: strength_db -9 is not a finite value in [-40, -10] dB"),
                      ((1, 0, -41.0), "watermark: strength_db -41 is not a finite value in [-40, -10] dB"),
                      ((1, 0, float("nan")), "watermark: strength_db nan is not a finite value"),
                      ((1, 0, "loud"), "watermark: strength_db 'loud' is not a finite value")]:
        with pytest.raises(OperationError) as e:
            check_watermark(*args)
        assert msg in str(e.value), (args, str(e.value))


def _c_error(fn):
    err = N.sb200_error()
    rc = fn(C.byref(err))
    return rc, C.string_at(err.message).decode() if err.message else ""


def test_library_checks_and_messages(lib_built):
    lib = N.lib()
    x = np.zeros(4, np.float32)
    p = x.ctypes.data_as(C.POINTER(C.c_float))
    for payload, db in ((4096, -26.0), (-1, -26.0), (0, -9.0), (0, -41.0), (0, float("nan")), (0, float("inf"))):
        wm = N.sb200_watermark(1, payload, db)
        rc, msg = _c_error(lambda e: lib.sb200_debug_watermark(p, 4, 16000, C.byref(wm), p, e))
        with pytest.raises(OperationError) as want:
            check_watermark(1, payload, db)
        assert rc == 19 and msg == str(want.value), (payload, db, msg)
    offs = np.array([0, 4], np.uint64)
    out = (N.sb200_watermark_result * 1)()
    rc, msg = _c_error(lambda e: lib.sb200_watermark_detect(0, 1, 2, x.ctypes.data_as(C.c_void_p),
                                                            offs.ctypes.data_as(C.POINTER(C.c_size_t)), 1, out, e))
    assert rc == 19 and msg == "watermark detect: format 2 is not 0 (f32) or 1 (i16)"


def test_header_declares_the_interface():
    h = open(os.path.join(ROOT, "include", "sonata_b200.h")).read()
    for name in ("sb200_voice_set_watermark", "sb200_voice_watermark", "sb200_watermark_detect",
                 "sb200_debug_watermark", "sb200_watermark_stream_create", "sb200_watermark_stream_free",
                 "sb200_watermark_stream_profile", "sb200_decode_chunks_marked"):
        assert name + "(" in h and name in N.SIGNATURES


# ---------------------------------------------------------------------------------------------------- detection
def _white(rng, n):
    return (0.25 * rng.standard_normal(n)).astype(np.float32)


def _harmonic(rng, n, rate):
    t = np.arange(n) / rate
    f0 = 120 + 40 * np.sin(2 * np.pi * 0.7 * t)
    ph = 2 * np.pi * np.cumsum(f0) / rate
    x = sum(np.sin(k * ph) / k for k in range(1, 12)) * (0.5 + 0.5 * np.sin(2 * np.pi * 3 * t) ** 2)
    return (0.2 * x + 0.01 * rng.standard_normal(n)).astype(np.float32)


@pytest.mark.parametrize("kind", ("white", "harmonic"))
def test_crops_are_detected_with_their_offset_and_payload(kind):
    rng, rate, c = np.random.default_rng(7), 16000, wr.chips(KEY)
    for t in range(6):
        n = 6 * rate
        x = _white(rng, n) if kind == "white" else _harmonic(rng, n, rate)
        payload = int(rng.integers(0, 4096))
        y = wr.embed(x, rate, KEY, payload, -20.0, c)
        lo = int(rng.integers(0, 2 * rate))
        clip = y[lo:lo + 3 * rate]
        d = wr.detect(clip, KEY, c)
        assert d["marked"] and d["payload"] == payload and d["offset"] == lo % 4096, (t, d)
        i16 = np.trunc(np.clip(clip, -1, 1) * 20000).astype(np.int16)        # a gain and i16: the same decision
        assert wr.detect(i16, KEY, c)["payload"] == payload
        assert not wr.detect(clip, KEY + 1)["marked"]                       # a wrong key finds nothing
        assert not wr.detect(x[lo:lo + 3 * rate], KEY, c)["marked"]          # nor does the unmarked signal


def test_unmarked_clips_are_never_detected_and_lags_are_standard():
    rng, c = np.random.default_rng(11), wr.chips(KEY)
    lags = []
    for t in range(2000):
        n = int(rng.integers(4096, 30000))
        x = _white(rng, n) if t % 2 else _harmonic(rng, n, 16000)
        d = wr.detect(x, KEY, c)
        assert not d["marked"], (t, d)
        if t < 200:
            lags.append(wr.standardised_lags(x, KEY, c))
    z = np.concatenate(lags)
    assert abs(z.mean()) < 0.01 and abs(z.std() - 1.0) < 0.01


def test_expected_strength_formula_matches_a_white_signal():
    rng, rate, c = np.random.default_rng(3), 16000, wr.chips(KEY)
    x = _white(rng, 10 * rate)
    d = wr.detect(wr.embed(x, rate, KEY, 9, -26.0, c), KEY, c)
    want = wr.expected_z(-26.0, x.size)
    assert 0.7 * want < d["z0"] < 1.3 * want, (d, want)


def test_cli_options():
    from sonata_b200 import cli
    ap = cli.build_parser()
    a = ap.parse_args(["v.json", "--watermark-key", "0xFF", "--watermark-payload", "9", "--watermark-strength-db", "-20"])
    assert (a.watermark_key, a.watermark_payload, a.watermark_strength_db) == (255, 9, -20.0)
    assert ap.parse_args(["v.json", "--watermark-key", "1234"]).watermark_key == 1234

    class Model:
        def set_watermark(self, *args):
            self.args = args
    m = Model()
    cli.set_watermark_of(m, ap.parse_args(["v.json", "--watermark-key", "7"]))
    assert m.args == (7, 0, -26.0)
    with pytest.raises(OperationError, match="need --watermark-key"):
        cli.set_watermark_of(m, ap.parse_args(["v.json", "--watermark-payload", "3"]))


@pytest.mark.parametrize("rate", (8000, 22050, 48000))
def test_stream_emission_rule_equals_the_whole_signal(rate):
    rng, c, B = np.random.default_rng(rate), wr.chips(KEY), rate // 100
    x = (0.3 * rng.standard_normal(7 * B * 13 + 5)).astype(np.float32)
    x[: 3 * B] = 0.0
    whole = wr.embed(x, rate, KEY, 99, -26.0, c)
    for cuts in ([x.size], [1, B - 1, B, B + 1, 3 * B + 7], list(rng.integers(0, 5 * B, 40)), [0, 0, 2 * B, 0, 17]):
        edges = np.cumsum([0] + [int(v) for v in cuts])
        edges = np.minimum(edges, x.size)
        chunks = [x[a:b] for a, b in zip(edges[:-1], edges[1:])] + [x[edges[-1]:]]
        got = wr.stream(chunks, rate, KEY, 99, -26.0, c)
        assert len(got) == len(chunks)
        received = np.cumsum([ch.size for ch in chunks])
        emitted = np.cumsum([g.size for g in got])
        assert all(e == (r if i == len(chunks) - 1 else r // B * B) for i, (r, e) in enumerate(zip(received, emitted)))
        assert np.concatenate(got).tobytes() == whole.tobytes(), cuts
