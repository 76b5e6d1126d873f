"""CPU: the emission rule of streams with a formant ratio (formant_stream_reference) against the library's no-device
plan hook, for ratio, contour, tempo and formant-only streams at both rates; the creator's refusals; and the Python
layer's argument checks, with models that are not this library's streaming voices still refusing by name."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import formant_stream_reference as fsr
import prosody_stream_reference as psr
from test_prosody_contour_stream_host import _ends, contours
from sonata_b200 import OperationError, cli, piper
from sonata_b200 import _native as N
from sonata_b200.piper import StreamBatch, VitsStreamingModel, _stream_formant
from sonata_b200.synth import RealtimeBatch, SonataSpeechSynthesizer, _stream_prosody_extra

NAN = float("nan")
RATES = (16000, 22050)
p64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))


def _message(err):
    return C.string_at(err.message).decode() if err.message else ""


def lib_plan(rate, pitch, tempo, phi, lens, ends=None, ratios=None):
    """(rc, message, per-chunk counts) of sb200_debug_formant_stream_plan."""
    lens = np.ascontiguousarray(lens, np.int64)
    out = np.zeros(len(lens), np.int64)
    e = None if ends is None else np.ascontiguousarray(ends, np.int64)
    r = None if ratios is None else np.ascontiguousarray(ratios, np.float32)
    err = N.sb200_error()
    rc = N.lib().sb200_debug_formant_stream_plan(
        rate, NAN if pitch is None else pitch, NAN if tempo is None else tempo, None if e is None else p64(e),
        None if r is None else r.ctypes.data_as(C.POINTER(C.c_float)), 0 if e is None else len(e),
        NAN if phi is None else phi, p64(lens), len(lens), p64(out), C.byref(err))
    return rc, _message(err), out


def _check(rate, pitch, tempo, phi, n, ends=None, ratios=None, extra=()):
    chunkings = dict(psr.chunkings(n, rate))
    chunkings.update(extra)
    for name, lens in chunkings.items():
        rc, msg, got = lib_plan(rate, pitch, tempo, phi, lens, ends, ratios)
        assert rc == 0, (name, msg)
        ref = fsr.stream(rate, pitch, tempo, phi, lens, ends, ratios)
        np.testing.assert_array_equal(got, [r["emitted"] for r in ref], err_msg=name)
    return ref


# (pitch, tempo, phi): phi alone, on a pitch, on a tempo, on both, and phi equal to the pitch (no stage)
RATIO_CASES = [(None, None, 1.2), (None, None, 0.5), (1.25, None, 1.0), (0.8, 2.0, 1.0), (None, 1.5, 1.0),
               (None, 0.25, 2.0), (1.25, None, 1.25), (2.0, 0.5, 0.9)]


@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("pitch,tempo,phi", RATIO_CASES)
def test_ratio_streams_follow_the_rule(lib_built, rate, pitch, tempo, phi):
    n = int(0.8 * rate)
    ref = _check(rate, pitch, tempo, phi, n, extra={"single": [1] * 3000, "short": [100] * 40})
    if (pitch or 1.0) == phi:
        # phi equal to the pitch ratio asks nothing: the ratio stream's own counts
        for lens in psr.chunkings(n, rate).values():
            want = [r["emitted"] for r in psr.stream(rate, pitch, tempo, lens)]
            np.testing.assert_array_equal(lib_plan(rate, pitch, tempo, phi, lens)[2], want)


@pytest.mark.parametrize("n", [1, 255, 300, 767, 768, 1023, 1024, 1025, 5000])
def test_short_and_unaligned_signals(lib_built, n):
    """n2 < N, n2 not a multiple of H, and chunks that emit nothing; the total is always n2."""
    for lens in ([n], [1] * n, [n // 3, n - n // 3], [0, n, 0]):
        for pitch, phi in ((None, 1.3), (1.5, 1.0)):
            rc, msg, got = lib_plan(22050, pitch, None, phi, lens)
            assert rc == 0, msg
            ref = fsr.stream(22050, pitch, None, phi, lens)
            np.testing.assert_array_equal(got, [r["emitted"] for r in ref])
            if pitch is None:
                assert int(got.sum()) == n


def test_rule_holds_back_768_to_1023_and_carries_under_1792():
    rng = np.random.default_rng(3)
    lens = list(rng.integers(0, 3000, 200)) + [17]
    rows = fsr.rule(lens)
    for r in rows[:-1]:
        if r["inputs"] >= fsr.N - fsr.H:
            assert 768 <= r["inputs"] - sum(x["emitted"] for x in rows[:rows.index(r) + 1]) <= 1023
        assert r["held"] < fsr.N + 3 * fsr.H
    assert sum(r["emitted"] for r in rows) == sum(lens)
    lo, hi = fsr.hold_back_ms(22050)
    assert round(lo) == 35 and round(hi) == 46
    lo, hi = fsr.hold_back_ms(16000)
    assert round(lo) == 48 and round(hi) == 64


@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("tempo", [None, 0.8])
@pytest.mark.parametrize("name", ["uniform", "question", "alternating", "zero_frames"])
def test_contour_streams_follow_the_rule(lib_built, rate, tempo, name):
    frames, ratios = contours()[name]
    n, ends = _ends(frames)
    for phi in (1.0, 1.2):
        _check(rate, None, tempo, phi, n, ends, ratios)


def test_neutral_contour_with_phi_is_formant_only(lib_built):
    frames = np.full(20, 7)
    n, ends = _ends(frames)
    lens = [1000] * (n // 1000) + [n % 1000]
    rc, msg, got = lib_plan(22050, None, None, 1.2, lens, ends, [1.0] * 20)
    assert rc == 0, msg
    np.testing.assert_array_equal(got, [r["emitted"] for r in fsr.rule(lens)])
    # and a contour of one ratio 1.25 with phi 1.25 asks nothing of the stage
    rc, _, got = lib_plan(22050, None, None, 1.25, lens, ends, [1.25] * 20)
    np.testing.assert_array_equal(got, [r["emitted"] for r in psr.stream(22050, 1.25, None, lens)])


def test_creator_refusals(lib_built):
    lens = [5000]
    rc, msg, _ = lib_plan(22050, None, None, 2.5, lens)
    assert rc == 19 and "formant ratio 2.5" in msg
    rc, msg, _ = lib_plan(22050, None, None, float("inf"), lens)
    assert rc == 19 and "formant ratio" in msg
    # ratios and a phi that ask for nothing
    for pitch, phi in ((None, None), (None, 1.0), (1.0, 1.0)):
        rc, msg, _ = lib_plan(22050, pitch, None, phi, lens)
        assert rc == 19 and "asks for" in msg, (pitch, phi)
    assert lib_plan(22050, 1.25, None, 1.25, lens)[0] == 0          # the ratio stream, without the stage
    rc, msg, _ = lib_plan(22050, 3.0, None, 1.0, lens)
    assert rc == 19 and "pitch ratio 3" in msg
    rc, msg, _ = lib_plan(22050, None, 9.0, 1.0, lens)
    assert rc == 19 and "tempo ratio 9" in msg
    # a contour beside a pitch ratio, a bad contour ratio, and chunks past a contour's n
    frames = np.full(10, 4)
    n, ends = _ends(frames)
    rc, msg, _ = lib_plan(22050, 1.25, None, 1.0, [n], ends, [1.1] * 10)
    assert rc == 19 and "a pitch contour and a pitch ratio" in msg
    bad = [1.1] * 10
    bad[3] = 2.5
    rc, msg, _ = lib_plan(22050, None, None, 1.0, [n], ends, bad)
    assert rc == 19 and "id 3" in msg
    rc, msg, _ = lib_plan(22050, None, None, 1.0, [n, -1], ends, [1.1] * 10)
    assert rc == 19 and "negative length" in msg
    rc, msg, _ = lib_plan(5000000, None, None, 1.2, lens)
    assert rc == 19


def test_python_checks_name_the_stream():
    assert _stream_formant(None, "stream 3") is None
    assert _stream_formant(NAN, "stream 3") is None
    assert _stream_formant(1, "stream 3") == 1.0
    with pytest.raises(OperationError, match=r"stream 3: formant ratio 2.5 is not a finite value in \[0.5, 2.0\]"):
        _stream_formant(2.5, "stream 3")
    with pytest.raises(OperationError, match="stream 3: formant ratio 'x' is not a number"):
        _stream_formant("x", "stream 3")
    with pytest.raises(OperationError, match="stream 0: formant ratio True is not a number"):
        _stream_formant(True, "stream 0")


class _Streaming(VitsStreamingModel):
    """A streaming voice without a device: records what reaches the stream's creation."""

    def __init__(self):
        self.calls = []

    def get_speakers(self):
        return {}

    def phonemes_to_input_ids(self, phonemes):
        return [1, 2, 3]

    def audio_output_info(self):
        return type("Info", (), {"sample_rate": 22050})()

    def stream_synthesis(self, phonemes, chunk_size, chunk_padding, **kw):
        self.calls.append(kw)
        return iter([])

    def __del__(self):
        pass


def test_stream_batch_checks_each_stream_option(monkeypatch):
    m = _Streaming()
    sb = StreamBatch(m, 40, 3)
    sb.add([1, 2, 3])
    sb.add([1, 2, 3], formant_ratio=1.2)
    with pytest.raises(OperationError, match="stream 2: formant ratio 0.1"):
        sb.add([1, 2, 3], formant_ratio=0.1)
    with pytest.raises(OperationError, match="stream 2: formant ratio 'a' is not a number"):
        sb.add([1, 2, 3], formant_ratio="a")
    k = sb.add([1, 2, 3], formant_ratio=NAN, pitch=1.25)
    assert [o.formant for o in sb._pending] == [None, 1.2, None]
    assert sb._pending[-1].key == k == 2


def test_stream_prosody_decides_what_asks(monkeypatch):
    made = []

    class _Stream:
        def __init__(self, model, pitch=None, tempo=None, pitch_contour=None, enc=None, formant=None):
            made.append((pitch, tempo, pitch_contour, formant))
    monkeypatch.setattr(piper, "ProsodyStream", _Stream)
    m = object()
    assert piper._stream_prosody(m, None, None) is None
    assert piper._stream_prosody(m, None, None, formant=1.0) is None          # r_m = 1: no stage, the plain stream
    assert piper._stream_prosody(m, 1.25, None, formant=1.25) is not None
    assert made[-1] == (1.25, None, None, None)                               # phi equal to the pitch: dropped
    piper._stream_prosody(m, None, None, formant=1.2)
    assert made[-1] == (None, None, None, 1.2)                                # formant only
    piper._stream_prosody(m, 0.8, 1.5, formant=1.0)
    assert made[-1] == (0.8, 1.5, None, 1.0)

    class _Enc:
        p_duration = np.ones(3, np.int32)
    piper._stream_prosody(m, None, None, [1.2, 1.0, 1.3], _Enc(), formant=1.0)
    assert made[-1] == (None, None, [1.2, 1.0, 1.3], 1.0)                     # a contour stream with phi
    piper._stream_prosody(m, None, None, [1.0, None, 1.0], _Enc(), formant=1.2)
    assert made[-1] == (None, None, None, 1.2)                                # a neutral contour: formant only
    with pytest.raises(OperationError, match="stream: formant ratio 4.0"):
        piper._stream_prosody(m, None, None, formant=4.0)


def test_streaming_voices_pass_the_ratio_and_others_refuse():
    m = _Streaming()
    assert _stream_prosody_extra(m, None, None, "x", 1.2) == {"formant_ratio": 1.2}
    assert _stream_prosody_extra(m, 1.25, None, "x", NAN) == {"pitch": 1.25}
    with pytest.raises(OperationError, match="request: formant ratio 3.0"):
        _stream_prosody_extra(m, None, None, "x", 3.0)

    class _Other:
        pass
    with pytest.raises(OperationError, match="RealtimeBatch cannot apply a formant ratio"):
        _stream_prosody_extra(_Other(), None, None, "RealtimeBatch", 1.2)
    assert _stream_prosody_extra(_Other(), None, None, "x", None) == {}


def test_cli_realtime_mode_reaches_a_streaming_voice(monkeypatch):
    seen = {}

    def streamed(self, text, oc, chunk_size, chunk_padding, **kw):
        seen.update(kw)
        return iter([])
    monkeypatch.setattr(SonataSpeechSynthesizer, "synthesize_streamed", streamed)
    m = _Streaming()
    m.set_fallback_synthesis_config = lambda cfg: None
    cli.process_request(SonataSpeechSynthesizer(m), piper.PiperSynthesisConfig(None, 0.667, 1.0, 0.8),
                        {"text": "a", "mode": "realtime", "formant_ratio": 1.1}, None)
    assert seen["formant_ratio"] == 1.1
    with pytest.raises(OperationError, match="utterance 0: formant ratio 5.0"):
        cli.process_request(SonataSpeechSynthesizer(m), None, {"text": "a", "mode": "realtime", "formant_ratio": 5.0},
                            None)


def test_realtime_batch_checks_the_ratio_at_add():
    rb = RealtimeBatch(_Streaming())
    with pytest.raises(OperationError, match="request: formant ratio 0.2"):
        rb.add("a", formant_ratio=0.2)
