"""CPU: the pitch / tempo specification against itself and against the library's no-device plan hook, argument
checks, the refusals of the streaming modes and the CLI flags."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import prosody_reference as pr
import sonata_b200
from sonata_b200 import OperationError, cli
from sonata_b200 import _native as N
from sonata_b200.piper import PhonemeAlignment, StreamBatch, _alignment, _prosody_arrays, refuse_prosody
from sonata_b200.synth import RealtimeBatch, SonataSpeechSynthesizer

RATES = (22050, 16000)                       # medium / high and low / x_low
GRID = (0.5, 0.8, 1.0, 1.25, 2.0)


def _plan(rate, n, p, t):
    shape = (C.c_int64 * 6)()
    pos = np.zeros(max(8 * n // (rate // 100) + 8, 1), np.int64)
    rc = N.lib().sb200_debug_prosody_plan(rate, n, p, t, shape, pos.ctypes.data_as(C.POINTER(C.c_int64)), pos.size)
    return rc, list(shape), pos


@pytest.mark.parametrize("rate", RATES)
def test_plan_equals_the_library(lib_built, rate):
    for n in (1, 255, rate, 3 * rate + 17):
        for p in GRID:
            for t in GRID + (0.25, 4.0):
                pl = pr.plan(rate, n, p, t)
                rc, shape, pos = _plan(rate, n, p, t)
                assert rc == 0
                assert shape == [pl["Hs"], pl["N"], pl["D"], pl["n1"], pl["n2"], pl["F"]], (n, p, t)
                np.testing.assert_array_equal(pos[:pl["F"]], pl["a"])
    pl = pr.plan(rate, rate, None, None)
    assert (pl["n1"], pl["n2"], pl["F"]) == (rate, rate, 0)
    assert _plan(rate, rate, float("nan"), float("nan"))[1][3:] == [rate, rate, 0]
    assert (pl["Hs"], pl["N"], pl["D"]) == {22050: (220, 440, 137), 16000: (160, 320, 100)}[rate]
    assert np.allclose(pr.window(pl["N"])[:pl["Hs"]] + pr.window(pl["N"])[pl["Hs"]:], 1.0)


def test_plan_refuses_bad_arguments(lib_built):
    for p, t in ((0.49, 1.0), (2.01, 1.0), (1.0, 0.2), (1.0, 4.5), (float("inf"), 1.0), (1.0, -1.0)):
        assert _plan(22050, 1000, p, t)[0] == 19
    assert _plan(500, 1000, 1.25, 1.0)[0] == 19


@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("p", [0.5, 0.8, 1.25, 2.0])
def test_pitch_moves_the_tone_and_keeps_the_length(rate, p):
    f = 300.0
    x = pr.tone(rate, f, 0.5)
    r = pr.process(x, rate, pitch=p)
    assert abs(len(r["y"]) - len(x)) <= 1
    peak, res = pr.spectral_peak_hz(r["y"], rate)
    assert abs(peak - f * p) <= res + 1e-9
    assert np.abs(r["offsets"]).max() <= r["plan"]["D"]


@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("t", [0.25, 0.5, 0.8, 1.25, 2.0, 4.0])
def test_tempo_keeps_the_tone_and_scales_the_length(rate, t):
    f = 300.0
    x = pr.tone(rate, f, 0.5)
    r = pr.process(x, rate, tempo=t)
    assert len(r["y"]) == r["plan"]["n1"] and abs(len(r["y"]) - len(x) / t) <= 1
    peak, res = pr.spectral_peak_hz(r["y"], rate)
    assert abs(peak - f) <= res + 1e-9
    # the first synthesis hop is the input itself
    np.testing.assert_allclose(r["y"][:r["plan"]["Hs"]], x[:r["plan"]["Hs"]], atol=1e-12)


def test_both_ratios_compose():
    rate, f = 22050, 200.0
    x = pr.tone(rate, f, 0.5)
    r = pr.process(x, rate, pitch=1.25, tempo=2.0)
    assert abs(len(r["y"]) - len(x) / 2.0) <= 1
    peak, res = pr.spectral_peak_hz(r["y"], rate)
    assert abs(peak - f * 1.25) <= res + 1e-9
    same = pr.process(x, rate, pitch=2.0, tempo=2.0)              # alpha = 1: no stretch stage, resampled by 2
    assert same["s"] is None and len(same["offsets"]) == 0 and abs(len(same["y"]) - len(x) / 2.0) <= 1


def test_tie_rule():
    rate = 16000
    pl = pr.plan(rate, 4000, None, 2.0)
    # silence scores 0 at every lag: the tie goes to delta = 0
    assert not pr.offsets(np.zeros(4000, np.float32), pl).any()
    # On a period-4 square wave every lag congruent to m = (c - a_k) mod 4 has the top score: the smallest |delta| of
    # that class wins, and for m = 2 the tie between -2 and +2 goes to -2.
    x = np.tile(np.array([0.5, 0.5, -0.5, -0.5], np.float32), 1000)
    seen = set()
    for tempo in (2.0, 1.01, 0.77):
        pl = pr.plan(rate, len(x), None, tempo)
        d = pr.offsets(x, pl)
        a, Hs = pl["a"], pl["Hs"]
        for k in range(1, pl["F"]):
            c = a[k - 1] + d[k - 1] + Hs
            if max(c, a[k] + pl["D"]) + pl["N"] > len(x) or a[k] - pl["D"] < 0:
                continue
            m = int((c - a[k]) % 4)
            assert d[k] == {0: 0, 1: 1, 2: -2, 3: -1}[m], (tempo, k)
            seen.add(m)
    assert seen == {0, 1, 2, 3}


def test_argument_checks():
    assert _prosody_arrays(None, None, 3) == (None, None)
    assert _prosody_arrays([None, 1.0, float("nan")], [1, None, None], 3) == (None, None)
    p, t = _prosody_arrays([1.25, None], None, 2)
    assert t is None and p[0] == np.float32(1.25) and np.isnan(p[1])
    for bad, what in (([0.4], "pitch"), ([2.5], "pitch"), (["x"], "pitch"), ([True], "pitch"), ([float("inf")], "pitch")):
        with pytest.raises(OperationError, match="utterance 0: pitch"):
            _prosody_arrays(bad, None, 1)
    for bad in ([None, 0.2], [None, 5.0], [None, float("-inf")]):
        with pytest.raises(OperationError, match="utterance 1: tempo"):
            _prosody_arrays(None, bad, 2)
    with pytest.raises(OperationError, match="2 entries for 3"):
        _prosody_arrays([1.0, 1.0], None, 3)


def test_alignment_scales_with_the_warp():
    frames, src = [2, 3, 0, 5, 1], [-1, 0, 0, 1, -1]
    plain = _alignment("ab", src, frames, 11 * 256)
    assert [(a.start_sample, a.num_samples) for a in plain] == [(0, 512), (512, 768), (1280, 1280), (2560, 256)]
    for n in (11 * 256 // 2, 1877, 4 * 11 * 256 + 3):
        w = _alignment("ab", src, frames, n, warped=True)
        assert [a.phoneme for a in w] == [a.phoneme for a in plain]
        assert w[0].start_sample == 0 and sum(a.num_samples for a in w) == n
        for a, b in zip(w, w[1:]):
            assert b.start_sample == a.start_sample + a.num_samples
        for a, b in zip(w, plain):
            assert abs(a.start_sample - b.start_sample * n / (11 * 256)) <= 0.5
    assert isinstance(plain[0], PhonemeAlignment)


class _Fake:
    def audio_output_info(self):
        return sonata_b200.AudioInfo(22050, 1, 2)

    def phonemize_text(self, text):
        raise sonata_b200.SonataError("no phonemizer")

    def phonemes_to_input_ids(self, p):
        return [1, 2]

    def get_speakers(self):
        return None


def test_streaming_modes_refuse_by_name():
    refuse_prosody(None, 1.0, "x")
    synth = SonataSpeechSynthesizer(_Fake())
    with pytest.raises(OperationError, match="synthesize_streamed cannot shift pitch or tempo"):
        next(synth.synthesize_streamed("a", pitch_ratio=1.25))
    with pytest.raises(OperationError, match="RealtimeBatch cannot shift pitch or tempo"):
        RealtimeBatch(_Fake()).add("a", tempo=2.0)
    with pytest.raises(OperationError, match="StreamBatch cannot shift pitch or tempo"):
        StreamBatch(_Fake(), 72, 3).add([1, 2], tempo=0.5)
    with pytest.raises(OperationError, match="stream_synthesis cannot shift pitch or tempo"):
        sonata_b200.VitsStreamingModel.stream_synthesis(_Fake(), "a", 72, 3, pitch=0.8)
    with pytest.raises(OperationError, match="pitch ratio 3.0"):
        next(synth.synthesize_lazy("a", pitch_ratio=3.0))
    with pytest.raises(OperationError, match="tempo ratio 9.0"):
        synth.synthesize_parallel("a", tempo=9.0)


def test_cli_flags_and_refusal():
    args = cli.build_parser().parse_args(["v.json", "--pitch-ratio", "1.25", "--tempo", "0.5"])
    assert (args.pitch_ratio, args.tempo) == (1.25, 0.5)
    args = cli.build_parser().parse_args(["v.json"])
    assert args.pitch_ratio is None and args.tempo is None
    synth = SonataSpeechSynthesizer(_Fake())
    with pytest.raises(OperationError, match="realtime mode cannot shift pitch or tempo"):
        cli.process_request(synth, None, {"text": "a", "mode": "realtime", "tempo": 2.0}, None)
    with pytest.raises(OperationError, match="utterance 0: pitch ratio 0.1"):
        cli.process_request(synth, None, {"text": "a", "pitch_ratio": 0.1}, None)
