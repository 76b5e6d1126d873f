"""Host (no GPU): the formant stage's specification (tests/formant_reference.py) does what it claims on a constructed
vowel, measured independently of it (LPC formants, F0 from the harmonic spacing), and the Python layer checks its
arguments and refuses formant ratios on the streaming surfaces."""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import formant_reference as fr
import prosody_reference as pr
import sonata_b200
from sonata_b200 import cli
from sonata_b200.core import OperationError
from sonata_b200.piper import StreamBatch, _formant_array, refuse_formants
from sonata_b200.synth import RealtimeBatch, SonataSpeechSynthesizer


def _shifted(x, rate, pitch):
    return pr.process(x, rate, pitch=pitch)["y"].astype(np.float32) if pitch != 1.0 else x


@pytest.mark.parametrize("rate", [22050, 16000])
def test_pitch_shift_keeps_formants(rate):
    x = fr.vowel(rate)
    src = fr.lpc_formants(x, rate)
    assert len(src) == 3 and np.all(np.abs(src / np.array([700.0, 1220.0, 2600.0]) - 1) < 0.05)
    y = _shifted(x, rate, 1.5)
    # without a formant ratio the formants move with the pitch: the measurement tells the two cases apart
    moved = fr.lpc_formants(y, rate)
    assert np.all(np.abs(moved / (1.5 * src) - 1) < 0.1), moved
    z = fr.apply(y, rate, 1.0, pitch=1.5).astype(np.float32)
    kept = fr.lpc_formants(z, rate)
    assert len(kept) == 3 and np.all(np.abs(kept / src - 1) < 0.1), kept
    f0 = fr.f0_from_harmonics(z, rate, 180.0)
    assert abs(f0 / (1.5 * fr.f0_from_harmonics(x, rate, 120.0)) - 1) < 0.01, f0


@pytest.mark.parametrize("rate", [22050, 16000])
def test_formant_ratio_alone_moves_formants_at_the_same_pitch(rate):
    x = fr.vowel(rate)
    src = fr.lpc_formants(x, rate)
    z = fr.apply(x, rate, 1.25).astype(np.float32)
    got = fr.lpc_formants(z, rate)
    assert len(got) == 3 and np.all(np.abs(got / (1.25 * src) - 1) < 0.1), got
    assert abs(fr.f0_from_harmonics(z, rate, 120.0) / fr.f0_from_harmonics(x, rate, 120.0) - 1) < 0.01
    assert len(z) == len(x)


def test_high_voice_keeps_formants():
    """A 220 Hz voice (the harmonics 4.5 ms apart, near the 4 ms cutoff): a formant-preserving shift by 1.25 still
    keeps every formant within 10 %."""
    rate = 22050
    x = fr.vowel(rate, f0=220.0)
    src = fr.lpc_formants(x, rate)
    z = fr.apply(_shifted(x, rate, 1.25), rate, 1.0, pitch=1.25).astype(np.float32)
    kept = fr.lpc_formants(z, rate)
    assert len(kept) == 3 and np.all(np.abs(kept / src - 1) < 0.1), (src, kept)


def test_silence_gives_silence():
    out = fr.apply(np.zeros(5000, np.float32), 22050, 1.3, pitch=1.1)
    assert np.all(out == 0)


@pytest.mark.parametrize("n2", [1, 255, 256, 1023, 1024, 1025])
def test_short_signals(n2):
    rng = np.random.default_rng(n2)
    y = (0.3 * rng.standard_normal(n2)).astype(np.float32)
    out = fr.apply(y, 22050, 0.8, pitch=1.2)
    assert out.shape == (n2,) and np.all(np.isfinite(out))
    # with r_m = 1 everywhere the stage would be the identity up to rounding (it is skipped instead)
    same = fr.apply(y, 22050, 1.2, pitch=1.2)
    np.testing.assert_allclose(same, y, atol=1e-6)


def test_skipping():
    assert not fr.asks(10000, None, pitch=1.25)
    assert not fr.asks(10000, float("nan"), pitch=1.25)
    assert not fr.asks(10000, 1.25, pitch=1.25)          # phi == p without a contour keeps its bits
    assert not fr.asks(10000, 1.0)
    assert fr.asks(10000, 1.0, pitch=1.25)               # an explicit 1 asks under a pitch ratio
    assert fr.asks(10000, 1.2)
    # a contour: only frames whose centre lies in a piece with p_r != phi ask
    assert fr.asks(10000, 1.0, Q=[0.0, 4000.0], P=[1.0, 1.3])
    assert not fr.asks(10000, 1.0, Q=[0.0, 20000.0], P=[1.0, 1.3])     # the second piece holds no frame centre


def test_argument_checks():
    assert _formant_array(None, 3) is None
    assert _formant_array([None, float("nan"), None], 3) is None
    a = _formant_array([None, 1.0, 0.5], 3)
    assert math.isnan(a[0]) and a[1] == 1.0 and a[2] == 0.5
    for bad, msg in ((2.5, "utterance 1: formant ratio 2.5"), (0.25, "utterance 1: formant ratio 0.25"),
                     (float("inf"), "utterance 1: formant ratio inf"), ("x", "utterance 1: formant ratio 'x'"),
                     (True, "utterance 1: formant ratio True")):
        with pytest.raises(OperationError, match=msg):
            _formant_array([None, bad], 2)
    with pytest.raises(OperationError):
        _formant_array([1.0], 2)


class _Fake:
    """A model without a device: records what the synthesizer's batch modes ask of it."""

    def __init__(self):
        self.calls = []

    def audio_output_info(self):
        return sonata_b200.AudioInfo(22050, 1, 2)

    def phonemize_text(self, text):
        raise sonata_b200.SonataError("no phonemizer")

    def phonemes_to_input_ids(self, p):
        return [1, 2]

    def get_speakers(self):
        return None

    def speak_batch(self, phs, **kw):
        self.calls.append(kw)
        return [sonata_b200.Audio(sonata_b200.AudioSamples(np.zeros(8, np.float32)), 22050) for _ in phs]


def test_streaming_surfaces_refuse_by_name():
    refuse_formants(None, "x")
    refuse_formants(float("nan"), "x")
    synth = SonataSpeechSynthesizer(_Fake())
    with pytest.raises(OperationError, match="stream_synthesis cannot apply a formant ratio"):
        sonata_b200.VitsStreamingModel.stream_synthesis(_Fake(), "a", 72, 3, formant_ratio=1.0)
    with pytest.raises(OperationError, match="StreamBatch cannot apply a formant ratio"):
        StreamBatch(_Fake(), 72, 3).add([1, 2], formant_ratio=1.2)
    with pytest.raises(OperationError, match="synthesize_streamed cannot apply a formant ratio"):
        next(synth.synthesize_streamed("a", formant_ratio=1.2))
    with pytest.raises(OperationError, match="RealtimeBatch cannot apply a formant ratio"):
        RealtimeBatch(_Fake()).add("a", formant_ratio=0.8)


def test_synthesizer_modes_pass_the_ratio():
    m = _Fake()
    synth = SonataSpeechSynthesizer(m)
    list(synth.synthesize_lazy("a\nb", formant_ratio=1.2, pitch_ratio=1.25))
    assert m.calls[-1] == {"pitches": [1.25], "formants": [1.2]}
    list(synth.synthesize_parallel("a\nb", formant_ratio=1.0))
    assert m.calls[-1] == {"formants": [1.0, 1.0]}
    list(synth.synthesize_parallel("a", formant_ratio=float("nan")))
    assert m.calls[-1] == {}
    with pytest.raises(OperationError, match="formant ratio 3.0"):
        next(synth.synthesize_lazy("a", formant_ratio=3.0))
    with pytest.raises(OperationError, match="formant ratio 0.1"):
        synth.synthesize_parallel("a", formant_ratio=0.1)


def test_cli_flag_json_and_realtime_refusal():
    args = cli.build_parser().parse_args(["v.json", "--formant-ratio", "1.1"])
    assert args.formant_ratio == 1.1
    assert cli.build_parser().parse_args(["v.json"]).formant_ratio is None
    m = _Fake()
    synth = SonataSpeechSynthesizer(m)
    with pytest.raises(OperationError, match="realtime mode cannot apply a formant ratio"):
        cli.process_request(synth, None, {"text": "a", "mode": "realtime", "formant_ratio": 1.0}, None)
    with pytest.raises(OperationError, match="utterance 0: formant ratio 5.0"):
        cli.process_request(synth, None, {"text": "a", "formant_ratio": 5.0}, None)
