"""CPU: live loudness streams' host side -- the float64 meter against the batch meter, its independence of chunking,
its ramp and its convergence, and the refusals of the Python and CLI layers that need no device."""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import loudness_reference as lr
import loudness_stream_reference as lsr
from sonata_b200.core import OperationError
from sonata_b200.piper import _check_live_loudness, _check_max_gain


def _speechlike(rate, seconds, seed=0):
    """Noise bursts under a slow envelope with pauses: a signal whose level moves, as speech does."""
    rng = np.random.default_rng(seed)
    n = int(rate * seconds)
    t = np.arange(n) / rate
    env = 0.05 + 0.2 * np.abs(np.sin(2 * np.pi * 0.7 * t)) * (np.sin(2 * np.pi * 0.23 * t) > -0.6)
    return (env * rng.standard_normal(n) * 0.5).astype(np.float32)


@pytest.mark.parametrize("rate", (8000, 22050, 48000))
def test_readings_from_step_four_are_the_batch_meter(rate):
    x = _speechlike(rate, 2.3, seed=rate)
    L = lsr.readings(x, rate)
    S = lr.step(rate)
    assert len(L) == len(x) // S
    for m in range(4, len(L) + 1):
        want = lr.integrated(x[:m * S], rate)
        assert L[m - 1] == pytest.approx(want, abs=1e-9) or (L[m - 1] == want == -math.inf), m


def test_provisional_readings_and_silence():
    rate = 16000
    S = lr.step(rate)
    x = np.zeros(10 * S, np.float32)
    assert np.all(lsr.readings(x, rate) == -math.inf)
    y, L, a, clipped = lsr.meter(x, rate, -16.0)
    assert np.all(a == 1.0) and clipped == 0 and not y.any()
    x = lr.sine(rate, 0.35, peak=0.1)
    L = lsr.readings(x, rate)
    assert len(L) == 3 and np.all(np.isfinite(L))


@pytest.mark.parametrize("rate", (11025, 24000))
def test_output_does_not_depend_on_the_chunking(rate):
    x = _speechlike(rate, 1.7, seed=3)
    whole, _, _, _ = lsr.meter(x, rate, -18.0)
    rng = np.random.default_rng(5)
    S = lr.step(rate)
    for cuts in ([len(x)], [1, 1, S - 2, S, 3 * S + 7], list(rng.integers(1, 3 * S, 12))):
        m = lsr.Meter(rate, -18.0)
        parts, pos = [], 0
        for c in cuts:
            parts.append(m.push(x[pos:pos + c]))
            pos += c
        parts.append(m.push(x[pos:]))
        assert np.concatenate(parts).tobytes() == whole.tobytes(), cuts


def test_ramp_is_continuous_across_step_boundaries():
    rate = 22050
    S = lr.step(rate)
    x = _speechlike(rate, 3.0, seed=7)
    _, _, a, _ = lsr.meter(x, rate, -14.0)
    a_all = np.concatenate([[np.float32(1.0)], a])
    G = lsr.sample_gains(len(x), a_all, S).astype(np.float64)
    # each step ends on its boundary's gain, and the next step starts one ramp increment from it
    for m in range(1, len(a) - 1):
        assert G[(m + 1) * S - 1] == a_all[m]
        assert abs(G[(m + 1) * S] - a_all[m]) <= abs(float(a_all[m + 1]) - float(a_all[m])) / S + 1e-6
    # no jump between neighbours larger than the steepest ramp, give or take the f32 rounding of G
    assert np.max(np.abs(np.diff(G))) <= np.max(np.abs(np.diff(a_all.astype(np.float64)))) / S + 1e-6


@pytest.mark.parametrize("target", (-23.0, -16.0))
def test_a_constant_level_converges_to_the_target(target):
    rate = 16000
    x = lr.sine(rate, 20.0, peak=0.03)
    y, L, a, clipped = lsr.meter(x, rate, target)
    assert clipped == 0
    assert abs(lr.integrated(y[-3 * rate:], rate) - target) < 0.1
    assert abs(L[-1] - lr.integrated(x[:len(L) * lr.step(rate)], rate)) < 1e-9


def test_max_gain_caps_the_gain_and_the_clamp_counts():
    rate = 8000
    quiet = lr.sine(rate, 2.0, peak=0.001)
    _, _, a, _ = lsr.meter(quiet, rate, -10.0, max_gain_db=6.0)
    assert np.max(a) == np.float32(10 ** (6.0 / 20.0))
    loud = lr.sine(rate, 2.0, peak=0.9)
    _, _, _, clipped = lsr.meter(loud, rate, 0.0, max_gain_db=40.0)
    assert clipped > 0


@pytest.mark.parametrize("bad", (1.0, -80.0, float("inf"), "x", True))
def test_bad_targets_are_refused_naming_the_stream(bad):
    with pytest.raises(OperationError, match="stream 4"):
        _check_live_loudness(bad, None, None, "stream 4")


@pytest.mark.parametrize("bad", (-1.0, 41.0, float("nan"), float("inf"), "20"))
def test_bad_max_gains_are_refused_naming_the_stream(bad):
    with pytest.raises(OperationError, match="stream 2"):
        _check_max_gain(bad, "stream 2")
    with pytest.raises(OperationError, match="stream 2"):
        _check_live_loudness(-16.0, bad, None, "stream 2")


def test_flac_and_a_lone_max_gain_are_refused():
    with pytest.raises(OperationError, match="FLAC"):
        _check_live_loudness(-16.0, None, "flac", "stream 0")
    with pytest.raises(OperationError, match="live_loudness"):
        _check_live_loudness(None, 12.0, None, "stream 0")
    _check_live_loudness(-16.0, 12.0, "mulaw", "stream 0")
    _check_live_loudness(None, None, None, "stream 0")


def test_cli_live_loudness_only_in_realtime_mode(voice_paths, tmp_path):
    from sonata_b200 import cli
    (tmp_path / "in.txt").write_text("hɛloʊ\n", encoding="utf-8")
    base = [voice_paths["medium"], "-f", str(tmp_path / "in.txt"), "--device", "-1"]
    for mode in ("lazy", "parallel"):
        with pytest.raises(OperationError, match="--loudness"):
            cli.main(base + ["--mode", mode, "--live-loudness", "-16"])
    with pytest.raises(OperationError, match="--loudness"):
        cli.main(base + ["--live-loudness", "-16"])
    with pytest.raises(OperationError, match="--loudness"):
        cli.main(base + ["--mode", "realtime", "--live-loudness", "-16", "-o", str(tmp_path / "o.wav")])
    # the batch target keeps refusing realtime mode
    with pytest.raises(OperationError, match="realtime"):
        cli.main(base + ["--mode", "realtime", "--loudness", "-23"])
    for bad in ("1", "-80", "inf"):
        with pytest.raises(OperationError, match="request"):
            cli.main(base + ["--mode", "realtime", "--live-loudness", bad])
    with pytest.raises(OperationError, match="maximum gain"):
        cli.main(base + ["--mode", "realtime", "--live-loudness", "-16", "--max-gain-db", "50"])
    with pytest.raises(OperationError, match="live_loudness"):
        cli.main(base + ["--mode", "realtime", "--max-gain-db", "10"])


def test_cli_realtime_refuses_live_loudness_on_a_voice_without_device_streaming(voice_paths, tmp_path):
    from sonata_b200 import cli
    (tmp_path / "in.txt").write_text("hɛloʊ\n", encoding="utf-8")
    base = [voice_paths["medium"], "-f", str(tmp_path / "in.txt"), "--device", "-1"]
    with pytest.raises(OperationError, match="live loudness"):
        cli.main(base + ["--mode", "realtime", "--live-loudness", "-16"])
