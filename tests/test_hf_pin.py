"""The oracle and the CUDA path against an implementation we did not write.

`tests/hf_reference.py` loads the synthetic *high* voice (ResBlock1, the en_US-ryan-high architecture of BASELINE
config 3) into Hugging Face transformers' `VitsModel` and runs ITS forward.  The committed fixtures under
`tests/golden/hf/` hold what transformers produced (generator: `tests/golden/hf/make_hf_golden.py`): ids, scales, the
Gaussian draws of the forward, frame count, waveform.

* CPU: the oracle reproduces the transformers waveform to ~3e-6, deterministic AND stochastic paths, and -- when
  transformers is importable -- on fresh inputs run live.  This is what pins the oracle (DESIGN.md section 0).
* GPU: the CUDA path against the same fixtures and live runs, through the C ABI, within the north-star tolerance.
"""
import glob
import os
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from oracle import vits_oracle as vo  # noqa: E402
from sonata_b200 import PiperSynthesisConfig, voicegen  # noqa: E402

HF_GOLD = sorted(glob.glob(os.path.join(HERE, "golden", "hf", "*.npz")))
TOL_ORACLE = 2e-5       # fp32 vs fp32, different operation order (measured 2e-6 .. 4e-6)
TOL_WAV = 1e-3          # BASELINE.json: "waveform max-abs error <1e-3"


def _weights_crc(t):
    c = 0
    for k in sorted(t):
        c = zlib.crc32(np.ascontiguousarray(t[k]).tobytes(), c)
    return c


@pytest.fixture(scope="module")
def high_tensors():
    return voicegen.make_tensors("high")


def test_fixtures_present():
    assert len(HF_GOLD) >= 3


@pytest.mark.parametrize("path", HF_GOLD, ids=[os.path.basename(p) for p in HF_GOLD])
def test_oracle_reproduces_transformers_vits(path, high_tensors, oracle_weights):
    g = np.load(path)
    assert int(g["weights_crc"]) == _weights_crc(high_tensors), "fixture was made from another synthetic voice"
    W = oracle_weights("high")
    ew = g["eps_w"].T[None] if "eps_w" in g else None
    ez = g["eps_z"].T[None] if "eps_z" in g else None
    st = {}
    wav = vo.infer(W, g["ids"], [float(s) for s in g["scales"]], eps_w=ew, eps_z=ez, stages=st).numpy()
    assert st["y_len"] == int(g["y_len"]) and wav.shape == g["wav"].shape       # every ceil'd duration agrees
    assert float(np.abs(wav - g["wav"]).max()) < TOL_ORACLE


@pytest.fixture(scope="module")
def hf_model(high_tensors):
    pytest.importorskip("transformers")
    import hf_reference as hf
    a = voicegen.ARCH["high"]
    return hf.load_piper_tensors(hf.build_hf_model(a), high_tensors, a)


def test_oracle_against_live_transformers_run(hf_model, oracle_weights):
    """Fresh inputs, not fixtures: 24 phonemes, three settings of (noise_scale, length_scale, noise_w)."""
    import hf_reference as hf
    W = oracle_weights("high")
    ids = vo.synthetic_ids(24, utt=7)
    for scales, seed in (((0.0, 1.0, 0.0), 0), ((0.667, 1.0, 0.8), 3), ((0.5, 1.3, 0.6), 5)):
        wav, ew, ez = hf.hf_infer(hf_model, ids, *scales, seed=seed)
        got = vo.infer(W, ids, list(scales), eps_w=ew[None] if scales[2] else None, eps_z=ez[None] if scales[0] else None).numpy()
        assert got.shape == wav.shape, (scales, got.shape, wav.shape)
        assert float(np.abs(got - wav).max()) < TOL_ORACLE, scales


def test_medium_voice_up_to_the_vocoder_against_live_transformers_run(oracle_weights):
    """transformers has no ResBlock2, so the medium voice cannot be run end to end there; everything in FRONT of the
    vocoder can: text encoder, duration predictor, alignment and flow of the medium voice (its own weights and gains)
    against `VitsModelOutput.spectrogram`."""
    pytest.importorskip("transformers")
    import hf_reference as hf
    a = voicegen.ARCH["medium"]
    m = hf.load_piper_tensors(hf.build_hf_model(a, decoder=False), voicegen.make_tensors("medium"), a, decoder=False)
    W = oracle_weights("medium")
    ids = vo.synthetic_ids(40, utt=3)
    for scales, seed in (((0.0, 1.0, 0.0), 0), ((0.667, 1.1, 0.8), 9)):
        _, ew, ez = hf.hf_infer(m, ids, *scales, seed=seed)
        z_hf = hf.hf_infer.last_spectrogram
        st = {}
        vo.encode(W, ids, list(scales), eps_w=ew[None] if scales[2] else None, eps_z=ez[None] if scales[0] else None, stages=st)
        z = st["z"][0].numpy()
        assert z.shape == z_hf.shape, (scales, z.shape, z_hf.shape)           # identical frame count
        assert float(np.abs(z - z_hf).max()) < 5e-5, scales                    # z is O(1..5)


def test_multi_speaker_conditioning_against_live_transformers_run():
    """The N1 row: `sid` -> emb_g -> 1x1 conditioning convs in the duration predictor, all four WaveNets and the vocoder
    input (piper/src/lib.rs:353-358), on a 3-speaker high voice, two speakers, stochastic path."""
    pytest.importorskip("transformers")
    import hf_reference as hf
    a = voicegen.ARCH["high"]
    T = voicegen.make_tensors("high", n_speakers=3)
    m = hf.load_piper_tensors(hf.build_hf_model(a, n_speakers=3), T, a)
    W = vo.to_torch(T)
    ids = vo.synthetic_ids(16, utt=11)
    outs = []
    for sid, scales, seed in ((0, (0.667, 1.0, 0.8), 2), (2, (0.667, 1.0, 0.8), 2), (2, (0.0, 1.0, 0.0), 0)):
        wav, ew, ez = hf.hf_infer(m, ids, *scales, seed=seed, speaker_id=sid)
        got = vo.infer(W, ids, list(scales), eps_w=ew[None] if scales[2] else None, eps_z=ez[None] if scales[0] else None,
                       sid=sid).numpy()
        assert got.shape == wav.shape, (sid, got.shape, wav.shape)
        assert float(np.abs(got - wav).max()) < TOL_ORACLE, sid
        outs.append(wav)
    assert outs[0].shape != outs[1].shape or float(np.abs(outs[0] - outs[1]).max()) > 1e-2      # the speaker matters


# ------------------------------------------------------------------------------------------------ CUDA path
def _run_cuda(m, ids, scales, eps_w, eps_z):
    from sonata_b200.job import SynthesisJob
    m.set_fallback_synthesis_config(PiperSynthesisConfig(None, float(scales[0]), float(scales[1]), float(scales[2])))
    job = SynthesisJob(m, [ids], None if eps_w is None else [eps_w], None if eps_z is None else [eps_z])
    job.run()
    frames = job.lengths()[0][0]
    wav = job.fetch()[0].samples.as_slice().copy()
    job.close()
    return frames, wav


@pytest.fixture(scope="module")
def high_model(voice_paths):
    import sonata_b200
    m = sonata_b200.from_config_path(voice_paths["high"], device=0)
    yield m
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("path", HF_GOLD, ids=[os.path.basename(p) for p in HF_GOLD])
def test_cuda_path_reproduces_transformers_vits(path, high_model):
    g = np.load(path)
    frames, wav = _run_cuda(high_model, g["ids"], g["scales"], g["eps_w"] if "eps_w" in g else None,
                            g["eps_z"] if "eps_z" in g else None)
    assert frames == int(g["y_len"]) and wav.shape == g["wav"].shape
    assert float(np.abs(wav - g["wav"]).max()) < TOL_WAV


@pytest.mark.gpu
def test_cuda_path_against_live_transformers_run(hf_model, high_model):
    """60 phonemes (122 ids), stochastic path, the noise transformers drew fed to the CUDA path through the C ABI."""
    import hf_reference as hf
    ids = vo.synthetic_ids(60, utt=1)
    worst = 0.0
    for scales, seed in (((0.0, 1.0, 0.0), 0), ((0.667, 1.0, 0.8), 3)):
        wav, ew, ez = hf.hf_infer(hf_model, ids, *scales, seed=seed)
        frames, got = _run_cuda(high_model, ids, scales, np.ascontiguousarray(ew.T) if scales[2] else None,
                                np.ascontiguousarray(ez.T) if scales[0] else None)
        if got.shape != wav.shape:
            # a duration sitting on the ceil cliff may flip between fp32 implementations (DESIGN.md section 4); the two
            # implementations must then still agree on all but that frame count
            assert abs(got.shape[0] - wav.shape[0]) <= 256 * 2, (got.shape, wav.shape)
            continue
        worst = max(worst, float(np.abs(got - wav).max()))
    assert worst < TOL_WAV
