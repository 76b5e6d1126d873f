"""GPU (-m gpu): the reverse coupling flow and the HiFi-GAN decoder stage by stage against float64 (tests/dec_reference.py),
each stage recomputed from the kernel's own captured input so that errors do not compound:
    z_p -> flow.3 -> flow.2 -> flow.1 -> flow.0 (= z) -> dec.pre -> dec.up{i} -> dec.mrf{i} -> wav.
Backend 1 (bf16x2 wgmma) stages are held per 128-row tile to dec_reference.tc_bound, the waveform and backend 0 (fp32
CUDA cores) per utterance to dec_reference.f32_bound.  Run with -s to print the per-stage tables: max |got - ref|, the
emulation's (or the fp32 host run's) max error, and the largest ratio of a tile's error to its bound."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import sonata_b200  # noqa: E402
from sonata_b200 import PiperSynthesisConfig, voicegen, workload  # noqa: E402
from sonata_b200.job import SynthesisJob  # noqa: E402

pytestmark = pytest.mark.gpu

# frame counts at and around the 128-frame granule and the decoder's 128 U-row tiles, plus one long utterance
EDGE_FRAMES = (1, 2, 127, 128, 129, 255, 257, 700)
EDGE_IDS = 12
# name -> (quality, speakers, speaker of each utterance of the edge batch or None)
VOICES = {"medium": ("medium", 1, None), "high": ("high", 1, None), "x_low": ("x_low", 1, None),
          "medium_spk4": ("medium", 4, (0, 3, 1, 2, 3, 0, 2, 1))}
EDGE_CASES = [("medium", 1), ("medium", 0), ("high", 1), ("high", 0), ("x_low", 1), ("medium_spk4", 1)]


@pytest.fixture(scope="module")
def models(lib_built):
    d = voicegen.default_voice_dir()
    ms = {}

    def get(voice):
        if voice not in ms:
            quality, nspk, _ = VOICES[voice]
            ms[voice] = sonata_b200.from_config_path(voicegen.write_voice(d, quality, n_speakers=nspk), device=0)
        return ms[voice]
    yield get
    for m in ms.values():
        m.close()


_TENSORS = {}


def _tensors(voice):
    if voice not in _TENSORS:
        quality, nspk, _ = VOICES[voice]
        _TENSORS[voice] = voicegen.make_tensors(quality, n_speakers=nspk)
    return _TENSORS[voice]


def _frames(n_ids, y_len):
    """Per-id frame counts summing to y_len."""
    return np.diff(np.rint(np.linspace(0, y_len, n_ids + 1))).astype(np.int32)


def _check_job(voice, backend, job, utts, sids, table):
    """Every stage of utterances `utts` of a run debug job against float64; returns the failures."""
    import dec_reference as dr
    t = _tensors(voice)
    a = dr.arch(t)
    half = a["inter"] // 2
    wavs = job.fetch()
    fails = []
    for b in utts:
        sid = sids[b] if sids else None
        u = {"wav": wavs[b].samples.as_slice().astype(np.float32).reshape(-1, 1)}
        for name, src, _ in dr.stages(t, sid):
            if name != "wav":
                u[name] = job.debug_fetch(name, b)
        u["z_p"], u["z"] = job.debug_fetch("z_p", b), job.debug_fetch("z", b)
        assert np.array_equal(u["z"], u["flow.0"]), (voice, b)
        y_len = u["z"].shape[0]
        for s_i, (name, src, fn) in enumerate(dr.stages(t, sid)):
            x, got = u[src], u[name]
            ref = fn(x, dr.Arith("f64"))
            assert got.shape == tuple(ref.shape), (voice, b, name, got.shape, tuple(ref.shape))
            assert np.isfinite(got).all(), (voice, b, name)
            if name.startswith("flow."):
                # the conditioning half passes through bit for bit (step s even: the target is z[:half], odd: z[half:])
                keep = slice(half, None) if s_i % 2 == 0 else slice(0, half)
                assert np.array_equal(got[:, keep], x[:, keep]), (voice, b, name)
            if name == "wav" or backend == 0:
                e, e_yard, r = dr.f32_check(got, ref, fn(x, dr.Arith("f32")))
                tile = -1
            else:
                e, e_yard, r, tile = dr.tc_check(got, ref, fn(x, dr.Arith("emu")), dr.tc_mult(t, name))
            row = table.setdefault((voice, backend, name), [0.0, 0.0, 0.0, ""])
            if r >= row[2]:
                row[2], row[3] = r, f"utt {b} y_len {y_len} tile {tile}"
            row[0], row[1] = max(row[0], e), max(row[1], e_yard)
            if r > 1.0:
                fails.append((voice, backend, b, y_len, name, tile, r))
    return fails


def _print(table, title):
    print(f"\n{title}\n{'voice':12s} be {'stage':9s} {'max|err|':>9s} {'emu/fp32':>9s} {'of bound':>8s}  worst")
    for (voice, backend, name), (e, ey, r, where) in table.items():
        print(f"{voice:12s} {backend:2d} {name:9s} {e:9.2e} {ey:9.2e} {r:8.3f}  {where}")


@pytest.mark.parametrize("voice,backend", EDGE_CASES)
def test_flow_decoder_stages_at_edge_lengths(models, voice, backend):
    """One batch whose utterances have EDGE_FRAMES frames (forced per id), zero noise, default scales: every stage of
    every utterance within its bound; the multi-speaker voice's batch mixes speakers (per-granule bias slots)."""
    quality, nspk, spk = VOICES[voice]
    m = models(voice)
    m.set_backend(backend)
    try:
        batches = [workload.synthetic_ids(EDGE_IDS // 2, utt=40 + i)[:EDGE_IDS] for i in range(len(EDGE_FRAMES))]
        configs = [PiperSynthesisConfig(None if spk is None else spk[b], 0.0, 1.0, 0.0) for b in range(len(batches))]
        job = SynthesisJob(m, batches, debug=True, configs=configs)
        job.set_durations(None, [_frames(EDGE_IDS, y) for y in EDGE_FRAMES])
        job.run()
        assert job.lengths()[0] == list(EDGE_FRAMES)
        table = {}
        fails = _check_job(voice, backend, job, range(len(batches)), spk, table)
        job.close()
    finally:
        m.set_backend(1)
    _print(table, f"{voice} backend {backend}, frames {EDGE_FRAMES}")
    assert not fails, fails


@pytest.mark.parametrize("voice,batch,phonemes", [("medium", 32, 256), ("high", 16, 512)])
def test_flow_decoder_stages_full_size(models, voice, batch, phonemes):
    """The production launches (hundreds of tiles per CTA): a batch of `batch` utterances of `phonemes` phonemes at the
    voice's default noise, backend 1; every stage of the first, second, middle and last utterance within its bound."""
    m = models(voice)
    batches = [workload.synthetic_ids(phonemes, utt=200 + i) for i in range(batch)]
    job = SynthesisJob(m, batches, debug=True)
    job.run()
    table = {}
    fails = _check_job(voice, 1, job, sorted({0, 1, batch // 2, batch - 1}), None, table)
    frames = job.lengths()[0]
    job.close()
    torch.cuda.empty_cache()
    _print(table, f"{voice} {batch} x {phonemes} phonemes, {sum(frames)} frames")
    assert not fails, fails
