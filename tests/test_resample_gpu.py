"""GPU (-m gpu): results at a caller-chosen output sample rate, resampled on the device.

The resampled waveform is resample_poly of the voice-rate waveform (float64 reference, error bound per sample); a rate
of 0 or the voice's own changes no bit; an utterance resampled in a mixed batch equals itself run alone; the i16 paths
convert the resampled f32; and alignment, WAV header and length agree with the output rate."""
import ctypes as C
import os
import struct
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import resample_reference as rr
import sonata_b200
from sonata_b200 import OperationError, PiperSynthesisConfig, cli, voicegen, workload
from sonata_b200 import _native as N
from sonata_b200.core import AudioSamples
from sonata_b200.job import SynthesisJob

pytestmark = pytest.mark.gpu

DEFAULT = PiperSynthesisConfig(None, 0.667, 1.0, 0.8)


@pytest.fixture(scope="module")
def voices(lib_built):
    d = voicegen.default_voice_dir()
    paths = {q: voicegen.write_voice(d, q) for q in ("medium", "high", "low", "x_low")}
    ms = {}

    def get(q):
        if q not in ms:
            ms[q] = sonata_b200.from_config_path(paths[q], device=0)
            ms[q].set_fallback_synthesis_config(DEFAULT)
        return ms[q]
    get.paths = paths
    yield get
    for m in ms.values():
        m.close()


def _ids(n, utt):
    return list(workload.synthetic_ids(n, utt=utt))


def _run(m, batches, seeds, rates=None):
    job = SynthesisJob(m, batches, seeds=seeds, output_rates=rates)
    job.run()
    audio = job.fetch()
    out = dict(wav=[a.samples.as_slice().copy() for a in audio], sr=[a.info.sample_rate for a in audio],
               i16=job.fetch_i16(), lengths=job.lengths(), profile=job.profile())
    total = sum(len(w) for w in out["wav"])
    f32 = np.zeros(total, np.float32)
    i16 = np.zeros(total, np.int16)
    assert job.copy_out(f32.ctypes.data, f32.nbytes, 0) == f32.nbytes
    assert job.copy_out(i16.ctypes.data, i16.nbytes, 1) == i16.nbytes
    out["f32_copy"], out["i16_copy"] = f32, i16
    job.close()
    return out


def _debug_resample(x, in_rate, out_rate):
    up, down = rr.ratio(in_rate, out_rate)
    x = np.ascontiguousarray(x, np.float32)
    y = np.zeros(rr.n_out(len(x), up, down), np.float32)
    err = N.sb200_error()
    rc = N.lib().sb200_debug_resample(0, x.ctypes.data_as(C.POINTER(C.c_float)), x.size, in_rate, out_rate,
                                      y.ctypes.data_as(C.POINTER(C.c_float)), C.byref(err))
    assert rc == 0
    return y


@pytest.mark.parametrize("quality", ["medium", "high", "low", "x_low"])
def test_accuracy_against_resample_poly(voices, quality):
    m = voices(quality)
    vr = m.audio_output_info().sample_rate
    batches = [_ids(20, 1), _ids(7, 2)]
    seeds = [11, 12]
    base = _run(m, batches, seeds)
    for target in rr.TARGETS:
        if target == vr:
            continue
        up, down = rr.ratio(vr, target)
        got = _run(m, batches, seeds, [target, target])
        for b in range(len(batches)):
            x = base["wav"][b]
            y = got["wav"][b]
            assert got["sr"][b] == target
            assert len(y) == rr.n_out(len(x), up, down)
            err = np.abs(y.astype(np.float64) - rr.resample64(x, up, down))
            tol = rr.bound(x, up, down)
            assert np.all(err <= tol), (quality, target, b, float(np.max(err - tol)))
            # the kernel over one host buffer gives the job's bits
            np.testing.assert_array_equal(_debug_resample(x, vr, target), y)
        assert any(r["name"] == "resample" for r in got["profile"])
        assert not any(r["name"] == "resample" for r in base["profile"])


def test_identity_rates_change_no_bit(voices):
    m = voices("medium")
    batches = [_ids(30, 3), _ids(9, 4), _ids(14, 5)]
    base = _run(m, batches, [1, 2, 3])
    for rates in ([0, 0, 0], [22050, 0, 22050], [None, 22050, None]):
        got = _run(m, batches, [1, 2, 3], rates)
        for key in ("wav", "i16"):
            for a, b in zip(base[key], got[key]):
                np.testing.assert_array_equal(a, b)
        np.testing.assert_array_equal(base["f32_copy"], got["f32_copy"])
        np.testing.assert_array_equal(base["i16_copy"], got["i16_copy"])
        assert base["lengths"] == got["lengths"]
        assert not any(r["name"] == "resample" for r in got["profile"])
    ids = [m.phonemes_to_input_ids("hɛloʊ wɜːld"), m.phonemes_to_input_ids("ab")]
    plain = m.infer_batch_with_values(ids, seeds=[5, 6])
    same = m.infer_batch_with_values(ids, seeds=[5, 6], output_rates=[0, 22050])
    for a, b in zip(plain, same):
        np.testing.assert_array_equal(a.samples.as_slice(), b.samples.as_slice())
        assert b.info.sample_rate == 22050


@pytest.mark.parametrize("size", ["small", "c2"])
def test_mixed_batch_equals_alone(voices, size):
    m = voices("medium")
    B, n = (6, 24) if size == "small" else (32, 256)
    batches = [_ids(n - 3 * (b % 5), 100 + b) for b in range(B)]
    rates = [(0, 8000, 48000, 22050, 11025, 44100, 24000, 16000, 32000)[b % 9] for b in range(B)]
    seeds = [1000 + b for b in range(B)]
    mixed = _run(m, batches, seeds, rates)
    frames, samples, offs = mixed["lengths"]
    for b in range(B):
        alone = _run(m, [batches[b]], [seeds[b]], [rates[b]])
        np.testing.assert_array_equal(mixed["wav"][b], alone["wav"][0])
        np.testing.assert_array_equal(mixed["i16"][b], alone["i16"][0])
        assert mixed["sr"][b] == (rates[b] or 22050)
        up, down = rr.ratio(22050, rates[b] or 22050)
        assert samples[b] == len(mixed["wav"][b]) == rr.n_out(frames[b] * 256, up, down)
        np.testing.assert_array_equal(mixed["f32_copy"][offs[b]:offs[b] + samples[b]], mixed["wav"][b])
        np.testing.assert_array_equal(mixed["i16_copy"][offs[b]:offs[b] + samples[b]], mixed["i16"][b])
        # i16 is to_i16_vec of the resampled f32
        np.testing.assert_array_equal(mixed["i16"][b], AudioSamples(mixed["wav"][b]).to_i16_vec())


def test_caller_device_buffer_holds_the_resampled_result(voices):
    import torch
    m = voices("medium")
    batches = [_ids(40, 7), _ids(12, 8)]
    ref = _run(m, batches, [7, 8], [48000, 8000])
    total = sum(len(w) for w in ref["wav"])
    job = SynthesisJob(m, batches, seeds=[7, 8], output_rates=[48000, 8000])
    small = torch.zeros(total - 1, dtype=torch.float32, device="cuda:0")
    with pytest.raises(OperationError):
        job.run(small.data_ptr(), small.numel())
    buf = torch.zeros(total, dtype=torch.float32, device="cuda:0")
    job.run(buf.data_ptr(), buf.numel())
    torch.cuda.synchronize()
    np.testing.assert_array_equal(buf.cpu().numpy(), np.concatenate(ref["wav"]))
    job.close()


def test_unsupported_rates_are_operation_errors(voices):
    m = voices("medium")
    batches = [_ids(10, 9), _ids(11, 10)]
    job = SynthesisJob(m, batches, seeds=[1, 2], output_rates=[8000, 48000])
    # the C layer checks too: bypass the Python check
    bad = np.array([8000, 12345], np.uint32)
    err = N.sb200_error()
    rc = m._lib.sb200_job_set_output_rates(job._h, bad.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(err))
    assert rc == 19 and err.code == 19
    msg = C.string_at(err.message).decode()
    N.lib().sb200_string_free(err.message)
    assert "utterance 1" in msg and "12345" in msg
    job.run()                                            # the failed call left the rates as they were
    assert [a.info.sample_rate for a in job.fetch()] == [8000, 48000]
    job.close()
    with pytest.raises(OperationError, match="utterance 0"):
        m.speak_batch(["ab"], output_rates=[96000])
    with pytest.raises(OperationError, match="utterance 1"):
        m.infer_batch_with_values(batches, output_rates=[8000, 44000])


def test_alignment_and_wav_at_output_rate(voices, tmp_path):
    m = voices("medium")
    phs = ["hɛloʊ", "ðɪs ɪz ə tɛst"]
    res = m.speak_batch_with_alignment(phs, seeds=[3, 4], output_rates=[8000, 48000])
    for (audio, al), rate in zip(res, (8000, 48000)):
        assert audio.info.sample_rate == rate
        assert al[0].start_sample == 0
        for a, b in zip(al, al[1:]):
            assert a.start_sample + a.num_samples == b.start_sample
        assert al[-1].start_sample + al[-1].num_samples == len(audio)
    plain = m.speak_batch_with_alignment(phs, seeds=[3, 4])
    for (a, _), (p, _), rate in zip(res, plain, (8000, 48000)):
        up, down = rr.ratio(22050, rate)
        assert len(a) == rr.n_out(len(p), up, down)
    m.set_fallback_synthesis_config(DEFAULT)
    (tmp_path / "in.txt").write_text("hɛloʊ\nwɜːld\n", encoding="utf-8")
    out = tmp_path / "o.wav"
    assert cli.main([voices.paths["medium"], "-f", str(tmp_path / "in.txt"), "-o", str(out), "--output-rate", "16000",
                     "--seed", "5"]) == 0
    raw = open(out, "rb").read()
    rate, = struct.unpack("<I", raw[24:28])
    data_bytes, = struct.unpack("<I", raw[40:44])
    assert rate == 16000
    m.set_fallback_synthesis_config(DEFAULT)
    ref = m.speak_batch(["hɛloʊ", "wɜːld"], seeds=[5, 6], output_rates=[16000, 16000])
    assert data_bytes == 2 * sum(len(a) for a in ref)
