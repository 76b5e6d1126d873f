"""GPU (-m gpu): streams at an output sample rate.

A resampled stream's chunks, concatenated, are bit for bit its whole input resampled at once (sb200_debug_resample of
the concatenation of its chunks after the same post-path), and within the float64 bound of resample_poly; i16 chunks
are to_i16_vec of the f32 ones; streams sharing a pass equal themselves alone; a rate of 0 or the voice's own changes no
bit; misuse of a resampler is an OPERATION_ERROR."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import resample_reference as rr
from sonata_b200 import OperationError, PiperSynthesisConfig, voicegen, workload
from sonata_b200 import _native as N
from sonata_b200.core import AudioSamples
from sonata_b200.piper import Resampler, StreamBatch, VitsStreamingModel, _Stream, _trim_frames
from sonata_b200.synth import RealtimeBatch

pytestmark = pytest.mark.gpu

DEFAULT = PiperSynthesisConfig(None, 0.667, 1.0, 0.8)
CS, PAD = 40, 3


@pytest.fixture(scope="module")
def voices(lib_built):
    d = voicegen.default_voice_dir()
    ms = {}

    def get(q):
        if q not in ms:
            ms[q] = VitsStreamingModel(voicegen.write_voice(d, q), device=0)
            ms[q].set_fallback_synthesis_config(DEFAULT)
        return ms[q]
    yield get
    for m in ms.values():
        m.close()


def _ids(n, utt):
    return list(workload.synthetic_ids(n, utt=utt))


def _debug_resample(x, in_rate, out_rate):
    up, down = rr.ratio(in_rate, out_rate)
    x = np.ascontiguousarray(x, np.float32)
    y = np.zeros(rr.n_out(len(x), up, down), np.float32)
    err = N.sb200_error()
    assert N.lib().sb200_debug_resample(0, x.ctypes.data_as(C.POINTER(C.c_float)), x.size, in_rate, out_rate,
                                        y.ctypes.data_as(C.POINTER(C.c_float)), C.byref(err)) == 0
    return y


def _schedule(enc):
    """SpeechStreamer's chunks of a latent: (chunk tuple with trims, fade, last)."""
    s = _Stream(0, enc, CS, PAD)
    out = []
    while not s.done:
        lo, hi, trim = s.next_chunk()
        out.append(((enc, lo, hi) + ((0, 0) if trim is None else _trim_frames(trim)), 0 if trim is None else 42, s.done))
    return out


def _run_stream(m, enc, resampler, pcm16=False):
    return [m.infer_decoder_batch([c], fade=f, resamplers=[resampler], last=[last], pcm16=pcm16)[0]
            for c, f, last in _schedule(enc)]


def _f32(chunks):
    return np.concatenate([c.as_slice() for c in chunks]) if chunks else np.zeros(0, np.float32)


SENTENCES = [(60, 1), (9, 2), (150, 3), (25, 4)]         # ids per sentence: long, one-shot, longer, short


def test_stream_batch_mixed_rates(voices):
    m = voices("medium")
    rates = [48000, None, 8000, 16000]
    seeds = [21, 22, 23, 24]
    sb = StreamBatch(m, CS, PAD)
    keys = [sb.add(_ids(n, u), seed=s, output_rate=r) for (n, u), s, r in zip(SENTENCES, seeds, rates)]
    got = {k: [] for k in keys}
    while len(sb):
        for k, a in sb.step():
            assert not isinstance(a, Exception), a
            got[k].append(a)
    encs = m.infer_encoder_batch([_ids(n, u) for n, u in SENTENCES], seeds=seeds)
    for k, enc, r in zip(keys, encs, rates):
        if r is None:
            ref = StreamBatch(m, CS, PAD)
            ref.add(_ids(*SENTENCES[keys.index(k)]), seed=seeds[keys.index(k)])
            alone = [a for _ in range(64) if len(ref) for _, a in ref.step()]
            assert len(alone) == len(got[k])
            for a, b in zip(alone, got[k]):
                np.testing.assert_array_equal(a.as_slice(), b.as_slice())
            continue
        # the same post-path at the voice's rate, chunk by chunk, then the kernel over the concatenation
        plain = _f32(_run_stream(m, enc, None))
        np.testing.assert_array_equal(_f32(got[k]), _debug_resample(plain, 22050, r))
        up, down = rr.ratio(22050, r)
        err = np.abs(_f32(got[k]).astype(np.float64) - rr.resample64(plain, up, down))
        assert np.all(err <= rr.bound(plain, up, down))
        # the stream alone, through its own resampler, gives the same chunks
        alone = _run_stream(m, enc, Resampler(m, r))
        assert [len(c) for c in alone] == [len(c) for c in got[k]]
        for a, b in zip(alone, got[k]):
            np.testing.assert_array_equal(a.as_slice(), b.as_slice())
        # i16 chunks are to_i16_vec of the f32 chunks
        i16 = _run_stream(m, enc, Resampler(m, r), pcm16=True)
        for a, b in zip(i16, alone):
            np.testing.assert_array_equal(a, b.to_i16_vec())


def test_host_and_device_post_paths_agree(voices):
    """Chunks at the voice's rate through the device post-path match the host's trim and crossfade."""
    m = voices("medium")
    enc = m.infer_encoder_batch([_ids(150, 3)], seeds=[5])[0]
    dev = _run_stream(m, enc, None)
    sb = StreamBatch(m, CS, PAD)
    sb.add(_ids(150, 3), seed=5)
    host = [a for _ in range(64) if len(sb) for _, a in sb.step()]
    assert len(dev) == len(host)
    for a, b in zip(dev, host):
        np.testing.assert_allclose(a.as_slice(), b.as_slice(), rtol=0, atol=2e-7)


def test_identity_rates_change_no_stream_bit(voices):
    m = voices("medium")
    out = []
    for rate in (None, 0, 22050):
        sb = StreamBatch(m, CS, PAD)
        sb.add(_ids(120, 7), seed=3, output_rate=rate)
        out.append([a.as_slice().copy() for _ in range(64) if len(sb) for _, a in sb.step()])
    for o in out[1:]:
        assert len(o) == len(out[0])
        for a, b in zip(o, out[0]):
            np.testing.assert_array_equal(a, b)


def test_one_frame_utterance_and_low_voice(voices):
    m = voices("medium")
    enc = m.infer_encoder_batch([_ids(5, 9)], durations=[[0] * 11 + [1]], seeds=[1])[0]
    assert enc.num_frames == 1
    y = m.infer_decoder_batch([(enc, 0, 1, 0, 0)], resamplers=[Resampler(m, 8000)], last=[True])[0]
    plain = m.infer_decoder_batch([(enc, 0, 1, 0, 0)], resamplers=[None])[0]
    np.testing.assert_array_equal(y.as_slice(), _debug_resample(plain.as_slice(), 22050, 8000))
    low = voices("low")
    enc = low.infer_encoder_batch([_ids(150, 4)], seeds=[2])[0]
    got = _f32(_run_stream(low, enc, Resampler(low, 11025)))
    np.testing.assert_array_equal(got, _debug_resample(_f32(_run_stream(low, enc, None)), 16000, 11025))


def test_stream_synthesis_and_realtime_batch(voices):
    m = voices("medium")
    ph = "hɛloʊ wɜːld ðɪs ɪz ə lɔŋ sɛntəns"
    chunks = list(m.stream_synthesis(ph, CS, PAD, seed=4, output_rate=24000))
    enc = m.infer_encoder_batch([m.phonemes_to_input_ids(ph)], seeds=[4])[0]
    np.testing.assert_array_equal(_f32(chunks), _f32(_run_stream(m, enc, Resampler(m, 24000))))
    rb = RealtimeBatch(m, CS, PAD)
    rb.add(ph, seed=4, output_rate=24000)
    items = [a for _ in range(64) if len(rb) for _, a in rb.step()]
    np.testing.assert_array_equal(_f32(items), _f32(chunks))


def test_resampler_misuse_is_an_operation_error(voices):
    m, low = voices("medium"), voices("low")
    enc = m.infer_encoder_batch([_ids(150, 3)], seeds=[5])[0]
    r = Resampler(m, 48000)
    with pytest.raises(OperationError, match="chunk 1.*twice"):
        m.infer_decoder_batch([(enc, 0, 10, 0, 0), (enc, 10, 20, 0, 0)], resamplers=[r, r])
    with pytest.raises(OperationError, match="another voice"):
        m.infer_decoder_batch([(enc, 0, 10, 0, 0)], resamplers=[Resampler(low, 48000)])
    m.infer_decoder_batch([(enc, 0, 10, 0, 0)], resamplers=[r], last=[True])
    with pytest.raises(OperationError, match="flushed"):
        m.infer_decoder_batch([(enc, 10, 20, 0, 0)], resamplers=[r])
    for bad in (12345, 22050):
        with pytest.raises(OperationError):
            h, err = C.c_void_p(), N.sb200_error()
            from sonata_b200.piper import _check
            _check(m._lib.sb200_resampler_create(m._h, bad, C.byref(h), C.byref(err)), err)
    with pytest.raises(OperationError):
        StreamBatch(m, CS, PAD).add("ab", output_rate=44000)
