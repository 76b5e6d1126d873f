"""GPU (-m gpu): pitch and tempo on realtime streams.

The contract: the concatenation of a warped stream's chunks equals, bit for bit, sb200_debug_prosody of the
concatenation of the chunks the same stream yields without ratios; with an output rate, sb200_debug_resample of that;
with i16 / G.711, each chunk converted as the resampled route converts its chunks.  Streams sharing a pass equal
themselves alone, plain streams keep their bits, and misuse fails naming the chunk without touching the stream."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import g711_reference as gr
import prosody_reference as pr
import prosody_stream_reference as psr
from sonata_b200 import OperationError, PiperSynthesisConfig, voicegen, workload
from sonata_b200 import _native as N
from sonata_b200.core import AudioSamples
from sonata_b200.piper import (ProsodyStream, Resampler, SpeechStreamer, StreamBatch, VitsStreamingModel,
                               _trim_frames)
from sonata_b200.synth import AudioOutputConfig, RealtimeBatch, SonataSpeechSynthesizer

pytestmark = pytest.mark.gpu

DEFAULT = PiperSynthesisConfig(None, 0.667, 1.0, 0.8)
QUALITIES = ("x_low", "low", "medium", "high")
LONG = "hɛloʊ wɜːld ðɪs ɪz ə lɔŋɡɚ sɛntəns ðæt ɪz spoʊkən ɪn tʃʌŋks ænd ðɛn sʌm moʊr wɜːdz"


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


def _nan(v):
    return float("nan") if v is None else float(v)


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def debug_prosody(x, rate, p, t):
    x = np.ascontiguousarray(x, np.float32)
    pl = pr.plan(rate, len(x), p, t)
    y = np.zeros(pl["n2"] + 1, np.float32)
    off = np.zeros(pl["F"] + 1, np.int32)
    err = N.sb200_error()
    assert N.lib().sb200_debug_prosody(0, _fp(x), x.size, rate, _nan(p), _nan(t), _fp(y), y.size,
                                       off.ctypes.data_as(C.POINTER(C.c_int32)), off.size, None, 0, C.byref(err)) == 0
    return y[:pl["n2"]], off[:pl["F"]]


def debug_stream(x, lens, rate, p, t):
    x = np.ascontiguousarray(x, np.float32)
    lens = np.ascontiguousarray(lens, np.int64)
    pl = pr.plan(rate, len(x), p, t)
    y = np.zeros(pl["n2"] + 1, np.float32)
    got = np.zeros(len(lens), np.int64)
    off = np.zeros(pl["F"] + 1, np.int32)
    err = N.sb200_error()
    rc = N.lib().sb200_debug_prosody_stream(0, _fp(x), lens.ctypes.data_as(C.POINTER(C.c_int64)), len(lens), rate,
                                            _nan(p), _nan(t), _fp(y), y.size,
                                            got.ctypes.data_as(C.POINTER(C.c_int64)),
                                            off.ctypes.data_as(C.POINTER(C.c_int32)), off.size, C.byref(err))
    assert rc == 0, _message(err)
    return y[:pl["n2"]], got, off[:pl["F"]]


def _message(err):
    return C.string_at(err.message).decode() if err.message else ""


def debug_resample(x, in_rate, out_rate):
    x = np.ascontiguousarray(x, np.float32)
    g = np.gcd(in_rate, out_rate)
    y = np.zeros(-(-len(x) * (out_rate // g) // (in_rate // g)), np.float32)
    err = N.sb200_error()
    assert N.lib().sb200_debug_resample(0, _fp(x), x.size, in_rate, out_rate, _fp(y), C.byref(err)) == 0
    return y


def signal(rate, seconds, seed=0):
    rng = np.random.default_rng(seed)
    n = int(rate * seconds)
    t = np.arange(n) / rate
    f0 = 120 + 40 * np.sin(2 * np.pi * 1.3 * t)
    x = 0.4 * np.sin(2 * np.pi * np.cumsum(f0) / rate) + 0.2 * np.sin(2 * np.pi * 3 * np.cumsum(f0) / rate)
    return (x * (0.6 + 0.4 * np.sin(2 * np.pi * 0.7 * t)) + 0.02 * rng.standard_normal(n)).astype(np.float32)


RAW = [(0.5, 0.25), (2.0, 4.0), (0.5, 4.0), (1.25, 1.25), (1.25, None), (None, 1.5), (0.8, 2.0)]


@pytest.mark.parametrize("rate", (22050, 16000))
@pytest.mark.parametrize("p,t", RAW)
def test_raw_push_equals_the_whole_signal(lib_built, rate, p, t):
    x = signal(rate, 1.0, seed=rate)
    want, want_off = debug_prosody(x, rate, p, t)
    pl = pr.plan(rate, len(x), p, t)
    ref_off = pr.offsets(x, pl) if pl["stretch"] else np.zeros(0, np.int64)
    np.testing.assert_array_equal(want_off, ref_off)
    for name, lens in psr.chunkings(len(x), rate).items():
        y, got, off = debug_stream(x, lens, rate, p, t)
        np.testing.assert_array_equal(got, [r["emitted"] for r in psr.stream(rate, p, t, lens)], err_msg=name)
        assert y.tobytes() == want.tobytes(), name
        np.testing.assert_array_equal(off, ref_off, err_msg=name)


@pytest.mark.parametrize("p,t", [(0.5, 4.0), (2.0, 0.25), (1.25, None), (0.8, 0.8)])
def test_raw_push_single_samples(lib_built, p, t):
    rate = 16000
    x = signal(rate, 0.3, seed=3)
    want, _ = debug_prosody(x, rate, p, t)
    y, _, _ = debug_stream(x, [1] * len(x), rate, p, t)
    assert y.tobytes() == want.tobytes()


def _streamer(m, ids, seed, cs, pad, **kw):
    enc = m.infer_encoder_batch([ids], seeds=[seed])[0]
    return SpeechStreamer(enc, cs, pad, **kw)


def _cat(chunks):
    return np.concatenate([c.as_slice() for c in chunks]) if chunks else np.zeros(0, np.float32)


def _schedule(enc, cs, pad):
    """SpeechStreamer's chunks of a latent: (chunk tuple with trims, fade, last)."""
    st = SpeechStreamer(enc, cs, pad)
    out = []
    while st.chunker.last_end_index is not None:
        (m0, m1), (a0, a1) = next(st.chunker)
        if st.one_shot:
            st.chunker.consume()
            out.append(((enc, 0, enc.num_frames, 0, 0), 0, True))
            break
        hi = enc.num_frames if m1 is None else m1
        out.append(((enc, m0, hi) + _trim_frames(slice(a0, a1)), 42, st.chunker.last_end_index is None))
    return out


def _plain(m, enc, cs, pad):
    """The chunks the stream yields without ratios, after the device post-path (trims, crossfade(42)) that a warped
    stream's chunks go through: its fade table is the library's, which may differ from the host crossfade's by an
    ulp on the faded samples."""
    return [m.infer_decoder_batch([c], fade=f, resamplers=[None], last=[last])[0] for c, f, last in _schedule(enc, cs, pad)]


@pytest.mark.parametrize("quality", QUALITIES)
@pytest.mark.parametrize("cs,pad", [(55, 3), (72, 3), (4000, 3)])
def test_stream_equals_whole_on_every_voice(voices, quality, cs, pad):
    m = voices(quality)
    rate = m.audio_output_info().sample_rate
    ids = list(workload.synthetic_ids(120, utt=7))
    plain = _cat(_plain(m, m.infer_encoder_batch([ids], seeds=[9])[0], cs, pad))
    for p, t in ((1.25, None), (None, 1.5), (0.8, 2.0)):
        warped = list(_streamer(m, ids, 9, cs, pad, warp=ProsodyStream(m, p, t)))
        assert _cat(warped).tobytes() == debug_prosody(plain, rate, p, t)[0].tobytes(), (p, t)
    # stream_synthesis builds the same streamer
    enc = m.infer_encoder_batch([m.phonemes_to_input_ids(LONG)], seeds=[4])[0]
    a = _cat(_plain(m, enc, cs, pad))
    b = _cat(list(m.stream_synthesis(LONG, cs, pad, seed=4, pitch=1.25, tempo=0.8)))
    assert b.tobytes() == debug_prosody(a, rate, 1.25, 0.8)[0].tobytes()
    # the plain stream_synthesis (crossfade on the host, another sine) differs from the device post-path's chunks by a
    # few ulps at most, and only on faded samples
    c = _cat(list(m.stream_synthesis(LONG, cs, pad, seed=4)))
    assert len(c) == len(a)
    diff = np.abs(c.astype(np.float64) - a.astype(np.float64))
    assert np.all(diff <= 4 * 2.0 ** -23 * np.abs(a.astype(np.float64)))
    assert int(np.count_nonzero(diff)) <= 2 * 42 * len(_schedule(enc, cs, pad))


def test_composition_with_rates_i16_and_g711(voices):
    m = voices("medium")
    rate = m.audio_output_info().sample_rate
    ids = list(workload.synthetic_ids(150, utt=3))
    enc = m.infer_encoder_batch([ids], seeds=[5])[0]
    plain = _cat(_plain(m, enc, 55, 3))
    warped_f32 = list(_streamer(m, ids, 5, 55, 3, warp=ProsodyStream(m, 1.25, None)))
    whole = debug_prosody(plain, rate, 1.25, None)[0]
    assert _cat(warped_f32).tobytes() == whole.tobytes()
    for out_rate in (16000, 48000, 8000):
        rs = list(_streamer(m, ids, 5, 55, 3, warp=ProsodyStream(m, 1.25, None), resampler=Resampler(m, out_rate)))
        assert _cat(rs).tobytes() == debug_resample(whole, rate, out_rate).tobytes(), out_rate
    # i16: to_i16_vec of each emitted f32 chunk
    w = ProsodyStream(m, 1.25, None)
    got = [m.infer_decoder_batch([c], fade=f, pcm16=True, warps=[w], last=[last])[0]
           for c, f, last in _schedule(enc, 55, 3)]
    assert len(got) == len(warped_f32)
    for g, f in zip(got, warped_f32):
        np.testing.assert_array_equal(g, AudioSamples(f.as_slice()).to_i16_vec())
    # G.711 with a gain: the gain scales the warped samples before their conversion
    for law in ("mulaw", "alaw"):
        g711 = list(_streamer(m, ids, 5, 55, 3, warp=ProsodyStream(m, 1.25, None), encoding=law, gain=0.3))
        assert len(g711) == len(warped_f32)
        for g, f in zip(g711, warped_f32):
            assert g == gr.encode_bytes(AudioSamples(f.as_slice() * np.float32(0.3)).to_i16_vec(), law)


SHORT = "ænd ə sɛkənd wʌn"
# (phonemes, stream kinds): plain, resampled, encoded and warped streams with different ratios, long and one-shot
MIXED = [(LONG, dict()), (LONG, dict(output_rate=16000)), (SHORT, dict(encoding="mulaw", gain=0.5)),
         (LONG, dict(pitch=1.25)), (LONG, dict(tempo=1.5, output_rate=8000)), (SHORT, dict(pitch=0.8, tempo=2.0)),
         (LONG, dict(pitch=2.0, tempo=0.5, encoding="alaw", gain=0.7)), (SHORT, dict(tempo=0.8, encoding="mulaw"))]


def _drain(sb):
    got = {}
    while len(sb):
        for k, a in sb.step():
            assert not isinstance(a, Exception), a
            got.setdefault(k, []).append(a)
    return got


def _same(a, b):
    if isinstance(a[0], bytes):
        return a == b
    return len(a) == len(b) and all(x.as_slice().tobytes() == y.as_slice().tobytes() for x, y in zip(a, b))


def test_mixed_stream_batch(voices):
    m = voices("medium")
    sb = StreamBatch(m, 40, 3)
    keys = [sb.add(ph, seed=10 + i, **kw) for i, (ph, kw) in enumerate(MIXED)]
    got = _drain(sb)
    # each stream equals its stream_synthesis alone, chunk for chunk
    for i, (ph, kw) in enumerate(MIXED):
        want = list(m.stream_synthesis(ph, 40, 3, seed=10 + i, **kw))
        assert _same(got[keys[i]], want), (i, kw)
    # the unwarped streams keep their bits without the warped ones
    sb = StreamBatch(m, 40, 3)
    plain = [i for i, (_, kw) in enumerate(MIXED) if "pitch" not in kw and "tempo" not in kw]
    keys2 = [sb.add(MIXED[i][0], seed=10 + i, **MIXED[i][1]) for i in plain]
    got2 = _drain(sb)
    for i, k2 in zip(plain, keys2):
        assert _same(got[keys[i]], got2[k2]), i


def test_one_shot_encoded_warped_stream_is_flushed(voices):
    """A one-shot sentence whose frames lie past chunk + padding + 44 (the chunker's first window) but within the
    one-shot limit: its only chunk ends the stream, encoded or not, with or without an output rate."""
    m = voices("medium")
    rate = m.audio_output_info().sample_rate
    ids = m.phonemes_to_input_ids(LONG)
    enc = m.infer_encoder_batch([ids], seeds=[3])[0]
    pad = 3
    cs = enc.num_frames - pad - 45              # num_frames in (cs + pad + 44, 2 cs + 2 pad]
    assert cs + pad + 44 < enc.num_frames <= 2 * cs + 2 * pad
    plain = _cat(_plain(m, enc, cs, pad))
    whole = debug_prosody(plain, rate, 1.25, 0.8)[0]
    f32 = list(m.stream_synthesis(LONG, cs, pad, seed=3, pitch=1.25, tempo=0.8))
    assert len(f32) == 1 and f32[0].as_slice().tobytes() == whole.tobytes()
    for out_rate in (None, 16000):
        ref = whole if out_rate is None else debug_resample(whole, rate, out_rate)
        for law in ("mulaw", "alaw"):
            g = list(m.stream_synthesis(LONG, cs, pad, seed=3, pitch=1.25, tempo=0.8, output_rate=out_rate,
                                        encoding=law, gain=0.5))
            assert len(g) == 1 and len(g[0]) == len(ref), (out_rate, law)
            assert g[0] == gr.encode_bytes(AudioSamples(ref * np.float32(0.5)).to_i16_vec(), law), (out_rate, law)


def test_realtime_batch_equals_synthesize_streamed(voices):
    m = voices("medium")
    synth = SonataSpeechSynthesizer(m)
    text = LONG + "\n" + "ænd ə sɛkənd wʌn" + "\n" + LONG
    oc = AudioOutputConfig(None, 80, None, 30)
    for kw in (dict(pitch_ratio=1.25), dict(tempo=0.75, output_rate=16000), dict(pitch_ratio=0.8, tempo=2.0)):
        st = list(synth.synthesize_streamed(text, oc, 30, 3, seed=6, **kw))
        rb = RealtimeBatch(m, 30, 3)
        k = rb.add(text, oc, seed=6, **kw)
        other = rb.add(text, oc, seed=6)
        items = {k: [], other: []}
        while len(rb):
            for key, c in rb.step():
                assert not isinstance(c, Exception), c
                items[key].append(c)
        assert len(items[k]) == len(st), kw
        for a, b in zip(items[k], st):
            assert a.as_slice().tobytes() == b.as_slice().tobytes(), kw


def test_misuse_names_the_chunk_and_keeps_the_stream(voices):
    m = voices("medium")
    rate = m.audio_output_info().sample_rate
    ids = list(workload.synthetic_ids(150, utt=3))
    enc = m.infer_encoder_batch([ids], seeds=[5])[0]
    chunks = [(enc, 0, 40, 0, 3), (enc, 37, 80, 3, 3), (enc, 77, enc.num_frames, 3, 0)]
    w = ProsodyStream(m, None, 1.5)
    out = [m.infer_decoder_batch([chunks[0]], fade=42, warps=[w], last=[False])[0]]
    with pytest.raises(OperationError, match="chunk 1: the prosody stream of chunk 0 appears twice"):
        m.infer_decoder_batch([chunks[1], chunks[1]], fade=42, warps=[w, w], last=[False, False])
    other = voices("low")
    wo = ProsodyStream(other, None, 1.5)
    with pytest.raises(OperationError, match="chunk 0: the prosody stream was made for another voice"):
        m.infer_decoder_batch([chunks[1]], fade=42, warps=[wo])
    out.append(m.infer_decoder_batch([chunks[1]], fade=42, warps=[w], last=[False])[0])
    out.append(m.infer_decoder_batch([chunks[2]], fade=42, warps=[w], last=[True])[0])
    with pytest.raises(OperationError, match="chunk 0: the prosody stream has already been flushed"):
        m.infer_decoder_batch([chunks[2]], fade=42, warps=[w], last=[True])
    plain = m.infer_decoder_batch(chunks, fade=42, resamplers=[None] * 3)
    assert _cat(out).tobytes() == debug_prosody(_cat(plain), rate, None, 1.5)[0].tobytes()
    # a last flag other than 0 / 1 (reachable through the C ABI only) names the chunk and leaves the stream as it was
    w2 = ProsodyStream(m, 1.25, None)
    lo, hi = np.array([0], np.int64), np.array([40], np.int64)
    tlo, thi = np.array([0], np.int64), np.array([3], np.int64)
    p64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))
    outs, lens, err = (C.c_void_p * 1)(), (C.c_size_t * 1)(), N.sb200_error()
    rc = N.lib().sb200_decode_chunks_warped(m._h, (C.c_void_p * 1)(enc._h.value), p64(lo), p64(hi), p64(tlo), p64(thi),
                                            1, 42, None, (C.c_void_p * 1)(None), (C.c_void_p * 1)(w2._h.value),
                                            (C.c_int32 * 1)(2), 0, outs, lens, C.byref(err))
    assert rc == 19 and "chunk 0: last flag 2 is neither 0 nor 1" in _message(err)
    out2 = [m.infer_decoder_batch([c], fade=42, warps=[w2], last=[k == 2])[0] for k, c in enumerate(chunks)]
    assert _cat(out2).tobytes() == debug_prosody(_cat(plain), rate, 1.25, None)[0].tobytes()
    with pytest.raises(OperationError):
        ProsodyStream(m, 1.0, None)
    with pytest.raises(OperationError, match="pitch ratio 3.0"):
        ProsodyStream(m, 3.0, None)


def test_no_warps_is_the_resampled_call(voices):
    m = voices("medium")
    ids = list(workload.synthetic_ids(80, utt=2))
    enc = m.infer_encoder_batch([ids], seeds=[8])[0]
    chunks = [(enc, 0, 40, 0, 3), (enc, 37, enc.num_frames, 3, 0)]
    lib = N.lib()
    n0 = lib.sb200_launch_count()
    a = m.infer_decoder_batch(chunks, fade=42, resamplers=[None, Resampler(m, 16000)], last=[False, True])
    n1 = lib.sb200_launch_count()
    b = m.infer_decoder_batch(chunks, fade=42, resamplers=[None, Resampler(m, 16000)], last=[False, True],
                              warps=[None, None])
    n2 = lib.sb200_launch_count()
    assert n2 - n1 == n1 - n0
    assert _cat(a).tobytes() == _cat(b).tobytes()
