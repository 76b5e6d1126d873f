"""GPU (-m gpu): live loudness on realtime streams.

The contract (include/sonata_b200.h, sb200_loudness_stream_create): joined, what a metered stream delivers is, bit
for bit, sb200_debug_loudness_stream over the joined chunks the same stream delivers without a meter, however either
is chunked; its readings from 400 ms on are the batch meter's bits; its readings, gains and samples agree with the
float64 reference; streams without a meter keep their bits and launches."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import g711_reference as gr
import loudness_reference as lr
import loudness_stream_reference as lsr
from test_loudness_stream_host import _speechlike
from sonata_b200 import OperationError, voicegen, workload
from sonata_b200 import _native as N
from sonata_b200.piper import (LoudnessStream, PiperSynthesisConfig, SpeechStreamer, StreamBatch, VitsStreamingModel,
                               _stream_prosody, _stream_resampler, _trim_frames)
from sonata_b200.synth import AudioOutputConfig, RealtimeBatch, SonataSpeechSynthesizer

pytestmark = pytest.mark.gpu
f32p = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
f64p = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
DEFAULT = PiperSynthesisConfig(None, 0.667, 1.0, 0.8)
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


def _message(err):
    return C.string_at(err.message).decode() if err.message else ""


def hook(x, lens, rate, target, max_gain_db=20.0):
    """(y, L_1 .. L_M, a_1 .. a_M, clipped) of sb200_debug_loudness_stream over x in chunks of lens."""
    x = np.ascontiguousarray(x, np.float32)
    lens = np.ascontiguousarray(lens, np.uint64)
    assert int(lens.sum()) == len(x)
    M = len(x) // lr.step(rate)
    y, L, a = np.zeros(len(x) + 1, np.float32), np.zeros(M + 1), np.zeros(M + 1, np.float32)
    clipped, err = C.c_int64(), N.sb200_error()
    rc = N.lib().sb200_debug_loudness_stream(0, f32p(x), lens.ctypes.data_as(C.POINTER(C.c_size_t)), len(lens), rate,
                                             target, max_gain_db, f32p(y), f64p(L), f32p(a), C.byref(clipped),
                                             C.byref(err))
    assert rc == 0, _message(err)
    return y[:len(x)], L[:M], a[:M], clipped.value


def batch_lufs(x, rate):
    x = np.ascontiguousarray(x, np.float32)
    out, err = C.c_double(), N.sb200_error()
    rc = N.lib().sb200_debug_loudness(0, f32p(x), len(x), rate, C.byref(out), C.byref(err))
    assert rc == 0, _message(err)
    return out.value


def _signal(rate, seed):
    """Speech-like level changes, a silent gap and a loud burst that the gain drives into the clamp."""
    x = _speechlike(rate, 2.6, seed)
    x[int(0.9 * rate):int(1.2 * rate)] = 0.0
    x[int(2.0 * rate):int(2.1 * rate)] *= 6.0
    return x


def _chunkings(n, S, seed):
    rng = np.random.default_rng(seed)
    out = [[n], [S] * (n // S) + ([n % S] if n % S else [])]
    lens = []
    while sum(lens) < n:
        lens.append(int(rng.choice([1, 2, S - 1, S // 3, S + 1, 2 * S + 5, 7])))
    lens[-1] -= sum(lens) - n
    out.append([c for c in lens if c > 0])
    out.append([1] * 5 + [S - 5] + [3 * S] + [n - 4 * S])
    return out


@pytest.mark.parametrize("rate", lr.RATES)
def test_hook_does_not_depend_on_the_chunking(rate):
    x = _signal(rate, rate)
    S = lr.step(rate)
    runs = [hook(x, lens, rate, -16.0) for lens in _chunkings(len(x), S, rate)]
    for y, L, a, clipped in runs[1:]:
        assert y.tobytes() == runs[0][0].tobytes()
        assert L.tobytes() == runs[0][1].tobytes() and a.tobytes() == runs[0][2].tobytes()
        assert clipped == runs[0][3]


@pytest.mark.parametrize("rate", lr.RATES)
def test_hook_against_the_batch_meter_and_the_reference(rate):
    x = _signal(rate, 100 + rate)
    S = lr.step(rate)
    y, L, a, clipped = hook(x, [len(x)], rate, -16.0)
    for m in range(4, len(L) + 1):
        assert L[m - 1] == batch_lufs(x[:m * S], rate), m      # the batch kernel's bits
    yr, Lr, ar, cr = lsr.meter(x, rate, -16.0)
    fin = np.isfinite(Lr)
    assert np.array_equal(np.isfinite(L), fin)
    np.testing.assert_allclose(L[fin], Lr[fin], rtol=0, atol=1e-6)
    ulps = np.abs(a.view(np.int32).astype(np.int64) - ar.view(np.int32).astype(np.int64))
    assert ulps.max() <= 2
    G = lsr.sample_gains(len(x), np.concatenate([[np.float32(1)], ar]), S)
    v = np.abs(x * G)
    assert np.all(np.abs(y - yr) <= 4 * np.spacing(np.maximum(v, np.float32(1e-30))))
    assert clipped == cr and clipped > 0


def _unmetered(m, enc, cs, pad, output_rate, pitch=None, contour=None, formant=None):
    """The chunks a stream delivers through sb200_decode_chunks_warped without a meter (f32), with its own fresh
    resampler and prosody stream."""
    rs = _stream_resampler(m, output_rate)
    w = _stream_prosody(m, pitch, None, contour, enc, formant)
    st = SpeechStreamer(enc, cs, pad)
    out = []
    while st.chunker.last_end_index is not None:
        (m0, m1), (a0, a1) = next(st.chunker)
        if st.one_shot:
            st.chunker.consume()
            chunk, fade = (enc, 0, enc.num_frames, 0, 0), 0
        else:
            chunk, fade = (enc, m0, enc.num_frames if m1 is None else m1) + _trim_frames(slice(a0, a1)), 42
        out.append(m.infer_decoder_batch([chunk], fade=fade, resamplers=[rs], warps=[w],
                                         last=[st.chunker.last_end_index is None])[0].as_slice())
    return out


def _metered(m, enc, cs, pad, output_rate, meter, pitch=None, contour=None, formant=None, encoding=None, gain=1.0,
             pcm16=False):
    rs = _stream_resampler(m, output_rate)
    w = _stream_prosody(m, pitch, None, contour, enc, formant)
    st = SpeechStreamer(enc, cs, pad, rs, encoding, gain, w, meter)
    if not pcm16:
        return list(st)
    out = []
    while st.chunker.last_end_index is not None:
        (m0, m1), (a0, a1) = next(st.chunker)
        if st.one_shot:
            st.chunker.consume()
            chunk, fade = (enc, 0, enc.num_frames, 0, 0), 0
        else:
            chunk, fade = (enc, m0, enc.num_frames if m1 is None else m1) + _trim_frames(slice(a0, a1)), 42
        out.append(m.infer_decoder_batch([chunk], pcm16=True, fade=fade, resamplers=[rs], warps=[w], meters=[meter],
                                         last=[st.chunker.last_end_index is None])[0])
    return out


def _fixed_i16(y):
    return np.trunc(np.clip(y.astype(np.float32) * np.float32(32767), -32768, 32767)).astype(np.int16)


VARIANTS = [dict(), dict(pitch=1.25), dict(contour=True), dict(formant=1.2)]


@pytest.mark.parametrize("quality", ("medium", "x_low"))
@pytest.mark.parametrize("out_rate", (None, 48000, 8000))
def test_joined_chunks_are_the_hook_over_the_unmetered_stream(voices, quality, out_rate):
    m = voices(quality)
    rate = out_rate or m.audio_output_info().sample_rate
    ids = list(workload.synthetic_ids(160, utt=5))
    enc = m.infer_encoder_batch([ids], seeds=[21])[0]
    for kw in VARIANTS:
        kw = dict(kw)
        if kw.pop("contour", False):
            kw["contour"] = [0.8 + 0.5 * ((i * 7) % 5) / 4 for i in range(len(ids))]
        plain = _unmetered(m, enc, 55, 3, out_rate, **kw)
        meter = LoudnessStream(m, -16.0, output_rate=out_rate)
        got = [c.as_slice() for c in _metered(m, enc, 55, 3, out_rate, meter, **kw)]
        assert [len(c) for c in got] == [len(c) for c in plain], kw
        want = hook(np.concatenate(plain), [len(c) for c in plain], rate, -16.0)
        assert np.concatenate(got).tobytes() == want[0].tobytes(), kw
        st = meter.state()
        assert st["samples"] == len(want[0]) and st["clipped"] == want[3]
        assert st["gain"] == want[2][-1] and st["lufs"] == want[1][-1]
        # i16 at the fixed scale of the metered f32, and G.711 of those samples after the gain
        meter16 = LoudnessStream(m, -16.0, output_rate=out_rate)
        i16 = _metered(m, enc, 55, 3, out_rate, meter16, pcm16=True, **kw)
        assert np.concatenate(i16).tobytes() == _fixed_i16(want[0]).tobytes(), kw
    meter = LoudnessStream(m, -16.0, output_rate=out_rate)
    g = _metered(m, enc, 55, 3, out_rate, meter, encoding="mulaw", gain=0.5)
    plain = _unmetered(m, enc, 55, 3, out_rate)
    y = hook(np.concatenate(plain), [sum(len(c) for c in plain)], rate, -16.0)[0]
    assert b"".join(g) == gr.encode_bytes(_fixed_i16(y * np.float32(0.5)), "mulaw")


def test_stream_batch_and_stream_synthesis_agree(voices):
    m = voices("medium")
    kws = [dict(live_loudness=-16.0), dict(live_loudness=-20.0, output_rate=48000, pitch=1.25),
           dict(live_loudness=-16.0, output_rate=8000, encoding="alaw", gain=0.7), dict(live_loudness=-23.0,
                                                                                          formant_ratio=1.2)]
    sb = StreamBatch(m, 55, 3)
    keys = [sb.add(LONG, seed=40 + i, **kw) for i, kw in enumerate(kws)]
    got = {}
    while len(sb):
        for k, a in sb.step():
            assert not isinstance(a, Exception), a
            got.setdefault(k, []).append(a)
    for i, kw in enumerate(kws):
        want = list(m.stream_synthesis(LONG, 55, 3, seed=40 + i, **kw))
        if isinstance(want[0], bytes):
            assert got[keys[i]] == want
        else:
            assert b"".join(c.as_slice().tobytes() for c in got[keys[i]]) == \
                b"".join(c.as_slice().tobytes() for c in want)


TEXT = "hɛloʊ wɜːld ðɪs ɪz ðə fɜːst wʌn\nænd ə sɛkənd sɛntəns hɪɹ\nðə θɜːd ænd lɑːst sɛntəns ɪz lɔŋɡɚ θæn ðə ʌðɚz"


def test_realtime_request_is_one_meter_across_its_sentences(voices):
    m = voices("medium")
    synth = SonataSpeechSynthesizer(m)
    plain = [c.as_slice() for c in synth.synthesize_streamed(TEXT, None, 55, 3, seed=5, output_rate=16000)]
    metered = [c.as_slice() for c in synth.synthesize_streamed(TEXT, None, 55, 3, seed=5, output_rate=16000,
                                                               live_loudness=-18.0)]
    want = hook(np.concatenate(plain), [len(c) for c in plain], 16000, -18.0)[0]
    assert np.concatenate(metered).tobytes() == want.tobytes()
    # with silence after each sentence: RealtimeBatch equals synthesize_streamed, and the silence is not metered
    oc = AudioOutputConfig(appended_silence_ms=120)
    streamed = [c.as_slice() for c in synth.synthesize_streamed(TEXT, oc, 55, 3, seed=5, output_rate=16000,
                                                                live_loudness=-18.0)]
    rb = RealtimeBatch(m, 55, 3)
    key = rb.add(TEXT, oc, seed=5, output_rate=16000, live_loudness=-18.0)
    batched = []
    while len(rb):
        for k, a in rb.step():
            assert k == key and not isinstance(a, Exception), a
            batched.append(a.as_slice())
    assert np.concatenate(batched).tobytes() == np.concatenate(streamed).tobytes()
    sil = int(0.12 * 16000)
    speech = [c for c in streamed if not (len(c) == sil and not c.any())]
    assert len(streamed) - len(speech) == 3
    assert np.concatenate(speech).tobytes() == want.tobytes()


MIXED = [dict(), dict(live_loudness=-16.0), dict(output_rate=16000), dict(live_loudness=-20.0, output_rate=48000),
         dict(pitch=1.25), dict(live_loudness=-16.0, pitch=1.25, output_rate=8000), dict(encoding="mulaw"),
         dict(live_loudness=-14.0, encoding="alaw", gain=0.5)]


def _drain(sb):
    got = {}
    while len(sb):
        for k, a in sb.step():
            assert not isinstance(a, Exception), a
            got.setdefault(k, []).append(a)
    return got


def _bits(chunks):
    return [c if isinstance(c, bytes) else c.as_slice().tobytes() for c in chunks]


def test_metered_streams_in_a_mixed_batch_equal_themselves_alone(voices):
    m = voices("medium")
    lib = m._lib
    sb = StreamBatch(m, 55, 3)
    keys = [sb.add(LONG, seed=60 + i, **kw) for i, kw in enumerate(MIXED)]
    got = _drain(sb)
    for i, kw in enumerate(MIXED):
        alone = StreamBatch(m, 55, 3)
        k = alone.add(LONG, seed=60 + i, **kw)
        assert _bits(got[keys[i]]) == _bits(_drain(alone)[k]), kw
    # the streams without a meter: the same bits and launches as a batch without any meter.  Every stream is encoded
    # in the first step, so the launches after it are the decoder passes, each group's its own
    def run(kws):
        sb = StreamBatch(m, 55, 3)
        ks = [sb.add(LONG, seed=60 + MIXED.index(kw), **kw) for kw in kws]
        got = {}
        for k, a in sb.step():
            got.setdefault(k, []).append(a)
        l0 = lib.sb200_launch_count()
        for k, a in _drain(sb).items():
            got.setdefault(k, []).extend(a)
        return {MIXED.index(kw): _bits(got[k]) for kw, k in zip(kws, ks)}, lib.sb200_launch_count() - l0
    plain = [kw for kw in MIXED if "live_loudness" not in kw]
    mixed, n_mixed = run(MIXED)
    alone, n_plain = run(plain)
    _, n_metered = run([kw for kw in MIXED if "live_loudness" in kw])
    assert {i: b for i, b in mixed.items() if "live_loudness" not in MIXED[i]} == alone
    assert n_mixed == n_plain + n_metered


def test_misuse_fails_naming_the_chunk_and_leaves_the_meter(voices):
    m = voices("medium")
    ids = list(workload.synthetic_ids(60, utt=2))
    enc = m.infer_encoder_batch([ids], seeds=[3])[0]
    chunk = (enc, 0, enc.num_frames, 0, 0)
    meter = LoudnessStream(m, -16.0)
    m.infer_decoder_batch([chunk], meters=[meter], last=[True])
    before = meter.state()
    with pytest.raises(OperationError, match="chunk 1: the loudness stream of chunk 0 appears twice"):
        m.infer_decoder_batch([chunk, chunk], meters=[meter, meter])
    assert meter.state() == before
    with pytest.raises(OperationError, match="chunk 0: the chunk is delivered at 16000 Hz"):
        m.infer_decoder_batch([chunk], resamplers=[_stream_resampler(m, 16000)], meters=[meter])
    assert meter.state() == before
    other = voices("x_low")
    foreign = LoudnessStream(other, -16.0, output_rate=m.audio_output_info().sample_rate)
    with pytest.raises(OperationError, match="chunk 0: the loudness stream was made for another voice"):
        m.infer_decoder_batch([chunk], meters=[foreign])
    assert foreign.state()["samples"] == 0
    for bad in (dict(target=1.0), dict(target=float("nan")), dict(target=-16.0, max_gain_db=45.0),
                dict(target=-16.0, max_gain_db=float("inf"))):
        with pytest.raises(OperationError):
            LoudnessStream(m, **bad)
    # the C layer's own checks of T and M
    h, err = C.c_void_p(), N.sb200_error()
    assert m._lib.sb200_loudness_stream_create(m._h, 0, 3.0, 20.0, C.byref(h), C.byref(err)) != 0
    assert "target" in _message(err)
    assert m._lib.sb200_loudness_stream_create(m._h, 0, -16.0, -1.0, C.byref(h), C.byref(err)) != 0
    assert "maximum gain" in _message(err)
    # capacity: 2^16 steps
    S = lr.step(16000)
    x = np.zeros((1 << 16) * S + S, np.float32)
    y, L, a, clipped = np.zeros(1, np.float32), np.zeros(1), np.zeros(1, np.float32), C.c_int64()
    lens = np.array([len(x)], np.uint64)
    rc = N.lib().sb200_debug_loudness_stream(0, f32p(x), lens.ctypes.data_as(C.POINTER(C.c_size_t)), 1, 16000,
                                             -16.0, 20.0, f32p(y), f64p(L), f32p(a), C.byref(clipped), C.byref(err))
    assert rc != 0 and "capacity" in _message(err)
    # a StreamBatch refuses a meter that an unfinished stream carries
    sb = StreamBatch(m, 55, 3)
    shared = LoudnessStream(m, -16.0)
    sb.add(LONG, live_loudness=shared)
    with pytest.raises(OperationError, match="stream 1: the LoudnessStream is already carried"):
        sb.add(LONG, live_loudness=shared)
    _drain(sb)
    assert shared.state()["samples"] > 0
