"""CPU: StreamBatch and RealtimeBatch against SpeechStreamer and synthesize_streamed on a fake model.

The fake's decoder output encodes (latent, frame, sample), so any chunk taken from the wrong latent, the wrong frames,
with the wrong trim or without its crossfade differs.  The fake also logs every encoder and decoder call, which shows
how the schedulers batch."""
import ctypes as C

import numpy as np
import pytest

from sonata_b200 import (AudioInfo, AudioOutputConfig, AudioSamples, OperationError, PiperSynthesisConfig, RealtimeBatch,
                         SonataError, SpeechStreamer, StreamBatch, SonataSpeechSynthesizer, VitsStreamingModel)
from sonata_b200.piper import HOP, MAX_CHUNK_SIZE, EncoderOutputs
from sonata_b200.synth import next_chunk_size


POISON_ENCODE, POISON_DECODE = 999, 998     # ids the fake's encoder, or decoder, fails on (as the library can)


class FakeEnc:
    def __init__(self, m, ids, cfg):
        self._m = m
        self.bad_decode = POISON_DECODE in ids
        self.tag = (sum(ids) * 31 + len(ids) * 7 + (cfg.speaker or 0) * 1009) % 9973
        self.num_frames = max(1, int(round(len(ids) * 3 * cfg.length_scale)))

    def wave(self, lo, hi):
        f = np.arange(lo, hi, dtype=np.float64)[:, None]
        j = np.arange(HOP, dtype=np.float64)[None, :]
        return (0.5 * np.sin(self.tag * 0.37 + f * 0.11 + j * 0.013) + 0.001 * self.tag).astype(np.float32).reshape(-1)

    def infer_decoder(self, lo=0, hi=None):
        return AudioSamples(self.wave(lo, self.num_frames if hi is None else hi))


class FakeModel:
    def __init__(self):
        self.fallback = PiperSynthesisConfig()
        self.log = []

    def audio_output_info(self):
        return AudioInfo(22050, 1, 2)

    def phonemize_text(self, text):
        raise SonataError("no phonemizer")

    def phonemes_to_input_ids(self, ph):
        return [POISON_ENCODE if c == "~" else ord(c) % 50 + 1 for c in ph]

    def get_speakers(self):
        return {0: "a", 1: "b", 2: "c", 3: "d"}

    def _encode(self, ids, cfg, who):
        if (cfg.speaker or 0) not in self.get_speakers():
            raise OperationError(f"Failed to run model inference. Error: speaker id out of range ({who})")
        if POISON_ENCODE in ids:
            raise OperationError(f"Failed to run model inference. Error: predicted durations are unreasonably long ({who})")
        return FakeEnc(self, ids, cfg)

    def get_fallback_synthesis_config(self):
        return self.fallback

    def set_fallback_synthesis_config(self, cfg):
        self.fallback = cfg

    def infer_encoder(self, ids):
        return self._encode(ids, self.fallback, "utterance 0")

    def stream_synthesis(self, phonemes, chunk_size, chunk_padding):
        return SpeechStreamer(self.infer_encoder(self.phonemes_to_input_ids(phonemes)), chunk_size, chunk_padding)

    def infer_encoder_batch(self, batches, configs=None):
        self.log.append(("enc", len(batches)))
        configs = configs or [self.fallback] * len(batches)
        return [self._encode(ids, c, f"utterance {i}") for i, (ids, c) in enumerate(zip(batches, configs))]

    def infer_decoder_batch(self, chunks, pcm16=False):
        self.log.append(("dec", [(c[0].tag, c[1], c[2]) for c in chunks]))
        for k, c in enumerate(chunks):
            if c[0].bad_decode:
                raise OperationError(f"chunk {k}: decoder failed")
        return [AudioSamples(c[0].wave(c[1], c[2])) for c in chunks]


def _ids(n, seed):
    return [int(x) for x in np.random.default_rng(seed).integers(1, 60, n)]


def _alone(m, ids, cfg, chunk_size, pad):
    saved = m.fallback
    m.fallback = cfg or saved
    out = [a.as_slice().copy() for a in SpeechStreamer(m.infer_encoder(ids), chunk_size, pad)]
    m.fallback = saved
    return out


def _drain(batch, got, admissions=None):
    step = 0
    while len(batch) or admissions:
        for fn in (admissions or {}).pop(step, []):
            fn()
        for key, a in batch.step():
            got.setdefault(key, []).append(a.as_slice().copy())
        step += 1
    return step


def _same(a, b):
    return len(a) == len(b) and all(x.shape == y.shape and np.array_equal(x, y) for x, y in zip(a, b))


def test_stream_batch_equals_speech_streamer_per_stream():
    m = FakeModel()
    cs, pad = 55, 3
    # frames = 3 * len * length_scale: one-shot (<= 116), a few chunks, many chunks up to the 1024 cap
    cases = [(10, None), (38, None), (39, PiperSynthesisConfig(2, 0.667, 1.0, 0.8)), (120, PiperSynthesisConfig(1)),
             (256, None), (700, PiperSynthesisConfig(None, 0.667, 1.7, 0.8)), (5, PiperSynthesisConfig(3)),
             (256, PiperSynthesisConfig(0, 0.0, 0.8, 0.0))]
    sb = StreamBatch(m, cs, pad)
    keys, expect, got = {}, {}, {}

    def admit(i):
        def f():
            n, cfg = cases[i]
            ids = _ids(n, i)
            keys[i] = sb.add(ids, cfg)
            expect[keys[i]] = _alone(m, ids, cfg, cs, pad)
        return f
    # staggered: three at t=0, then streams join while others are mid-way
    _drain(sb, got, {0: [admit(0), admit(1), admit(2)], 1: [admit(3)], 2: [admit(4), admit(5)], 5: [admit(6)],
                     6: [admit(7)]})
    assert set(got) == set(expect)
    for k in expect:
        assert _same(got[k], expect[k]), k
    assert len(expect[keys[0]]) == 1 and len(expect[keys[6]]) == 1            # one-shot streams


def test_stream_batch_calls_one_encoder_and_one_decoder_pass_per_step():
    m = FakeModel()
    sb = StreamBatch(m, 20, 2)
    for i, n in enumerate((30, 60, 8)):
        sb.add(_ids(n, 10 + i))
    active = 3
    sb.step()
    assert m.log == [("enc", 3), ("dec", m.log[1][1])] and len(m.log[1][1]) == active
    m.log.clear()
    sb.add(_ids(45, 20))
    sb.add("hello world")
    out = sb.step()
    kinds = [e[0] for e in m.log]
    assert kinds == ["enc", "dec"] and m.log[0][1] == 2
    assert len(m.log[1][1]) == len(out) == 4            # the one-shot stream finished in step 1; 2 old + 2 new
    while len(sb):
        m.log.clear()
        out = sb.step()
        assert [e[0] for e in m.log] == ["dec"] and len(m.log[0][1]) == len(out)
    m.log.clear()
    assert sb.step() == [] and m.log == []


def test_stream_batch_reaches_the_chunk_cap():
    m = FakeModel()
    cs, pad = 600, 3
    ids = _ids(1500, 3)                                   # 4500 frames: the second chunk asks for 1200 > 1024
    sb = StreamBatch(m, cs, pad)
    k = sb.add(ids)
    got = {}
    _drain(sb, got)
    assert _same(got[k], _alone(m, ids, None, cs, pad))
    lens = [hi - lo for _, chunks in m.log[1:] for _, lo, hi in chunks]
    assert max(lens) == MAX_CHUNK_SIZE + 3 * pad and len(lens) >= 3


def test_realtime_batch_equals_synthesize_streamed():
    m = FakeModel()
    texts = ["abcdefghij" * 4 + "\n" + "klmnop" * 9 + "\n" + "qr" * 30,
             "short",
             "x" * 40 + "\n" + "yz" * 25,
             "a" * 90 + "\n\n" + "b" * 12 + "\n" + "c" * 70]
    ocs = [None, AudioOutputConfig(volume=40), AudioOutputConfig(appended_silence_ms=120),
           AudioOutputConfig(volume=75, appended_silence_ms=30)]
    cfgs = [None, PiperSynthesisConfig(1, 0.667, 1.2, 0.8), None, PiperSynthesisConfig(2, 0.0, 0.9, 0.0)]
    syn = SonataSpeechSynthesizer(m)
    expect = []
    for t, oc, cfg in zip(texts, ocs, cfgs):
        m.fallback = cfg or PiperSynthesisConfig()
        expect.append([a.as_slice().copy() for a in syn.synthesize_streamed(t, oc, 24, 3)])
    m.fallback = PiperSynthesisConfig()
    rb = RealtimeBatch(m, 24, 3)
    got = {}
    keys = [rb.add(texts[0], ocs[0], cfgs[0]), rb.add(texts[1], ocs[1], cfgs[1])]
    step = 0
    while len(rb) or step < 3:
        if step == 2:
            keys += [rb.add(texts[2], ocs[2], cfgs[2]), rb.add(texts[3], ocs[3], cfgs[3])]
        for key, a in rb.step():
            got.setdefault(key, []).append(a.as_slice().copy())
        step += 1
    for k, e in zip(keys, expect):
        assert _same(got[k], e), k
    # the growth rule really applied: a later sentence of text 0 used a larger chunk size than 24
    assert next_chunk_size(24, 0) == 24 and next_chunk_size(24, 3) == 72
    assert max(hi - lo for e in m.log if e[0] == "dec" for _, lo, hi in e[1]) > 24 + 2 * 3 * 2


def test_argument_errors_before_any_native_call():
    m = FakeModel()
    with pytest.raises(OperationError):
        StreamBatch(m, 0, 3)
    with pytest.raises(OperationError):
        StreamBatch(m, 55, -1)
    sb = StreamBatch(m, 55, 3)
    with pytest.raises(OperationError):
        sb.add([1, 2, 3], config={"speaker": 1})
    with pytest.raises(OperationError):
        sb.add([])
    rb = RealtimeBatch(m)
    with pytest.raises(OperationError):
        rb.add("abc", AudioOutputConfig(rate=80))
    with pytest.raises(OperationError):
        rb.add("abc", None, config=3)
    assert m.log == [] and len(sb) == 0 and len(rb) == 0

    class Recorder:
        def __init__(self):
            self.calls = []

        def __getattr__(self, name):
            return lambda *a: self.calls.append(name) or 0

    def model():
        v = VitsStreamingModel.__new__(VitsStreamingModel)
        v._lib, v._h = Recorder(), C.c_void_p(1)
        return v
    a, b = model(), model()
    enc = EncoderOutputs.__new__(EncoderOutputs)
    enc._m, enc._h, enc.num_frames = b, C.c_void_p(8), 100
    with pytest.raises(OperationError, match="chunk 0"):
        a.infer_decoder_batch([(enc, 0, 10)])
    with pytest.raises(OperationError, match="chunk 0"):
        a.infer_decoder_batch([(enc, 0, 10, 1, 1)])                # trims need pcm16
    enc._m = a
    with pytest.raises(OperationError):
        a.infer_decoder_batch([(enc, 0, 10)], pcm16=True, gains=[1.0, 2.0])
    with pytest.raises(OperationError):
        a.infer_encoder_batch([[1, 2], [3]], [PiperSynthesisConfig()])
    with pytest.raises(OperationError):
        a.infer_encoder_batch([[1, 2], []])
    assert a.infer_encoder_batch([]) == [] and a.infer_decoder_batch([]) == []
    assert a._lib.calls == [] and b._lib.calls == []
    enc._h = None


def test_one_stream_failure_stays_that_streams():
    """A stream whose encoder or decoder work fails gets its error once and ends; every other stream, admitted with it
    or before it, still yields exactly its SpeechStreamer chunks, and later steps run normally."""
    m = FakeModel()
    sb = StreamBatch(m, 55, 3)
    with pytest.raises(OperationError, match="No speaker"):
        sb.add(_ids(40, 1), PiperSynthesisConfig(9))                 # refused at admission
    assert len(sb) == 0 and m.log == []
    good = {sb.add(ids, cfg): (ids, cfg) for ids, cfg in ((_ids(120, 30), None), (_ids(40, 31), PiperSynthesisConfig(2)))}
    got = {}
    for key, a in sb.step():
        got.setdefault(key, []).append(a)
    bad_enc = sb.add(_ids(60, 32) + [POISON_ENCODE])
    bad_dec = sb.add(_ids(90, 33) + [POISON_DECODE], PiperSynthesisConfig(1))
    more = sb.add(_ids(200, 34), PiperSynthesisConfig(3))
    good[more] = (_ids(200, 34), PiperSynthesisConfig(3))
    while len(sb):
        for key, a in sb.step():
            got.setdefault(key, []).append(a)
    for key in (bad_enc, bad_dec):
        assert len(got[key]) == 1 and isinstance(got[key][0], SonataError), key
    assert "durations" in str(got[bad_enc][0]) and "decoder failed" in str(got[bad_dec][0])
    for key, (ids, cfg) in good.items():
        assert all(isinstance(a, AudioSamples) for a in got[key])
        assert _same([a.as_slice() for a in got[key]], _alone(m, ids, cfg, 55, 3)), key
    assert sb.step() == []


def test_realtime_request_failure_stays_that_requests():
    m = FakeModel()
    texts = ["abcdefghij" * 5 + "\n" + "klm~no" * 6 + "\n" + "qr" * 30,      # the second sentence cannot be encoded
             "x" * 45 + "\n" + "yz" * 40]
    ocs = [AudioOutputConfig(appended_silence_ms=20), AudioOutputConfig(volume=50)]
    syn = SonataSpeechSynthesizer(m)
    expect = []
    for t, oc in zip(texts, ocs):
        items, err = [], None
        try:
            for a in syn.synthesize_streamed(t, oc, 24, 3):
                items.append(a.as_slice().copy())
        except SonataError as e:
            err = e
        expect.append((items, err))
    assert expect[0][1] is not None and expect[1][1] is None
    rb = RealtimeBatch(m, 24, 3)
    with pytest.raises(OperationError, match="No speaker"):
        rb.add("abc", None, PiperSynthesisConfig(7))
    keys = [rb.add(t, oc) for t, oc in zip(texts, ocs)]
    got = {}
    while len(rb):
        for key, a in rb.step():
            got.setdefault(key, []).append(a)
    bad = got[keys[0]]
    assert isinstance(bad[-1], SonataError) and not any(isinstance(a, SonataError) for a in bad[:-1])
    assert _same([a.as_slice() for a in bad[:-1]], expect[0][0])
    assert _same([a.as_slice() for a in got[keys[1]]], expect[1][0])
