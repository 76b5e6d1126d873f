"""GPU (-m gpu): many realtime streams in one encoder pass and one decoder pass per step.

Every comparison is bit for bit against the same work done one stream at a time: a latent of a batched encoder pass
against `infer_encoder` alone with its config as the fallback (zero noise, so the Philox draws' batch position plays no
part), a chunk of a batched decoder pass against `infer_decoder(lo, hi)` alone, and the schedulers against
`stream_synthesis` / `synthesize_streamed`."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from sonata_b200 import (AudioOutputConfig, AudioSamples, OperationError, PiperSynthesisConfig, RealtimeBatch,
                         SonataSpeechSynthesizer, SpeechStreamer, StreamBatch, VitsStreamingModel, voicegen, workload)
from sonata_b200.piper import AdaptiveMelChunker, HOP

pytestmark = pytest.mark.gpu

LENS = [1, 7, 64, 65, 130, 513, 33, 200, 2, 97, 300, 16]
SPEAKERS = [0, 3, 1, 3, None, 2, 0, None, 1, 2, 3, 0]
LENGTH_SCALES = (0.7, 1.0, 1.3)
ZERO = dict(noise_scale=0.0, noise_w=0.0)


def _ids(n, utt):
    return [int(i) for i in workload.synthetic_ids(n // 2 + 1, utt=utt)[:n]]


def _spk(s, n_speakers):
    return None if (s is None or n_speakers <= 1) else s % n_speakers


@pytest.fixture(scope="module")
def voices(lib_built):
    d = voicegen.default_voice_dir()
    paths = {"medium4": voicegen.write_voice(d, "medium", n_speakers=4),
             "high3": voicegen.write_voice(d, "high", n_speakers=3),
             "x_low3": voicegen.write_voice(d, "x_low", n_speakers=3),
             "medium": voicegen.write_voice(d, "medium"),
             "x_low": voicegen.write_voice(d, "x_low")}
    ms = {}

    def get(name):
        if name not in ms:
            ms[name] = VitsStreamingModel(paths[name], device=0)
        return ms[name]
    get.paths = paths
    yield get
    for m in ms.values():
        m.close()


def _set_fallback(m, cfg):
    """A batch entry without a speaker means speaker 0; a fallback set without one keeps the previous speaker."""
    if cfg.speaker is None and m.get_speakers():
        cfg = PiperSynthesisConfig(0, cfg.noise_scale, cfg.length_scale, cfg.noise_w)
    m.set_fallback_synthesis_config(cfg)


def _alone_latent(m, ids, cfg):
    saved = m.get_fallback_synthesis_config()
    _set_fallback(m, cfg)
    try:
        return m.infer_encoder(ids)
    finally:
        m.set_fallback_synthesis_config(saved)


def _eq(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a, b)


@pytest.mark.parametrize("voice,backend", [("medium4", 1), ("medium4", 0), ("medium4", 2), ("high3", 1), ("high3", 0),
                                           ("x_low3", 1), ("x_low3", 0)])
def test_batched_encode_equals_each_alone(voices, voice, backend):
    m = voices(voice)
    n_spk = int(voice[-1])
    m.set_backend(backend)
    try:
        batches = [_ids(n, 40 + i) for i, n in enumerate(LENS)]
        cfgs = [PiperSynthesisConfig(_spk(SPEAKERS[b], n_spk), length_scale=LENGTH_SCALES[b % 3], **ZERO)
                for b in range(len(LENS))]
        encs = m.infer_encoder_batch(batches, cfgs)
        for b, (ids, cfg) in enumerate(zip(batches, cfgs)):
            ref = _alone_latent(m, ids, cfg)
            assert encs[b].num_frames == ref.num_frames, (b, cfg)
            assert _eq(encs[b].infer_decoder().as_slice(), ref.infer_decoder().as_slice()), (b, cfg)
        # freed in any order: the shared allocation lives until the last latent goes
        for b in (3, 0, 11, 5):
            encs[b] = None
        assert _eq(encs[1].infer_decoder().as_slice(), _alone_latent(m, batches[1], cfgs[1]).infer_decoder().as_slice())
    finally:
        m.set_backend(1)


def test_zero_noise_utterances_unaffected_by_noisy_neighbours(voices):
    m = voices("medium4")
    batches = [_ids(n, 60 + i) for i, n in enumerate(LENS)]
    cfgs = [PiperSynthesisConfig(_spk(SPEAKERS[b], 4), 0.667 if b % 2 else 0.0, LENGTH_SCALES[b % 3],
                                 0.8 if b % 2 else 0.0) for b in range(len(LENS))]
    encs = m.infer_encoder_batch(batches, cfgs)
    for b in range(0, len(LENS), 2):
        ref = _alone_latent(m, batches[b], cfgs[b])
        assert encs[b].num_frames == ref.num_frames
        assert _eq(encs[b].infer_decoder().as_slice(), ref.infer_decoder().as_slice()), b


def _chunk_latents(m):
    """Nine latents of four speakers; the last is longer than 1024 frames."""
    lens = [60, 90, 75, 120, 66, 80, 100, 70, 520]
    batches = [_ids(n, 80 + i) for i, n in enumerate(lens)]
    cfgs = [PiperSynthesisConfig(i % 4, length_scale=1.6 if i == 8 else 1.0, **ZERO) for i in range(len(lens))]
    encs = m.infer_encoder_batch(batches, cfgs)
    assert encs[8].num_frames > 1100 and all(e.num_frames >= 160 for e in encs)
    return encs


def _chunk_set(encs):
    f = [e.num_frames for e in encs]
    return [(encs[0], 0, 1), (encs[1], 5, 133), (encs[2], 0, 129), (encs[3], f[3] - 129, f[3]),
            (encs[8], 0, 1100), (encs[5], f[5] - 1, f[5]), (encs[6], 10, 80), (encs[6], 60, 150),
            (encs[7], 3, 60), (encs[4], 0, f[4]), (encs[8], f[8] - 1030, f[8])]


def test_batched_decode_equals_each_chunk_alone(voices):
    m = voices("medium4")
    encs = _chunk_latents(m)
    chunks = _chunk_set(encs)
    got = m.infer_decoder_batch(chunks)
    assert len(got) == len(chunks)
    for k, (e, lo, hi) in enumerate(chunks):
        ref = e.infer_decoder(lo, hi).as_slice()
        assert ref.shape == ((hi - lo) * HOP,) and _eq(got[k].as_slice(), ref), (k, lo, hi)
    # alone through the batch entry point, and an empty pass
    assert _eq(m.infer_decoder_batch([chunks[4]])[0].as_slice(), got[4].as_slice())
    assert m.infer_decoder_batch([]) == []


def test_batched_i16_equals_n1_and_host_post_path(voices):
    m = voices("medium4")
    encs = _chunk_latents(m)
    base = _chunk_set(encs)
    trims = [(0, 0), (3, 3), (0, 3), (3, 0), (0, 3), (0, 0), (3, 3), (3, 3), (3, 0), (0, 0), (3, 0)]
    chunks = [c + t for c, t in zip(base, trims)]
    gains = [1.0 if k % 3 else 0.8 for k in range(len(chunks))]
    got = m.infer_decoder_batch(chunks, pcm16=True, fade=42, gains=gains)
    for k, (e, lo, hi, tl, th) in enumerate(chunks):
        one = m.infer_decoder_batch([chunks[k]], pcm16=True, fade=42, gains=[gains[k]])[0]
        assert _eq(got[k], one), k
        x = e.infer_decoder(lo, hi).as_slice()
        x = x[tl * HOP: len(x) - th * HOP]
        s = AudioSamples(x)
        s.crossfade(42)
        v = s.as_slice() if gains[k] == 1.0 else s.as_slice() * np.float32(gains[k])
        ref = AudioSamples(v).to_i16_vec()
        assert got[k].shape == ref.shape, k
        # the faded samples go through sinf in the library and numpy's float32 sin here: one LSB there, nothing else
        d = np.abs(got[k].astype(np.int32) - ref.astype(np.int32))
        n = min(42, len(x) // 2)
        assert d.max() <= 1 and not d[n:len(d) - n].any(), k


def test_i16_equals_facade_realtime_events(voices, lib_built):
    from test_libsonata_facade import CALLBACK, ExternError, PiperSynthConfig, SynthesisEvent, SynthesisParams
    lib = lib_built
    lib.libsonataLoadVoiceFromConfigPath.restype = C.c_void_p
    lib.libsonataLoadVoiceFromConfigPath.argtypes = [C.c_char_p, C.POINTER(ExternError)]
    lib.libsonataSpeak.argtypes = [C.c_void_p, C.c_char_p, SynthesisParams, C.POINTER(ExternError)]
    lib.libsonataSetPiperSynthConfig.argtypes = [C.c_void_p, PiperSynthConfig, C.POINTER(ExternError)]
    lib.libsonataFreeSynthesisEvent.argtypes = [SynthesisEvent]
    lib.libsonataUnloadSonataVoice.argtypes = [C.c_void_p]
    err = ExternError()
    path = voices.paths["medium"]
    v = lib.libsonataLoadVoiceFromConfigPath(path.encode(), C.byref(err))
    assert v and err.code == 0
    # zero noise; on a single-speaker voice the call sets the scales and then refuses Some(speaker)
    lib.libsonataSetPiperSynthConfig(v, PiperSynthConfig(0, 1.0, 0.0, 0.0), C.byref(err))
    events = []

    def cb(ev):
        pcm = np.ctypeslib.as_array(ev.data, shape=(max(ev.len, 1),))[:ev.len].copy()
        events.append((ev.event_type, pcm.view("<i2")))
        lib.libsonataFreeSynthesisEvent(ev)
        return 0
    text = "ðɪs ɪz ə tɛst əv ðə riːəltaɪm moʊd wɪð ə lɔŋɡɚ sɛntəns ðæt niːdz mɔːɹ ðæn wʌn tʃʌŋk ænd sʌm mɔːɹ"
    cb_c = CALLBACK(cb)
    lib.libsonataSpeak(v, text.encode("utf-8"), SynthesisParams(2, 10, 100, 50, 0, cb_c, 0), C.byref(err))
    assert err.code == 0
    lib.libsonataUnloadSonataVoice(v)
    got = [e[1] for e in events if e[0] == 0]
    m = voices("medium")
    saved = m.get_fallback_synthesis_config()
    m.set_fallback_synthesis_config(PiperSynthesisConfig(None, **ZERO))
    try:
        enc = m.infer_encoder(m.phonemes_to_input_ids(text))
    finally:
        m.set_fallback_synthesis_config(saved)
    assert enc.num_frames > 2 * 72 + 6                      # not one-shot
    chunks = []
    for (m0, m1), (a0, a1) in AdaptiveMelChunker(enc.num_frames, 72, 3):
        chunks.append((enc, m0, enc.num_frames if m1 is None else m1, a0 // HOP, 0 if a1 is None else -a1 // HOP))
    exp = m.infer_decoder_batch(chunks, pcm16=True, fade=42)
    assert len(got) == len(exp) > 1
    for g, e in zip(got, exp):
        assert _eq(g, e)


def test_chunk_entry_points_add_only_their_output_stage_launches(voices):
    """Over the same chunks every chunk entry point launches what sb200_decode_chunks launches, plus its output stage:
    the i16 conversion (peak, convert), the resample launch (also when every resampler is null), or both."""
    from sonata_b200 import _native as N
    from sonata_b200.piper import Resampler
    m = voices("medium4")
    chunks = _chunk_set(_chunk_latents(m))
    trimmed = [c + ((3, 3) if c[2] - c[1] > 6 else (0, 0)) for c in chunks]
    rs = [Resampler(m, (8000, 48000)[k % 2]) if k % 3 else None for k in range(len(chunks))]

    def launches(f):
        n0 = N.lib().sb200_launch_count()
        f()
        return N.lib().sb200_launch_count() - n0
    base = launches(lambda: m.infer_decoder_batch(chunks))
    assert base > 0
    assert launches(lambda: chunks[2][0].infer_decoder(chunks[2][1], chunks[2][2])) == \
        launches(lambda: m.infer_decoder_batch([chunks[2]]))
    extra = [launches(lambda: m.infer_decoder_batch(trimmed, pcm16=True, fade=42)),
             launches(lambda: m.infer_decoder_batch(trimmed, fade=42, resamplers=rs)),
             launches(lambda: m.infer_decoder_batch(trimmed, pcm16=True, fade=42, resamplers=rs)),
             launches(lambda: m.infer_decoder_batch(trimmed, fade=42, resamplers=[None] * len(chunks)))]
    assert [e - base for e in extra] == [2, 1, 3, 1]


def _alone_stream(m, ids, cfg, cs, pad):
    enc = _alone_latent(m, ids, cfg)
    return [a.as_slice().copy() for a in SpeechStreamer(enc, cs, pad)]


def test_stream_batch_equals_stream_synthesis(voices):
    m = voices("medium4")
    cs, pad = 55, 3
    lens = [256, 12, 90, 300, 40, 150, 256, 70, 200, 33, 120, 256, 60, 180, 95, 256]
    specs = [(_ids(n, 200 + i), PiperSynthesisConfig(i % 4, length_scale=LENGTH_SCALES[i % 3], **ZERO))
             for i, n in enumerate(lens)]
    admit_at = [0] * 6 + [1] * 4 + [3] * 3 + [6] * 3
    sb = StreamBatch(m, cs, pad)
    keys, got, step = {}, {}, 0
    while len(sb) or step <= max(admit_at):
        for i, t in enumerate(admit_at):
            if t == step:
                keys[i] = sb.add(*specs[i])
        for key, a in sb.step():
            got.setdefault(key, []).append(a.as_slice().copy())
        step += 1
    for i, (ids, cfg) in enumerate(specs):
        exp = _alone_stream(m, ids, cfg, cs, pad)
        assert len(got[keys[i]]) == len(exp), i
        assert all(_eq(g, e) for g, e in zip(got[keys[i]], exp)), i
    assert len(got[keys[1]]) == 1                           # the 12-id stream is one-shot
    # a stream whose chunks reach the 1024-frame cap (large chunk_size and length_scale), next to a short one
    sb = StreamBatch(m, 600, pad)
    long_spec = (_ids(600, 250), PiperSynthesisConfig(2, length_scale=1.6, **ZERO))
    short_spec = (_ids(120, 251), PiperSynthesisConfig(1, **ZERO))
    k1, k2 = sb.add(*long_spec), sb.add(*short_spec)
    got = {}
    while len(sb):
        for key, a in sb.step():
            got.setdefault(key, []).append(a.as_slice().copy())
    exp = _alone_stream(m, *long_spec, 600, pad)
    assert max(len(e) for e in exp) == (1024 + 3 * pad) * HOP - 2 * pad * HOP
    assert len(got[k1]) == len(exp) and all(_eq(g, e) for g, e in zip(got[k1], exp))
    exp = _alone_stream(m, *short_spec, 600, pad)
    assert len(got[k2]) == len(exp) and all(_eq(g, e) for g, e in zip(got[k2], exp))


@pytest.mark.parametrize("voice", ["medium", "x_low"])
def test_realtime_batch_equals_synthesize_streamed(voices, voice):
    m = voices(voice)
    saved = m.get_fallback_synthesis_config()
    a = "ðɪs ɪz ə tɛst əv ðə riːəltaɪm moʊd wɪð ə lɔŋɡɚ sɛntəns ðæt niːdz mɔːɹ ðæn wʌn tʃʌŋk"
    b = "hɛloʊ wɜːld"
    texts = ["\n".join([a, a + " " + a, b]), b, "\n".join([a + " " + b, b + " " + b]), "\n".join([a + " " + a + " " + a, b, a])]
    ocs = [None, AudioOutputConfig(volume=60), AudioOutputConfig(appended_silence_ms=50),
           AudioOutputConfig(volume=90, appended_silence_ms=20)]
    cfgs = [PiperSynthesisConfig(None, length_scale=ls, **ZERO) for ls in (1.0, 1.2, 0.8, 1.0)]
    syn = SonataSpeechSynthesizer(m)
    exp = []
    try:
        for t, oc, cfg in zip(texts, ocs, cfgs):
            m.set_fallback_synthesis_config(cfg)
            exp.append([a.as_slice().copy() for a in syn.synthesize_streamed(t, oc, 55, 3)])
    finally:
        m.set_fallback_synthesis_config(saved)
    rb = RealtimeBatch(m, 55, 3)
    keys = [rb.add(t, oc, cfg) for t, oc, cfg in zip(texts[:2], ocs[:2], cfgs[:2])]
    got, step = {}, 0
    while len(rb) or step < 2:
        if step == 1:
            keys += [rb.add(t, oc, cfg) for t, oc, cfg in zip(texts[2:], ocs[2:], cfgs[2:])]
        for key, a in rb.step():
            got.setdefault(key, []).append(a.as_slice().copy())
        step += 1
    for k, e in zip(keys, exp):
        assert len(got[k]) == len(e) and all(_eq(g, x) for g, x in zip(got[k], e)), k


def test_errors_name_the_index_and_leave_the_voice_working(voices):
    m, other = voices("medium4"), voices("high3")
    encs = m.infer_encoder_batch([_ids(40, 1), _ids(50, 2)], [PiperSynthesisConfig(1, **ZERO)] * 2)
    foreign = other.infer_encoder(_ids(30, 3))
    before = m.infer_decoder_batch([(encs[0], 0, 20), (encs[1], 5, 40)])
    with pytest.raises(OperationError, match="chunk 1"):
        m.infer_decoder_batch([(encs[0], 0, 20), (foreign, 0, 10)])
    f = encs[1].num_frames
    for bad, idx in (((encs[0], 0, 20), (encs[1], 0, f + 1)), 1), (((encs[0], -1, 20),), 0), \
                    (((encs[0], 0, 5), (encs[1], 7, 7)), 1), (((encs[0], 9, 3),), 0):
        with pytest.raises(OperationError, match=f"chunk {idx}"):
            m.infer_decoder_batch(list(bad))
    with pytest.raises(OperationError, match="chunk 0"):
        m.infer_decoder_batch([(encs[0], 0, 2, 1, 1)], pcm16=True)          # trims leave no sample
    with pytest.raises(OperationError, match="utterance 1"):
        m.infer_encoder_batch([_ids(10, 4), _ids(10, 5)], [PiperSynthesisConfig(1), PiperSynthesisConfig(9)])
    after = m.infer_decoder_batch([(encs[0], 0, 20), (encs[1], 5, 40)])
    assert all(_eq(a.as_slice(), b.as_slice()) for a, b in zip(before, after))
    again = m.infer_encoder_batch([_ids(40, 1)], [PiperSynthesisConfig(1, **ZERO)])[0]
    assert _eq(again.infer_decoder().as_slice(), encs[0].infer_decoder().as_slice())
    # the single-chunk entry point keeps its message
    with pytest.raises(OperationError) as e:
        encs[1].infer_decoder(0, f + 1)
    assert str(e.value) == "Invalid model audio output"


def test_a_failing_stream_leaves_the_others_running(voices):
    """A stream whose encoder pass fails on the device side (durations too long) gets its error once and ends; the
    streams encoded with it and before it still equal stream_synthesis, and a bad speaker is refused at admission."""
    m = voices("medium4")
    sb = StreamBatch(m, 55, 3)
    with pytest.raises(OperationError, match="No speaker"):
        sb.add(_ids(40, 400), PiperSynthesisConfig(9, **ZERO))
    specs = {sb.add(ids, cfg): (ids, cfg) for ids, cfg in ((_ids(150, 401), PiperSynthesisConfig(1, **ZERO)),
                                                          (_ids(60, 402), PiperSynthesisConfig(2, **ZERO)))}
    got = {}
    for key, a in sb.step():
        got.setdefault(key, []).append(a)
    bad = sb.add(_ids(80, 403), PiperSynthesisConfig(3, length_scale=1e9, **ZERO))
    later = (_ids(200, 404), PiperSynthesisConfig(0, **ZERO))
    specs[sb.add(*later)] = later
    while len(sb):
        for key, a in sb.step():
            got.setdefault(key, []).append(a)
    assert len(got[bad]) == 1 and isinstance(got[bad][0], OperationError) and "long" in str(got[bad][0])
    for key, (ids, cfg) in specs.items():
        exp = _alone_stream(m, ids, cfg, 55, 3)
        assert len(got[key]) == len(exp) and all(_eq(g.as_slice(), x) for g, x in zip(got[key], exp)), key
