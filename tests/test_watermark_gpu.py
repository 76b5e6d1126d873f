"""GPU (-m gpu): the watermark (include/sonata_b200.h, sb200_voice_set_watermark and sb200_watermark_detect).

Bit for bit against tests/watermark_reference.py: the test hook; a marked job against the contract applied to the same
seeded job on the unmarked voice, on all four voices, at the voice's rate and at 8 and 48 kHz, through every waveform
stage; loudness, i16, G.711 and FLAC on the marked samples; batch independence; an unmarked voice's bits and launches.
The device detector against numpy, and detection end to end at C2 through every route, cropped, with wrong keys and
unmarked audio never detected."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import watermark_reference as wr
from sonata_b200 import _native as N, voicegen, workload
from sonata_b200.core import AudioSamples, OperationError, flac_encode, watermark_detect
from sonata_b200.job import SynthesisJob
from sonata_b200.piper import PiperSynthesisConfig, StreamBatch, VitsStreamingModel

pytestmark = pytest.mark.gpu
NAN = float("nan")
QUALITIES = ("x_low", "low", "medium", "high")
KEY, PAYLOAD, DB = 0x5EC12E7_0DDBA11, 1234, -26.0
f32p = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))


def _message(err):
    return C.string_at(err.message).decode() if err.message else ""


def debug_watermark(x, rate, key=KEY, payload=PAYLOAD, db=DB):
    x = np.ascontiguousarray(x, np.float32)
    y, err = np.zeros_like(x), N.sb200_error()
    wm = N.sb200_watermark(key, payload, db)
    assert N.lib().sb200_debug_watermark(f32p(x), x.size, rate, C.byref(wm), f32p(y), C.byref(err)) == 0, \
        _message(err)
    return y


@pytest.fixture(scope="module")
def voices(lib_built):
    d = voicegen.default_voice_dir()
    ms = {}

    def get(q):
        if q not in ms:
            ms[q] = VitsStreamingModel(voicegen.write_voice(d, q), device=0)
            ms[q].set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.667, 1.0, 0.8))
        return ms[q]
    yield get
    for m in ms.values():
        m.close()


def _job(m, batches, seeds, **kw):
    j = SynthesisJob(m, batches, seeds=seeds, **kw)
    j.run()
    return j, [a.samples.as_slice().copy() for a in j.fetch()]


def _marked(m, fn, key=KEY, payload=PAYLOAD, db=DB):
    m.set_watermark(key, payload, db)
    try:
        return fn()
    finally:
        m.set_watermark(None)


# ---------------------------------------------------------------------------------------------------- the hook
@pytest.mark.parametrize("rate", (8000, 16000, 22050, 48000))
def test_hook_equals_the_contract(lib_built, rate):
    rng = np.random.default_rng(rate)
    B = rate // 100
    for n in (1, B - 1, B, B + 1, 3 * B + 7, 50 * B + 13, 40 * B * 32 + 5):
        x = (0.3 * rng.standard_normal(n)).astype(np.float32)
        x[::97] = 1.5
        x[: min(n, 2 * B)] = 0.0                     # leading silence: no mark
        for payload, db in ((0, -40.0), (4095, -10.0), (PAYLOAD, DB)):
            got = debug_watermark(x, rate, KEY, payload, db)
            assert got.tobytes() == wr.embed(x, rate, KEY, payload, db).tobytes(), (n, payload, db)
    assert debug_watermark(np.zeros(5000, np.float32), rate).tobytes() == np.zeros(5000, np.float32).tobytes()


# ---------------------------------------------------------------------------------------------------- batches
ARMS = [dict(), dict(pitches=[1.25, None, 0.8], tempos=[None, 1.3, 0.8]), dict(formants=[1.2, None, 0.9]),
        dict(pitch_contours="q", volume_contours="v", breaks="b"), dict(target_durations=[None, 3000.0, None])]


def _arm(kw, lens):
    kw = dict(kw)
    if kw.get("pitch_contours") == "q":
        kw["pitch_contours"] = [np.where(np.arange(n) > 2 * n // 3, 1.3, 1.0).astype(np.float32) if b != 1 else None
                                for b, n in enumerate(lens)]
        kw["volume_contours"] = [np.where(np.arange(n) % 9 == 4, 6.0, NAN).astype(np.float32) for n in lens]
        kw["breaks"] = [np.where(np.arange(n) % 23 == 11, 120.0, NAN).astype(np.float32) for n in lens]
    return kw


@pytest.mark.parametrize("quality", QUALITIES)
def test_marked_job_equals_the_contract(voices, quality):
    m = voices(quality)
    rate = m.audio_output_info().sample_rate
    batches = [list(workload.synthetic_ids(60 + 40 * b, utt=b + 3)) for b in range(3)]
    lens = [len(b) for b in batches]
    c = wr.chips(KEY)
    for i, kw in enumerate(ARMS):
        kw = _arm(kw, lens)
        for rates in (None, [8000, 48000, None]):
            r_kw = dict(kw, output_rates=rates) if rates else kw
            _, base = _job(m, batches, [11, 12, 13], **r_kw)
            j, got = _marked(m, lambda: _job(m, batches, [11, 12, 13], **r_kw))
            for b in range(3):
                rb = (rates[b] if rates else None) or rate
                assert got[b].tobytes() == wr.embed(base[b], rb, KEY, PAYLOAD, DB, c).tobytes(), (i, rates, b)
            assert [r["launches"] for r in j.profile() if r["name"] == "watermark"] == [1]


def test_loudness_i16_g711_and_flac_carry_the_marked_samples(voices):
    m = voices("medium")
    rate = m.audio_output_info().sample_rate
    batches = [list(workload.synthetic_ids(150, utt=b + 1)) for b in range(2)]
    c = wr.chips(KEY)
    _, base = _job(m, batches, [3, 4])
    marked = [wr.embed(x, rate, KEY, PAYLOAD, DB, c) for x in base]

    def run():
        jl, loud = _job(m, batches, [3, 4], loudness=[-23.0, None])
        j, _ = _job(m, batches, [3, 4])
        return jl.loudness(), loud, j.fetch_i16(), j.fetch_g711("mulaw"), j.fetch_g711("alaw"), j.fetch_flac()
    (lufs, gain), loud, i16, mu, al, fl = _marked(m, run)
    assert loud[0].tobytes() == (marked[0] * gain[0]).astype(np.float32).tobytes()
    assert loud[1].tobytes() == marked[1].tobytes()
    for b in range(2):
        want = AudioSamples(marked[b]).to_i16_vec()
        assert i16[b].tobytes() == want.tobytes()
        assert fl[b] == flac_encode(want, rate)
    import g711_reference as gr
    assert [bytes(x) for x in mu] == [gr.encode_bytes(x, "mulaw") for x in i16]
    assert [bytes(x) for x in al] == [gr.encode_bytes(x, "alaw") for x in i16]


def test_batch_independence_and_the_unmarked_voice(voices):
    m = voices("low")
    batches = [list(workload.synthetic_ids(90 + 30 * b, utt=b + 5)) for b in range(3)]
    _, mixed = _marked(m, lambda: _job(m, batches, [1, 2, 3], pitches=[None, 1.3, None], output_rates=[None, 8000, None]))
    for b in range(3):
        _, alone = _marked(m, lambda: _job(m, [batches[b]], [b + 1], pitches=[[None, 1.3, None][b]],
                                           output_rates=[[None, 8000, None][b]]))
        assert alone[0].tobytes() == mixed[b].tobytes(), b
    lib = N.lib()
    n0 = lib.sb200_launch_count()
    j0, plain = _job(m, batches, [1, 2, 3])
    n1 = lib.sb200_launch_count()
    m.set_watermark(KEY, 7, -20.0)
    assert m.watermark() == (KEY, 7, -20.0)
    m.set_watermark(None)
    assert m.watermark() is None
    n2 = lib.sb200_launch_count()
    j1, again = _job(m, batches, [1, 2, 3])
    n3 = lib.sb200_launch_count()
    assert n1 - n0 == n3 - n2
    assert all(a.tobytes() == b.tobytes() for a, b in zip(plain, again))
    assert not any(r["name"] == "watermark" for r in j0.profile() + j1.profile())


LONG = "hɛloʊ wɜːld ðɪs ɪz ə lɔŋɡɚ sɛntəns ðæt ɪz spoʊkən ɪn tʃʌŋks ænd ðɛn sʌm moʊr wɜːdz"
STREAM_KINDS = {
    "plain": dict(), "resampled": dict(output_rate=16000), "warped": dict(pitch=1.25, tempo=0.9),
    "contoured": dict(pitch_contour=[1.3 if i % 5 == 0 else None for i in range(len(LONG))]),
    "formant": dict(formant_ratio=1.2),
    "volume": dict(volume_contour=[6.0 if i % 7 == 3 else None for i in range(len(LONG))]),
    "paused": dict(breaks=[120.0 if i % 11 == 5 else None for i in range(len(LONG))], output_rate=48000),
}


def _device_plain(m, cs, pad, seed):
    """The plain stream's chunks through the device post-path, unmarked, as a marked plain stream runs them."""
    from sonata_b200.piper import SpeechStreamer, _device_post
    enc = m.infer_encoder_batch([m.phonemes_to_input_ids(LONG)], seeds=[seed])[0]
    s, out = SpeechStreamer(enc, cs, pad), []
    while not s.done:
        lo, hi, trim = s.next_chunk()
        s.resampler = None
        out.append(m.infer_decoder_batch([(enc, lo, hi) + ((0, 0) if trim is None else _trim_frames(trim))],
                                         fade=0 if trim is None else 42, resamplers=[None], last=[s.done])[0])
    return out


def _trim_frames(trim):
    from sonata_b200.piper import _trim_frames as t
    return t(trim)


def _stream(m, kw, cs=20, pad=3, seed=5):
    st = m.stream_synthesis(LONG, cs, pad, seed=seed, **kw)
    return list(st), st


@pytest.mark.parametrize("kind", sorted(STREAM_KINDS))
def test_marked_streams_equal_the_contract(voices, kind):
    m = voices("medium")
    kw = STREAM_KINDS[kind]
    rate = kw.get("output_rate") or m.audio_output_info().sample_rate
    base, sb = _stream(m, kw)
    if kind == "plain":
        base = _device_plain(m, 20, 3, 5)
    got, sm = _marked(m, lambda: _stream(m, kw))
    assert len(got) == len(base) > 2
    assert (sm.bounds is None) == (sb.bounds is None)
    if sb.bounds is not None:
        assert sm.bounds.tobytes() == sb.bounds.tobytes()
    joined = np.concatenate([a.as_slice() for a in got])
    want = wr.embed(np.concatenate([a.as_slice() for a in base]), rate, KEY, PAYLOAD, DB)
    assert joined.tobytes() == want.tobytes()
    # the chunks are the stream emission rule over the unmarked chunks
    ref = wr.stream([a.as_slice() for a in base], rate, KEY, PAYLOAD, DB)
    assert [a.as_slice().tobytes() for a in got] == [r.tobytes() for r in ref]


def test_metered_and_g711_streams(voices):
    import g711_reference as gr
    m = voices("medium")
    # G.711: each chunk's bytes are those of the marked f32 chunk, peak-normalised as an unmarked chunk is
    f32, _ = _marked(m, lambda: _stream(m, dict(output_rate=8000)))
    mu, _ = _marked(m, lambda: _stream(m, dict(output_rate=8000, encoding="mulaw")))
    plain_mu, _ = _stream(m, dict(output_rate=8000, encoding="mulaw"))
    assert len(mu) == len(plain_mu) == len(f32)
    assert [bytes(b) for b in mu] == [gr.encode_bytes(AudioSamples(a.as_slice()).to_i16_vec(), "mulaw") for a in f32]
    # metered: the meter reads the marked samples; the chunk count does not change and the mark is found
    met, _ = _marked(m, lambda: _stream(m, dict(live_loudness=-20.0)))
    plain_met, _ = _stream(m, dict(live_loudness=-20.0))
    assert len(met) == len(plain_met)
    assert sum(a.as_slice().size for a in met) == sum(a.as_slice().size for a in plain_met)


def test_a_stream_keeps_its_setting_and_stream_batch_marks(voices):
    m = voices("medium")
    base, _ = _stream(m, dict(output_rate=16000))
    # an unmarked stream stays unmarked when the voice is marked midway, and a marked one stays marked
    st = m.stream_synthesis(LONG, 20, 3, seed=5, output_rate=16000)
    first = [next(st)]
    m.set_watermark(KEY, PAYLOAD, DB)
    try:
        rest = list(st)
        st2 = m.stream_synthesis(LONG, 20, 3, seed=5, output_rate=16000)
        first2 = [next(st2)]
    finally:
        m.set_watermark(None)
    rest2 = list(st2)
    assert [a.as_slice().tobytes() for a in first + rest] == [a.as_slice().tobytes() for a in base]
    joined = np.concatenate([a.as_slice() for a in first2 + rest2])
    assert joined.tobytes() == wr.embed(np.concatenate([a.as_slice() for a in base]), 16000, KEY, PAYLOAD,
                                        DB).tobytes()
    # StreamBatch: marked and unmarked streams side by side
    ids = m.phonemes_to_input_ids(LONG)
    sb = StreamBatch(m, 20, 3)
    k0 = sb.add(ids, seed=5)
    m.set_watermark(KEY, PAYLOAD, DB)
    try:
        k1 = sb.add(ids, seed=5)
    finally:
        m.set_watermark(None)
    got = {}
    while len(sb):
        for k, a in sb.step():
            assert not isinstance(a, Exception), a
            got.setdefault(k, []).append(a.as_slice())
    plain = _device_plain(m, 20, 3, 5)
    assert len(got[k1]) == len(got[k0]) == len(plain)
    rate = m.audio_output_info().sample_rate
    assert np.concatenate(got[k1]).tobytes() == wr.embed(np.concatenate([a.as_slice() for a in plain]), rate, KEY,
                                                         PAYLOAD, DB).tobytes()


# ---------------------------------------------------------------------------------------------------- detection
def test_device_detector_equals_numpy(lib_built):
    rng = np.random.default_rng(5)
    c, rate = wr.chips(KEY), 16000
    clips = []
    for t in range(12):
        x = (0.2 * rng.standard_normal(int(rng.integers(2000, 120000)))).astype(np.float32)
        if t % 2:
            x = wr.embed(x, rate, KEY, (37 * t) % 4096, -20.0, c)
        lo = int(rng.integers(0, x.size // 3))
        clips.append(x[lo:])
    clips.append(np.zeros(5000, np.float32))
    clips.append(np.zeros(0, np.float32))
    for fmt in ("f32", "i16"):
        cl = clips if fmt == "f32" else [AudioSamples(x).to_i16_vec() if x.size else np.zeros(0, np.int16) for x in clips]
        got = watermark_detect(cl, KEY)
        for g, x in zip(got, cl):
            want = wr.detect(x, KEY, c)
            assert (g.marked, g.payload, g.offset) == (want["marked"], want["payload"], want["offset"])
            assert abs(g.z0 - want["z0"]) < 1e-9 and abs(g.z1 - want["z1"]) < 1e-9


def _g711_decode(b, law):
    u = np.frombuffer(bytes(b), np.uint8).astype(np.int32)
    if law == "mulaw":
        u = ~u & 0xFF
        t = (((u & 0x0F) << 3) + 0x84) << ((u & 0x70) >> 4)
        return np.where(u & 0x80, 0x84 - t, t - 0x84).astype(np.int16)
    a = u ^ 0x55
    seg = (a & 0x70) >> 4
    t = (a & 0x0F) << 4
    t = np.where(seg == 0, t + 8, (t + 0x108) << np.maximum(seg - 1, 0))
    return np.where(a & 0x80, t, -t).astype(np.int16)


def test_c2_every_route_is_detected(voices):
    m = voices("medium")
    qual, batch, n_ph = workload.CONFIGS["C2"]
    batches = [list(workload.synthetic_ids(n_ph, utt=u)) for u in range(batch)]
    seeds = list(range(100, 100 + batch))

    def routes():
        j = SynthesisJob(m, batches, seeds=seeds)
        j.run()
        f32 = [a.samples.as_slice().copy() for a in j.fetch()]
        i16, fl = j.fetch_i16(), j.fetch_flac()
        j8 = SynthesisJob(m, batches, seeds=seeds, output_rates=[8000] * batch)
        j8.run()
        mu = [_g711_decode(x, "mulaw") for x in j8.fetch_g711("mulaw")]
        al = [_g711_decode(x, "alaw") for x in j8.fetch_g711("alaw")]
        j48 = SynthesisJob(m, batches, seeds=seeds, output_rates=[48000] * batch, loudness=[-16.0] * batch)
        j48.run()
        loud = [a.samples.as_slice().copy() for a in j48.fetch()]
        return dict(f32=(f32, 22050), i16=(i16, 22050), flac=(i16, 22050), mulaw=(mu, 8000), alaw=(al, 8000),
                    loud48=(loud, 48000)), fl
    plain, _ = routes()
    marked, fl = _marked(m, routes)
    assert fl == [flac_encode(x, 22050) for x in marked["i16"][0]]
    for name, (clips, rate) in marked.items():
        crops = [x[x.size // 2 - 5 * rate // 2:][:5 * rate] for x in clips]      # 5 s from the middle
        for what, cl in (("whole", clips), ("5 s crop", crops)):
            got = watermark_detect(cl, KEY)
            found = sum(g.marked and g.payload == PAYLOAD for g in got)
            # at 8 kHz, -26 dB and 5 s (40 000 samples) sit near the threshold: (alpha / sqrt 2) sqrt(n) = 7.1 for a
            # white host, and 30 of these 32 crops pass (the batch is seeded, so on every run); -20 dB finds them all
            need = len(cl) if what == "whole" or rate > 8000 else int(np.ceil(0.9 * len(cl)))
            assert found >= need, (name, what, found, [(round(g.z0, 1), round(g.z1, 1)) for g in got])
            assert not any(g.marked for g in watermark_detect(cl, KEY + 1)), (name, what)
        assert not any(g.marked for g in watermark_detect(plain[name][0], KEY)), name

    def mulaw_8k():
        j8 = SynthesisJob(m, batches, seeds=seeds, output_rates=[8000] * batch)
        j8.run()
        return [_g711_decode(x, "mulaw") for x in j8.fetch_g711("mulaw")]
    crops = [x[x.size // 2 - 20000:][:40000] for x in _marked(m, mulaw_8k, db=-20.0)]
    assert all(g.marked and g.payload == PAYLOAD for g in watermark_detect(crops, KEY))
