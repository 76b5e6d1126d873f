"""GPU (-m gpu): breaks (include/sonata_b200.h, sb200_speak_batch_ids_breaks and sb200_prosody_stream_create_breaks).

Everything is bit for bit against tests/break_reference.py: the test hook; a paused batch against the contract applied
to the same seeded batch without breaks (with pitch, tempo, pitch contours, formants, volume contours and blends, an
output rate and a loudness target); the delivered ends every route reports; neutral images and batch independence;
the i16, G.711 and FLAC routes; and streams of every kind joined against the contract applied to the joined chunks of
the same stream without breaks."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import break_reference as br
import flac_reference as fr
import g711_reference as gr
from test_prosody_stream_gpu import LONG, SHORT, _cat, _drain, _plain, _same, debug_resample, voices  # noqa: F401
from test_volume_gpu import _stream_ends, debug_loudness, levels_for
from sonata_b200 import _native as N, voicegen, workload
from sonata_b200.core import AudioSamples
from sonata_b200.job import SynthesisJob
from sonata_b200.piper import (LoudnessStream, PiperSynthesisConfig, ProsodyStream, Resampler, SpeechStreamer,
                               StreamBatch, VitsStreamingModel, _char_breaks_to_ids)

pytestmark = pytest.mark.gpu
NAN = float("nan")
QUALITIES = ("x_low", "low", "medium", "high")
f32p = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
i64p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))


def debug_breaks(x, ends, ms, rate):
    x = np.ascontiguousarray(x, np.float32)
    e, b = np.ascontiguousarray(ends, np.int64), np.ascontiguousarray(ms, np.float32)
    cap = x.size + int(br.samples(b, rate).sum())
    y, n, err = np.zeros(max(cap, 1), np.float32), C.c_int64(), N.sb200_error()
    rc = N.lib().sb200_debug_breaks(0, f32p(x), x.size, i64p(e), f32p(b), e.size, rate, f32p(y), cap, C.byref(n),
                                    C.byref(err))
    assert rc == 0, C.string_at(err.message).decode() if err.message else rc
    assert n.value == cap
    return y[:cap]


def breaks_for(n_ids, kind, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "every10":               # 250 ms after every 10th id
        return np.where(np.arange(n_ids) % 10 == 9, 250.0, NAN).astype(np.float32)
    if kind == "few":                   # two pauses, one at the end
        v = np.full(n_ids, NAN, np.float32)
        v[n_ids // 3] = 120.0
        v[-1] = 300.0
        return v
    if kind == "wild":                  # close pauses, tiny ones that round to nothing, and merges on empty ids
        return rng.choice(np.array([NAN, 0.0, 0.01, 2.0, 7.5, 60.0], np.float32), n_ids)
    raise ValueError(kind)


# ---------------------------------------------------------------------------------------------------- the hook
@pytest.mark.parametrize("rate", (22050, 16000))
def test_hook_equals_the_contract(lib_built, rate):
    rng = np.random.default_rng(rate)
    for trial in range(8):
        n_ids = int(rng.integers(1, 60))
        lens = rng.choice([0, 1, 2, 5, 40, 111, 256, 700, 3000], n_ids)
        ends = np.cumsum(lens)
        if ends[-1] == 0:
            ends[-1] = lens[-1] = 1
        x = rng.standard_normal(int(ends[-1])).astype(np.float32)
        ms = rng.choice(np.array([NAN, 0.0, 0.01, 1.0, 3.3, 25.0, 400.0], np.float32), n_ids)
        assert debug_breaks(x, ends, ms, rate).tobytes() == br.apply(x, ends, ms, rate).tobytes(), trial
    # breaks at 0 and at n2, merged
    x = rng.standard_normal(5000).astype(np.float32)
    ends, ms = [0, 0, 2500, 5000, 5000], [3.0, 4.0, NAN, 10.0, 20.0]
    assert debug_breaks(x, ends, ms, rate).tobytes() == br.apply(x, ends, ms, rate).tobytes()


# ---------------------------------------------------------------------------------------------------- batches
def _job(m, batches, seeds, **kw):
    j = SynthesisJob(m, batches, seeds=seeds, **kw)
    j.run()
    out = [a.samples.as_slice().copy() for a in j.fetch()]
    return j, out


ARMS = [dict(), dict(pitches=[1.25, None, 0.8]), dict(tempos=[1.5, None, 0.7]),
        dict(pitches=[1.2, 0.9, None], tempos=[None, 1.3, 0.8], formants=[1.0, 1.1, None]),
        dict(pitch_contours="q"), dict(formants=[1.2, None, 0.9]), dict(volume_contours="v")]


def _arm(kw, lens):
    kw = dict(kw)
    if kw.get("pitch_contours") == "q":
        kw["pitch_contours"] = [np.where(np.arange(n) > 2 * n // 3, 1.3, 1.0).astype(np.float32) if b != 1 else None
                                for b, n in enumerate(lens)]
    if kw.get("volume_contours") == "v":
        kw["volume_contours"] = [levels_for(n, "mixed", b) for b, n in enumerate(lens)]
    return kw


@pytest.mark.parametrize("quality", QUALITIES)
def test_batch_equals_the_contract(voices, quality):
    m = voices(quality)
    rate = m.audio_output_info().sample_rate
    batches = [list(workload.synthetic_ids(60 + 40 * b, utt=b + 3)) for b in range(3)]
    lens = [len(b) for b in batches]
    seeds = [11, 12, 13]
    for i, kw in enumerate(ARMS):
        kw = _arm(kw, lens)
        jb, base = _job(m, batches, seeds, **kw)
        ends = jb.prosody_bounds()
        bks = [breaks_for(n, k, i) for n, k in zip(lens, ("every10", "few", "wild"))]
        bks[i % 3] = None if i % 2 else bks[i % 3]
        jk, got = _job(m, batches, seeds, breaks=bks, **kw)
        bounds = jk.prosody_bounds()
        for b in range(3):
            want = base[b] if bks[b] is None else br.apply(base[b], ends[b], bks[b], rate)
            assert got[b].tobytes() == want.tobytes(), (i, b)
            e2 = ends[b] if bks[b] is None else br.delivered_ends(ends[b], bks[b], rate)
            np.testing.assert_array_equal(bounds[b], e2)
            assert bounds[b][-1] == len(got[b])
        assert [int(n) for n in jk.lengths()[1]] == [len(g) for g in got]
        assert any(r["name"] == "break" and r["launches"] == 1 for r in jk.profile())
        # with an output rate: the contract at the voice's rate, then the resampler
        _, rs = _job(m, batches, seeds, breaks=bks, output_rates=[16000, None, 48000], **kw)
        for b, r in enumerate((16000, None, 48000)):
            want = base[b] if bks[b] is None else br.apply(base[b], ends[b], bks[b], rate)
            if r and r != rate:
                want = debug_resample(want, rate, r)
            assert rs[b].tobytes() == want.tobytes(), (i, b, r)


def test_loudness_normalises_the_paused_utterance(voices):
    m = voices("medium")
    rate = m.audio_output_info().sample_rate
    batches = [list(workload.synthetic_ids(150, utt=b + 1)) for b in range(2)]
    bks = [breaks_for(len(batches[0]), "every10"), breaks_for(len(batches[1]), "few")]
    jb, base = _job(m, batches, [3, 4])
    ends = jb.prosody_bounds()
    jk, got = _job(m, batches, [3, 4], breaks=bks, loudness=[-23.0, -16.0])
    lufs, gain = jk.loudness()
    for b in range(2):
        paused = br.apply(base[b], ends[b], bks[b], rate)
        assert lufs[b] == debug_loudness(paused, rate)
        assert got[b].tobytes() == (paused * gain[b]).astype(np.float32).tobytes()


def test_neutral_images_and_batch_independence(voices):
    m = voices("low")
    batches = [list(workload.synthetic_ids(90 + 30 * b, utt=b + 5)) for b in range(3)]
    lens = [len(b) for b in batches]
    lib = N.lib()
    n0 = lib.sb200_launch_count()
    _, plain = _job(m, batches, [1, 2, 3])
    n1 = lib.sb200_launch_count()
    _, neutral = _job(m, batches, [1, 2, 3], breaks=[[NAN] * n if b else [0.0] * n for b, n in enumerate(lens)])
    n2 = lib.sb200_launch_count()
    # breaks that ask but round to 0 samples reach the library, which plans no pause
    _, tiny = _job(m, batches, [1, 2, 3], breaks=[[0.01] * n for n in lens])
    n3 = lib.sb200_launch_count()
    assert n2 - n1 == n1 - n0 == n3 - n2
    assert all(a.tobytes() == b.tobytes() == c.tobytes() for a, b, c in zip(neutral, plain, tiny))
    # a paused utterance has the same bits alone and in any batch, and one without breaks beside it keeps its bits
    bks = [breaks_for(n, "wild", b) for b, n in enumerate(lens)]
    bks[1] = None
    _, mixed = _job(m, batches, [1, 2, 3], breaks=bks, pitches=[None, 1.3, None])
    for b in range(3):
        _, alone = _job(m, [batches[b]], [b + 1], breaks=[bks[b]], pitches=[[None, 1.3, None][b]])
        assert alone[0].tobytes() == mixed[b].tobytes(), b


def test_i16_g711_and_flac_of_a_paused_utterance(voices):
    m = voices("medium")
    rate = m.audio_output_info().sample_rate
    batches = [list(workload.synthetic_ids(120, utt=b + 2)) for b in range(2)]
    n = [len(ids) for ids in batches]
    bks = [np.where(np.arange(n[0]) == n[0] // 3, 1000.0, NAN).astype(np.float32), breaks_for(n[1], "few")]
    j = SynthesisJob(m, batches, seeds=[5, 6], breaks=bks)
    j.run()
    f32 = [a.samples.as_slice().copy() for a in j.fetch()]
    i16 = j.fetch_i16()
    for b in range(2):
        assert i16[b].tobytes() == AudioSamples(f32[b]).to_i16_vec().tobytes()
    for law in ("mulaw", "alaw"):
        got = j.fetch_g711(law, gains=[0.5, None])
        for b, g in enumerate((0.5, 1.0)):
            assert got[b] == gr.encode_bytes(AudioSamples(f32[b] * np.float32(g)).to_i16_vec(), law)
    flac = j.fetch_flac()
    for b in range(2):
        s = fr.decode(flac[b])
        assert s.sample_rate == rate and s.samples.astype(np.int16).tobytes() == i16[b].tobytes()
    # the 1 s pause spans whole all-zero blocks, coded CONSTANT
    s = fr.decode(flac[0])
    zero = [f for k, f in enumerate(s.frames) if not s.samples[k * 4096:(k + 1) * 4096].any()]
    assert zero and all(f.type == "CONSTANT" for f in zero)
    j.close()
    # the phoneme surfaces of the encoders take one break per character
    ph = [LONG, SHORT]
    cb = [[200.0 if c % 9 == 4 else None for c in range(len(LONG))], None]
    a = m.speak_batch(ph, seeds=[1, 2], breaks=cb)
    g = m.speak_batch_g711(ph, "mulaw", seeds=[1, 2], breaks=cb)
    fl = m.speak_batch_flac(ph, seeds=[1, 2], breaks=cb)
    for b in range(2):
        i = a[b].samples.to_i16_vec()
        assert g[b] == gr.encode_bytes(i, "mulaw")
        assert fr.decode(fl[b]).samples.astype(np.int16).tobytes() == i.tobytes()


def test_blends_alignment_and_the_phoneme_surfaces(lib_built):
    d = voicegen.default_voice_dir()
    m = VitsStreamingModel(voicegen.write_voice(d, "medium", n_speakers=4), device=0)
    m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.667, 1.0, 0.8))
    rate = m.audio_output_info().sample_rate
    try:
        ph = [LONG, SHORT]
        maps = [m.phonemes_to_input_ids_map(p) for p in ph]
        batches = [ids for ids, _ in maps]
        blends = [{0: 0.3, 2: 0.7}, None]
        cb = [[150.0 if i % 7 == 3 else None for i in range(len(LONG))], [None] * (len(SHORT) - 1) + [400.0]]
        per_id = [np.array(_char_breaks_to_ids(c, p, src, 0), np.float32) for c, p, (_, src) in zip(cb, ph, maps)]
        jb, base = _job(m, batches, [7, 8], speaker_blends=blends, tempos=[1.2, None])
        ends = jb.prosody_bounds()
        got = m.speak_batch(ph, seeds=[7, 8], speaker_blends=blends, tempos=[1.2, None], breaks=cb)
        al = m.speak_batch_with_alignment(ph, seeds=[7, 8], speaker_blends=blends, tempos=[1.2, None], breaks=cb,
                                          output_rates=[None, 16000])
        for b in range(2):
            want = br.apply(base[b], ends[b], per_id[b], rate)
            assert got[b].samples.as_slice().tobytes() == want.tobytes(), b
            audio, entries = al[b]
            n = len(audio.samples.as_slice())
            assert entries[0].start_sample == 0 and entries[-1].start_sample + entries[-1].num_samples == n
            assert all(e.start_sample + e.num_samples == f.start_sample for e, f in zip(entries, entries[1:]))
            # each entry ends at its last id's end after the pauses, at the output rate ceil(E' up / down)
            e2 = br.delivered_ends(ends[b], per_id[b], rate)
            up, down = (1, 1) if b == 0 else (16000 // 50, rate // 50)
            assert entries[-2].start_sample + entries[-2].num_samples == -((-int(e2[-2]) * up) // down)
        got = m.infer_batch_with_values(batches, seeds=[7, 8], speaker_blends=blends, tempos=[1.2, None],
                                        breaks=per_id)
        assert all(g.samples.as_slice().tobytes() == br.apply(base[b], ends[b], per_id[b], rate).tobytes()
                   for b, g in enumerate(got))
    finally:
        m.close()


# ---------------------------------------------------------------------------------------------------- streams
STREAM_ARMS = [dict(), dict(pitch=1.25), dict(tempo=1.4, pitch=0.9), dict(formant=1.2), dict(contour="q"),
               dict(volume="v"), dict(contour="q", tempo=0.8, formant=1.0)]


def _streams(m, ids, seed, arm):
    enc = m.infer_encoder_batch([ids], seeds=[seed])[0]
    contour = None
    if arm.get("contour") == "q":
        contour = np.where(np.arange(len(ids)) > len(ids) // 2, 1.3, NAN).astype(np.float32)
    vol = levels_for(len(ids), "mixed", 1) if arm.get("volume") == "v" else None
    w = lambda bk: ProsodyStream(m, arm.get("pitch"), arm.get("tempo"), contour, enc, arm.get("formant"), vol, bk) \
        if (bk is not None or arm) else None
    return enc, contour, w


@pytest.mark.parametrize("quality", QUALITIES)
def test_streams_equal_the_contract(voices, quality):
    m = voices(quality)
    rate = m.audio_output_info().sample_rate
    ids = list(workload.synthetic_ids(120, utt=7))
    bk = breaks_for(len(ids), "wild", 2)
    bk[0], bk[-1] = 30.0, 200.0
    for arm in STREAM_ARMS:
        for cs, pad in ((45, 3), (72, 3), (4000, 3)):
            enc, contour, w = _streams(m, ids, 9, arm)
            plain_chunks = list(SpeechStreamer(enc, cs, pad, warp=w(None))) if arm else _plain(m, enc, cs, pad)
            plain = _cat(plain_chunks)
            ends = _stream_ends(m, enc, arm.get("pitch"), arm.get("tempo"), contour)
            ps = w(bk)
            np.testing.assert_array_equal(ps.bounds, br.delivered_ends(ends, bk, rate))
            chunks = list(SpeechStreamer(enc, cs, pad, warp=ps))
            assert len(chunks) == len(plain_chunks), (arm, cs)
            got = _cat(chunks)
            assert got.tobytes() == br.apply(plain, ends, bk, rate).tobytes(), (arm, cs)
            assert ps.last_break_ms() > 0
            if quality == "medium" and cs == 45:
                # an output rate: the contract, then the resampler; bounds at the delivered rate
                st = SpeechStreamer(enc, cs, pad, Resampler(m, 16000), warp=w(bk))
                rs = _cat(list(st))
                assert rs.tobytes() == debug_resample(br.apply(plain, ends, bk, rate), rate, 16000).tobytes(), arm
                np.testing.assert_array_equal(st.bounds, -((-br.delivered_ends(ends, bk, rate) * 320) // 441))
                # G.711 of the f32 chunks of the same stream after its gain
                f32 = list(SpeechStreamer(enc, cs, pad, warp=w(bk)))
                g711 = list(SpeechStreamer(enc, cs, pad, encoding="alaw", gain=0.4, warp=w(bk)))
                assert len(g711) == len(f32)
                for g, f in zip(g711, f32):
                    assert g == gr.encode_bytes(AudioSamples(f.as_slice() * np.float32(0.4)).to_i16_vec(), "alaw")


def test_bounds_equal_the_batch_path(voices):
    m = voices("medium")
    ids = list(workload.synthetic_ids(90, utt=3))
    bk = breaks_for(len(ids), "every10")
    for kw in (dict(), dict(tempos=[1.3]), dict(pitches=[0.8])):
        j, audio = _job(m, [ids], [4], breaks=[bk], **kw)
        enc = m.infer_encoder_batch([ids], seeds=[4])[0]
        ps = ProsodyStream(m, (kw.get("pitches") or [None])[0], (kw.get("tempos") or [None])[0], enc=enc, breaks=bk)
        np.testing.assert_array_equal(ps.bounds, j.prosody_bounds()[0])
        assert ps.bounds[-1] == len(audio[0])


def test_stream_synthesis_and_stream_batch(voices):
    m = voices("medium")
    rate = m.audio_output_info().sample_rate
    _, src = m.phonemes_to_input_ids_map(LONG)
    cb = [250.0 if c % 10 == 9 else None for c in range(len(LONG))]
    per_id = np.array(_char_breaks_to_ids(cb, LONG, src, 0), np.float32)
    enc = m.infer_encoder_batch([m.phonemes_to_input_ids(LONG)], seeds=[4])[0]
    for kw in (dict(), dict(pitch=1.2), dict(formant_ratio=0.9, tempo=1.3)):
        plain = _cat(list(m.stream_synthesis(LONG, 55, 3, seed=4, **kw))) if kw else _cat(_plain(m, enc, 55, 3))
        ends = _stream_ends(m, enc, kw.get("pitch"), kw.get("tempo"))
        st = m.stream_synthesis(LONG, 55, 3, seed=4, breaks=cb, **kw)
        got = _cat(list(st))
        assert got.tobytes() == br.apply(plain, ends, per_id, rate).tobytes(), kw
        np.testing.assert_array_equal(st.bounds, br.delivered_ends(ends, per_id, rate))
    # StreamBatch: a paused stream beside plain, resampled, G.711 and metered streams equals itself alone
    sb = StreamBatch(m, 40, 3)
    mixed = [(LONG, dict(breaks=cb)), (SHORT, dict()), (LONG, dict(breaks=cb, output_rate=16000)),
             (SHORT, dict(encoding="mulaw", gain=0.5, breaks=[None] * (len(SHORT) - 1) + [100.0])),
             (LONG, dict(live_loudness=-20.0, breaks=cb))]
    keys = [sb.add(ph, seed=20 + i, **kw) for i, (ph, kw) in enumerate(mixed)]
    got = _drain(sb)
    for i, (ph, kw) in enumerate(mixed):
        assert _same(got[keys[i]], list(m.stream_synthesis(ph, 40, 3, seed=20 + i, **kw))), (i, kw)


def test_metered_stream_meters_the_paused_signal(voices):
    m = voices("medium")
    rate = m.audio_output_info().sample_rate
    ids = m.phonemes_to_input_ids(LONG)
    bk = breaks_for(len(ids), "every10")
    enc = m.infer_encoder_batch([ids], seeds=[6])[0]
    plain_chunks = _plain(m, enc, 55, 3)
    paused = br.apply(_cat(plain_chunks), _stream_ends(m, enc), bk, rate)
    got = list(SpeechStreamer(enc, 55, 3, warp=ProsodyStream(m, enc=enc, breaks=bk), meter=LoudnessStream(m, -18.0)))
    assert len(got) == len(plain_chunks)
    lens = np.array([len(c.as_slice()) for c in got], np.uint64)
    y = np.zeros(int(lens.sum()), np.float32)
    steps = int(lens.sum()) // ((rate + 5) // 10) + 2
    lufs, gains, clipped = np.zeros(steps), np.zeros(steps, np.float32), C.c_int64()
    err = N.sb200_error()
    rc = N.lib().sb200_debug_loudness_stream(0, f32p(paused), lens.ctypes.data_as(C.POINTER(C.c_size_t)), len(lens),
                                             rate, -18.0, 20.0, f32p(y), lufs.ctypes.data_as(C.POINTER(C.c_double)),
                                             f32p(gains), C.byref(clipped), C.byref(err))
    assert rc == 0
    assert _cat(got).tobytes() == y.tobytes()


def test_stream_neutral_breaks_are_the_stream_without_them(voices):
    m = voices("medium")
    ids = m.phonemes_to_input_ids(SHORT)
    enc = m.infer_encoder_batch([ids], seeds=[2])[0]
    lib = N.lib()

    def run(make):
        n0 = lib.sb200_launch_count()
        out = list(SpeechStreamer(enc, 40, 3, warp=make()))
        return out, lib.sb200_launch_count() - n0
    a, na = run(lambda: ProsodyStream(m, 1.25, enc=enc, breaks=[NAN] * len(ids)))
    b, nb = run(lambda: ProsodyStream(m, 1.25))
    c, nc = run(lambda: ProsodyStream(m, 1.25, enc=enc, breaks=[0.01] * len(ids)))
    assert _same(a, b) and _same(b, c) and na == nb == nc
