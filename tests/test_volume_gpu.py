"""GPU (-m gpu): volume contours (include/sonata_b200.h, sb200_speak_batch_ids_volume and
sb200_prosody_stream_create_volume).

Everything is bit for bit against tests/volume_reference.py: the test hook; a contoured batch against the contract
applied to the same seeded batch without the contour (with pitch, tempo, pitch contours, formants and blends, an output
rate and a loudness target); one piece, neutral contours and batch independence; and streams of every kind joined
against the contract applied to the joined chunks of the same stream without it."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import g711_reference as gr
import volume_reference as vr
from test_prosody_stream_gpu import LONG, SHORT, _cat, _drain, _plain, _same, debug_resample, voices  # noqa: F401
from sonata_b200 import _native as N, voicegen, workload
from sonata_b200.core import AudioSamples
from sonata_b200.job import SynthesisJob
from sonata_b200.piper import (LoudnessStream, PiperSynthesisConfig, ProsodyStream, Resampler, SpeechStreamer,
                               StreamBatch, VitsStreamingModel, _char_values_to_ids, _contour_value, _volume_value)

pytestmark = pytest.mark.gpu
NAN, INF = float("nan"), float("inf")
QUALITIES = ("x_low", "low", "medium", "high")
f32p = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
i64p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))


def _message(err):
    return C.string_at(err.message).decode() if err.message else ""


def debug_volume(x, ends, levels, rate):
    x = np.ascontiguousarray(x, np.float32)
    e, lv = np.ascontiguousarray(ends, np.int64), np.ascontiguousarray(levels, np.float32)
    y, err = np.zeros_like(x), N.sb200_error()
    rc = N.lib().sb200_debug_volume(0, f32p(x), x.size, i64p(e), f32p(lv), e.size, rate, f32p(y), C.byref(err))
    assert rc == 0, _message(err)
    return y


def debug_loudness(x, rate):
    x = np.ascontiguousarray(x, np.float32)
    out, err = C.c_double(), N.sb200_error()
    assert N.lib().sb200_debug_loudness(0, f32p(x), x.size, rate, C.byref(out), C.byref(err)) == 0, _message(err)
    return out.value


def levels_for(n_ids, kind, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "span":                  # +6 dB over 10 % of the ids
        v = np.full(n_ids, NAN, np.float32)
        a = n_ids // 3
        v[a:a + max(1, n_ids // 10)] = 6.0
        return v
    if kind == "mixed":                 # per id from {-6, 0, +6}
        return rng.choice(np.array([-6.0, 0.0, 6.0], np.float32), n_ids)
    if kind == "mute":                  # one word muted, the rest raised a little
        v = np.full(n_ids, 1.5, np.float32)
        v[n_ids // 2:n_ids // 2 + 3] = -INF
        return v
    if kind == "wild":                  # short runs and every kind of value
        return rng.choice(np.array([NAN, 0.0, -60.0, 20.0, -INF, 3.25, -0.5], np.float32), n_ids)
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
            ends[-1] = 1
        x = (rng.standard_normal(int(ends[-1])) * 0.7).astype(np.float32)
        x[::97] = 1.5                   # above full scale: no clamp
        for kind in ("span", "mixed", "mute", "wild"):
            lv = levels_for(n_ids, kind, trial)
            got = debug_volume(x, ends, lv, rate)
            assert got.tobytes() == vr.apply(x, ends, lv, rate).tobytes(), (trial, kind)
    # one piece, and a neutral contour
    x = rng.standard_normal(5000).astype(np.float32)
    ends = np.array([1000, 1000, 5000])
    assert debug_volume(x, ends, [-9.5] * 3, rate).tobytes() == (x * vr.gain_of(-9.5)).tobytes()
    assert debug_volume(x, ends, [NAN, 0.0, NAN], rate).tobytes() == x.tobytes()


# ---------------------------------------------------------------------------------------------------- batches
def _job(m, batches, seeds, **kw):
    j = SynthesisJob(m, batches, seeds=seeds, **kw)
    j.run()
    out = [a.samples.as_slice().copy() for a in j.fetch()]
    return j, out


ARMS = [dict(), dict(pitches=[1.25, None, 0.8]), dict(tempos=[1.5, None, 0.7]),
        dict(pitches=[1.2, 0.9, None], tempos=[None, 1.3, 0.8], formants=[1.0, 1.1, None]),
        dict(pitch_contours="q"), dict(formants=[1.2, None, 0.9])]


def _arm(kw, lens):
    kw = dict(kw)
    if kw.get("pitch_contours") == "q":
        kw["pitch_contours"] = [np.where(np.arange(n) > 2 * n // 3, 1.3, 1.0).astype(np.float32) if b != 1 else None
                                for b, n in enumerate(lens)]
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
        vols = [levels_for(n, k, i) for n, k in zip(lens, ("span", "mixed", "wild"))]
        vols[i % 3] = None if i % 2 else vols[i % 3]
        jv, got = _job(m, batches, seeds, volume_contours=vols, **kw)
        for b in range(3):
            want = base[b] if vols[b] is None else vr.apply(base[b], ends[b], vols[b], rate)
            assert got[b].tobytes() == want.tobytes(), (i, b)
        assert any(r["name"] == "volume" and r["launches"] == 1 for r in jv.profile())
        # with an output rate: the contract at the voice's rate, then the resampler
        _, rs = _job(m, batches, seeds, volume_contours=vols, output_rates=[16000, None, 48000], **kw)
        for b, r in enumerate((16000, None, 48000)):
            want = base[b] if vols[b] is None else vr.apply(base[b], ends[b], vols[b], rate)
            if r and r != rate:
                want = debug_resample(want, rate, r)
            assert rs[b].tobytes() == want.tobytes(), (i, b, r)


def test_loudness_normalises_the_contoured_utterance(voices):
    m = voices("medium")
    rate = m.audio_output_info().sample_rate
    batches = [list(workload.synthetic_ids(150, utt=b + 1)) for b in range(2)]
    vols = [levels_for(len(batches[0]), "mute"), levels_for(len(batches[1]), "span")]
    jb, base = _job(m, batches, [3, 4])
    ends = jb.prosody_bounds()
    jv, got = _job(m, batches, [3, 4], volume_contours=vols, loudness=[-23.0, -16.0])
    lufs, gain = jv.loudness()
    for b in range(2):
        contoured = vr.apply(base[b], ends[b], vols[b], rate)
        assert lufs[b] == debug_loudness(contoured, rate)
        assert got[b].tobytes() == (contoured * gain[b]).astype(np.float32).tobytes()
    # the contour's relative levels survive: the muted word stays silent
    assert np.all(got[0][ends[0][len(ends[0]) // 2 + 1] + rate // 200:ends[0][len(ends[0]) // 2 + 2] - rate // 200] == 0)


def test_one_piece_neutral_and_batch_independence(voices):
    m = voices("low")
    rate = m.audio_output_info().sample_rate
    batches = [list(workload.synthetic_ids(90 + 30 * b, utt=b + 5)) for b in range(3)]
    lens = [len(b) for b in batches]
    _, base = _job(m, batches, [1, 2, 3])
    # one piece: the utterance times its gain
    _, one = _job(m, batches, [1, 2, 3], volume_contours=[[-7.5] * n for n in lens])
    for b in range(3):
        assert one[b].tobytes() == (base[b] * vr.gain_of(-7.5)).tobytes()
    # neutral: the same bits and launches
    lib = N.lib()
    n0 = lib.sb200_launch_count()
    _, plain = _job(m, batches, [1, 2, 3])
    n1 = lib.sb200_launch_count()
    _, neutral = _job(m, batches, [1, 2, 3], volume_contours=[[NAN] * n if b else [0.0] * n for b, n in enumerate(lens)])
    n2 = lib.sb200_launch_count()
    # levels that ask but round to gain 1 reach the library, which plans no piece
    _, tiny = _job(m, batches, [1, 2, 3], volume_contours=[[1e-9] * n for n in lens])
    n3 = lib.sb200_launch_count()
    assert n2 - n1 == n1 - n0 == n3 - n2
    assert all(a.tobytes() == b.tobytes() == c.tobytes() for a, b, c in zip(neutral, plain, tiny))
    # a contoured utterance has the same bits alone and in any batch
    vols = [levels_for(n, "wild", b) for b, n in enumerate(lens)]
    _, mixed = _job(m, batches, [1, 2, 3], volume_contours=vols, pitches=[None, 1.3, None])
    for b in range(3):
        _, alone = _job(m, [batches[b]], [b + 1], volume_contours=[vols[b]], pitches=[[None, 1.3, None][b]])
        assert alone[0].tobytes() == mixed[b].tobytes(), b


def test_blends_and_the_phoneme_surfaces(lib_built):
    d = voicegen.default_voice_dir()
    m = VitsStreamingModel(voicegen.write_voice(d, "medium", n_speakers=4), device=0)
    m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.667, 1.0, 0.8))
    rate = m.audio_output_info().sample_rate
    try:
        ph = [LONG, SHORT]
        maps = [m.phonemes_to_input_ids_map(p) for p in ph]
        batches = [ids for ids, _ in maps]
        blends = [{0: 0.3, 2: 0.7}, None]
        cv = [[6.0 if i % 7 == 3 else None for i in range(len(LONG))], [-INF, 0.0] + [-3.0] * (len(SHORT) - 2)]
        per_id = [np.array([NAN if v is None else v for v in _char_values_to_ids(c, p, src, 0, "volume levels",
                                                                                  _volume_value, 0.0)], np.float32)
                  for c, p, (_, src) in zip(cv, ph, maps)]
        jb, base = _job(m, batches, [7, 8], speaker_blends=blends, tempos=[1.2, None])
        ends = jb.prosody_bounds()
        got = m.speak_batch(ph, seeds=[7, 8], speaker_blends=blends, tempos=[1.2, None], volume_contours=cv)
        al = m.speak_batch_with_alignment(ph, seeds=[7, 8], speaker_blends=blends, tempos=[1.2, None],
                                          volume_contours=cv)
        plain_al = m.speak_batch_with_alignment(ph, seeds=[7, 8], speaker_blends=blends, tempos=[1.2, None])
        for b in range(2):
            want = vr.apply(base[b], ends[b], per_id[b], rate)
            assert got[b].samples.as_slice().tobytes() == want.tobytes(), b
            assert al[b][0].samples.as_slice().tobytes() == want.tobytes(), b
            assert [(a.start_sample, a.num_samples) for a in al[b][1]] == \
                [(a.start_sample, a.num_samples) for a in plain_al[b][1]]
        got = m.infer_batch_with_values(batches, seeds=[7, 8], speaker_blends=blends, tempos=[1.2, None],
                                        volume_contours=per_id)
        assert all(g.samples.as_slice().tobytes() == vr.apply(base[b], ends[b], per_id[b], rate).tobytes()
                   for b, g in enumerate(got))
    finally:
        m.close()


# ---------------------------------------------------------------------------------------------------- streams
def _stream_ends(m, enc, pitch=None, tempo=None, contour=None):
    """Each id's delivered end as the batch path gives it for enc's sentence with these ratios or contour."""
    rate = m.audio_output_info().sample_rate
    ends = 256 * np.cumsum(np.asarray(enc.p_duration, np.int64))
    n = 256 * enc.num_frames
    ratios = np.full(len(ends), NAN if pitch is None else pitch, np.float32) if contour is None else \
        np.asarray(contour, np.float32)
    shape, bounds = np.zeros(6, np.int64), np.zeros(len(ends), np.int64)
    t = NAN if tempo is None else tempo
    assert N.lib().sb200_debug_prosody_contour_plan(rate, n, i64p(ends), f32p(ratios), len(ends), t, i64p(shape), None,
                                                    0, i64p(bounds)) == 0
    return bounds


STREAM_ARMS = [dict(), dict(pitch=1.25), dict(tempo=1.4, pitch=0.9), dict(formant=1.2), dict(contour="q"),
               dict(contour="q", tempo=0.8, formant=1.0)]


def _streams(m, ids, seed, arm):
    enc = m.infer_encoder_batch([ids], seeds=[seed])[0]
    contour = None
    if arm.get("contour") == "q":
        contour = np.where(np.arange(len(ids)) > len(ids) // 2, 1.3, NAN).astype(np.float32)
    w = lambda v: ProsodyStream(m, arm.get("pitch"), arm.get("tempo"), contour, enc, arm.get("formant"), v) \
        if (v is not None or arm) else None
    return enc, contour, w


@pytest.mark.parametrize("quality", QUALITIES)
def test_streams_equal_the_contract(voices, quality):
    m = voices(quality)
    rate = m.audio_output_info().sample_rate
    ids = list(workload.synthetic_ids(120, utt=7))
    vol = levels_for(len(ids), "mixed", 1)
    for arm in STREAM_ARMS:
        for cs, pad in ((45, 3), (72, 3), (4000, 3)):
            enc, contour, w = _streams(m, ids, 9, arm)
            plain = _cat(list(SpeechStreamer(enc, cs, pad, warp=w(None)))) if arm else _cat(_plain(m, enc, cs, pad))
            ends = _stream_ends(m, enc, arm.get("pitch"), arm.get("tempo"), contour)
            st = SpeechStreamer(enc, cs, pad, warp=w(vol))
            got = _cat(list(st))
            assert got.tobytes() == vr.apply(plain, ends, vol, rate).tobytes(), (arm, cs)
            if quality == "medium" and cs == 45:
                # an output rate: the contract, then the resampler
                rs = _cat(list(SpeechStreamer(enc, cs, pad, Resampler(m, 16000), warp=w(vol))))
                assert rs.tobytes() == debug_resample(vr.apply(plain, ends, vol, rate), rate, 16000).tobytes(), arm
                # G.711 of the f32 chunks of the same stream after its gain
                f32 = list(SpeechStreamer(enc, cs, pad, warp=w(vol)))
                g711 = list(SpeechStreamer(enc, cs, pad, encoding="alaw", gain=0.4, warp=w(vol)))
                assert len(g711) == len(f32)
                for g, f in zip(g711, f32):
                    assert g == gr.encode_bytes(AudioSamples(f.as_slice() * np.float32(0.4)).to_i16_vec(), "alaw")


def test_stream_synthesis_and_stream_batch(voices):
    m = voices("medium")
    rate = m.audio_output_info().sample_rate
    _, src = m.phonemes_to_input_ids_map(LONG)
    cv = [(-6.0, 0.0, 6.0)[c % 3] for c in range(len(LONG))]
    per_id = np.array(_char_values_to_ids(cv, LONG, src, 0, "volume levels", _volume_value, 0.0), np.float32)
    cc = [None] * len(LONG)
    cc[-8:] = [1.25] * 8
    ratios = np.array([NAN if v is None else v for v in _char_values_to_ids(cc, LONG, src, 0, "pitch ratios",
                                                                             _contour_value)], np.float32)
    enc = m.infer_encoder_batch([m.phonemes_to_input_ids(LONG)], seeds=[4])[0]
    for kw, contour in ((dict(), None), (dict(pitch=1.2), None), (dict(pitch_contour=cc), ratios),
                        (dict(formant_ratio=0.9, tempo=1.3), None)):
        plain = _cat(list(m.stream_synthesis(LONG, 55, 3, seed=4, **kw))) if kw else _cat(_plain(m, enc, 55, 3))
        ends = _stream_ends(m, enc, kw.get("pitch"), kw.get("tempo"), contour)
        got = _cat(list(m.stream_synthesis(LONG, 55, 3, seed=4, volume_contour=cv, **kw)))
        assert got.tobytes() == vr.apply(plain, ends, per_id, rate).tobytes(), kw
    # StreamBatch: a volume stream beside plain, resampled and G.711 streams equals itself alone
    sb = StreamBatch(m, 40, 3)
    mixed = [(LONG, dict(volume_contour=cv)), (SHORT, dict()), (LONG, dict(volume_contour=cv, output_rate=16000)),
             (SHORT, dict(encoding="mulaw", gain=0.5, volume_contour=[-3.0] * len(SHORT))),
             (LONG, dict(live_loudness=-20.0, volume_contour=cv))]
    keys = [sb.add(ph, seed=20 + i, **kw) for i, (ph, kw) in enumerate(mixed)]
    got = _drain(sb)
    for i, (ph, kw) in enumerate(mixed):
        assert _same(got[keys[i]], list(m.stream_synthesis(ph, 40, 3, seed=20 + i, **kw))), (i, kw)


def test_metered_stream_meters_the_contoured_signal(voices):
    m = voices("medium")
    rate = m.audio_output_info().sample_rate
    ids = m.phonemes_to_input_ids(LONG)
    vol = levels_for(len(ids), "mute")
    enc = m.infer_encoder_batch([ids], seeds=[6])[0]
    plain = _cat(_plain(m, enc, 55, 3))
    contoured = vr.apply(plain, _stream_ends(m, enc), vol, rate)
    got = list(SpeechStreamer(enc, 55, 3, warp=ProsodyStream(m, enc=enc, volume=vol), meter=LoudnessStream(m, -18.0)))
    lens = np.array([len(c.as_slice()) for c in got], np.uint64)
    y = np.zeros(int(lens.sum()), np.float32)
    steps = int(lens.sum()) // ((rate + 5) // 10) + 2
    lufs, gains, clipped = np.zeros(steps), np.zeros(steps, np.float32), C.c_int64()
    err = N.sb200_error()
    rc = N.lib().sb200_debug_loudness_stream(0, f32p(contoured), lens.ctypes.data_as(C.POINTER(C.c_size_t)), len(lens),
                                             rate, -18.0, 20.0, f32p(y), lufs.ctypes.data_as(C.POINTER(C.c_double)),
                                             f32p(gains), C.byref(clipped), C.byref(err))
    assert rc == 0, _message(err)
    assert _cat(got).tobytes() == y.tobytes()


def test_stream_neutral_contour_is_the_stream_without_it(voices):
    m = voices("medium")
    ids = m.phonemes_to_input_ids(SHORT)
    enc = m.infer_encoder_batch([ids], seeds=[2])[0]
    lib = N.lib()

    def run(make):
        n0 = lib.sb200_launch_count()
        out = list(SpeechStreamer(enc, 40, 3, warp=make()))
        return out, lib.sb200_launch_count() - n0
    a, na = run(lambda: ProsodyStream(m, 1.25, enc=enc, volume=[NAN] * len(ids)))
    b, nb = run(lambda: ProsodyStream(m, 1.25))
    assert _same(a, b) and na == nb
    # a uniform level on a ratio stream is that stream times its gain
    c, _ = run(lambda: ProsodyStream(m, 1.25, enc=enc, volume=[4.0] * len(ids)))
    assert _cat(c).tobytes() == (_cat(b) * vr.gain_of(4.0)).tobytes()
