"""GPU (-m gpu): formant ratios on realtime streams.

The contract: the concatenation of a formant stream's chunks equals, bit for bit, the y of sb200_debug_formant over the
concatenation of the chunks the same stream yields without phi (after the device post-path), with the stream's pitch,
tempo, contour (ends = 256 C_i) and phi; with an output rate, sb200_debug_resample of that; with i16 and G.711, each
chunk converted as the resampled route converts its chunks.  A phi that asks for nothing is the stream without it, in
bits and launches; streams sharing a pass equal themselves alone."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import formant_reference as fr
import formant_stream_reference as fsr
import g711_reference as gr
import prosody_stream_reference as psr
from test_prosody_contour_stream_gpu import KINDS, constructed
from test_prosody_contour_stream_host import _ends, contours
from test_prosody_stream_gpu import LONG, SHORT, _cat, _drain, _plain, _same, _schedule, debug_resample, voices
from sonata_b200 import OperationError, workload
from sonata_b200 import _native as N
from sonata_b200.core import AudioSamples
from sonata_b200.piper import ProsodyStream, Resampler, SpeechStreamer, StreamBatch
from sonata_b200.synth import AudioOutputConfig, RealtimeBatch, SonataSpeechSynthesizer

pytestmark = pytest.mark.gpu
NAN = float("nan")
QUALITIES = ("x_low", "low", "medium", "high")
f32p = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
i64p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))
_nan = lambda v: NAN if v is None else float(v)


def _message(err):
    return C.string_at(err.message).decode() if err.message else ""


def debug_formant(x, rate, phi, pitch=None, tempo=None, ends=None, ratios=None):
    """y of sb200_debug_formant over the whole buffer."""
    x = np.ascontiguousarray(x, np.float32)
    cap = 3 * len(x) + 4096
    pre, y = np.zeros(cap, np.float32), np.zeros(cap, np.float32)
    n2, err = C.c_int64(), N.sb200_error()
    e = None if ends is None else np.ascontiguousarray(ends, np.int64)
    r = None if ratios is None else np.ascontiguousarray(ratios, np.float32)
    rc = N.lib().sb200_debug_formant(0, f32p(x), len(x), rate, _nan(pitch), _nan(tempo), None if e is None else i64p(e),
                                     None if r is None else f32p(r), 0 if e is None else len(e), _nan(phi), f32p(pre),
                                     f32p(y), cap, C.byref(n2), C.byref(err))
    assert rc == 0, _message(err)
    return y[:n2.value]


def debug_formant_stream(x, lens, rate, phi, pitch=None, tempo=None, ends=None, ratios=None):
    """(joined output, per-chunk counts) of a fresh formant stream fed x in chunks of lens."""
    x = np.ascontiguousarray(x, np.float32)
    lens = np.ascontiguousarray(lens, np.int64)
    cap = 3 * len(x) + 4096
    y, got, err = np.zeros(cap, np.float32), np.zeros(len(lens), np.int64), N.sb200_error()
    e = None if ends is None else np.ascontiguousarray(ends, np.int64)
    r = None if ratios is None else np.ascontiguousarray(ratios, np.float32)
    rc = N.lib().sb200_debug_formant_stream(0, f32p(x), i64p(lens), len(lens), rate, _nan(pitch), _nan(tempo),
                                            None if e is None else i64p(e), None if r is None else f32p(r),
                                            0 if e is None else len(e), _nan(phi), f32p(y), cap, i64p(got),
                                            C.byref(err))
    assert rc == 0, _message(err)
    return y[:int(got.sum())], got


RAW = [(None, None, 1.2), (1.25, None, 1.0), (0.8, 2.0, 1.0), (None, 1.5, 0.8), (2.0, 0.5, 1.3)]


@pytest.mark.parametrize("rate", (22050, 16000))
@pytest.mark.parametrize("pitch,tempo,phi", RAW)
def test_raw_push_equals_the_whole_signal(lib_built, rate, pitch, tempo, phi):
    n = int(0.7 * rate) + 77                        # not a multiple of H
    kind = KINDS[RAW.index((pitch, tempo, phi)) % len(KINDS)]
    x = constructed(kind, n, rate, seed=rate + n)
    want = debug_formant(x, rate, phi, pitch, tempo)
    chunkings = dict(psr.chunkings(n, rate), short=[200] * (n // 200) + [n % 200])
    for name, lens in chunkings.items():
        y, got = debug_formant_stream(x, lens, rate, phi, pitch, tempo)
        np.testing.assert_array_equal(got, [r["emitted"] for r in fsr.stream(rate, pitch, tempo, phi, lens)],
                                      err_msg=name)
        assert y.tobytes() == want.tobytes(), (kind, name)


def test_raw_push_single_samples_and_short_signals(lib_built):
    rate = 16000
    x = constructed("sweep", 5000, rate, 1)
    for pitch, tempo, phi in ((None, None, 1.25), (1.5, None, 1.0)):
        y, _ = debug_formant_stream(x, [1] * len(x), rate, phi, pitch, tempo)
        assert y.tobytes() == debug_formant(x, rate, phi, pitch, tempo).tobytes(), (pitch, phi)
    for n in (1, 300, 1023, 1025):
        xs = constructed("clipped", n, rate, n)
        for lens in ([n], [n // 2, n - n // 2]):
            y, _ = debug_formant_stream(xs, lens, rate, 0.7)
            assert y.tobytes() == debug_formant(xs, rate, 0.7).tobytes(), (n, lens)


@pytest.mark.parametrize("rate", (22050, 16000))
@pytest.mark.parametrize("name", ["question", "alternating", "zero_frames"])
def test_raw_push_contour(lib_built, rate, name):
    frames, ratios = contours()[name]
    n, ends = _ends(frames)
    x = constructed(KINDS[len(name) % 3], n, rate, seed=n)
    for tempo, phi in ((None, 1.0), (0.8, 1.2)):
        want = debug_formant(x, rate, phi, None, tempo, ends, ratios)
        for cname, lens in psr.chunkings(n, rate).items():
            y, got = debug_formant_stream(x, lens, rate, phi, None, tempo, ends, ratios)
            np.testing.assert_array_equal(got, [r["emitted"] for r in fsr.stream(rate, None, tempo, phi, lens, ends,
                                                                                  ratios)], err_msg=cname)
            assert y.tobytes() == want.tobytes(), (cname, tempo, phi)


def _plain_join(m, ids, seed, cs, pad):
    return _cat(_plain(m, m.infer_encoder_batch([ids], seeds=[seed])[0], cs, pad))


def _streamer(m, ids, seed, cs, pad, **kw):
    return SpeechStreamer(m.infer_encoder_batch([ids], seeds=[seed])[0], cs, pad, **kw)


@pytest.mark.parametrize("quality", QUALITIES)
def test_decoder_path_on_every_voice(voices, quality):
    m = voices(quality)
    rate = m.audio_output_info().sample_rate
    ids = list(workload.synthetic_ids(120, utt=7))
    for cs, pad in ((55, 3), (72, 3), (4000, 3)):           # 4000: one-shot
        plain = _plain_join(m, ids, 9, cs, pad)
        # formant only: the post-path chunks of a NULL resampler, then the stage
        got = list(_streamer(m, ids, 9, cs, pad, warp=ProsodyStream(m, formant=1.2)))
        assert _cat(got).tobytes() == debug_formant(plain, rate, 1.2).tobytes(), (cs, "formant only")
        for p, t, phi in ((1.25, None, 1.0), (0.8, 1.5, 1.0), (None, 0.8, 1.1)):
            got = list(_streamer(m, ids, 9, cs, pad, warp=ProsodyStream(m, p, t, formant=phi)))
            assert _cat(got).tobytes() == debug_formant(plain, rate, phi, p, t).tobytes(), (cs, p, t, phi)
    # stream_synthesis with a contour and phi
    enc = m.infer_encoder_batch([m.phonemes_to_input_ids(LONG)], seeds=[4])[0]
    plain = _cat(_plain(m, enc, 55, 3))
    cc = [1.0] * len(LONG)
    cc[-6:] = [1.3] * 6
    st = m.stream_synthesis(LONG, 55, 3, seed=4, pitch_contour=cc, formant_ratio=1.0)
    got = _cat(list(st))
    _, src = m.phonemes_to_input_ids_map(LONG)
    from sonata_b200.piper import _char_values_to_ids, _contour_value
    ratios = [NAN if v is None else v for v in _char_values_to_ids(cc, LONG, src, 0, "pitch ratios", _contour_value)]
    ends = 256 * np.cumsum(enc.p_duration)
    assert got.tobytes() == debug_formant(plain, rate, 1.0, None, None, ends, ratios).tobytes()
    assert st.bounds[-1] == len(got)


def test_composition_with_rates_i16_and_g711(voices):
    m = voices("medium")
    rate = m.audio_output_info().sample_rate
    ids = list(workload.synthetic_ids(150, utt=3))
    enc = m.infer_encoder_batch([ids], seeds=[5])[0]
    plain = _cat(_plain(m, enc, 55, 3))
    for p, phi in ((1.25, 1.0), (None, 0.8)):
        whole = debug_formant(plain, rate, phi, p)
        f32 = list(_streamer(m, ids, 5, 55, 3, warp=ProsodyStream(m, p, formant=phi)))
        assert _cat(f32).tobytes() == whole.tobytes()
        for out_rate in (16000, 48000, 8000):
            rs = list(_streamer(m, ids, 5, 55, 3, warp=ProsodyStream(m, p, formant=phi),
                                resampler=Resampler(m, out_rate)))
            assert _cat(rs).tobytes() == debug_resample(whole, rate, out_rate).tobytes(), (p, out_rate)
        w = ProsodyStream(m, p, formant=phi)
        got = [m.infer_decoder_batch([c], fade=f, pcm16=True, warps=[w], last=[last])[0]
               for c, f, last in _schedule(enc, 55, 3)]
        assert len(got) == len(f32)
        for g, f in zip(got, f32):
            np.testing.assert_array_equal(g, AudioSamples(f.as_slice()).to_i16_vec())
        for law in ("mulaw", "alaw"):
            g711 = list(_streamer(m, ids, 5, 55, 3, warp=ProsodyStream(m, p, formant=phi), encoding=law, gain=0.3))
            assert len(g711) == len(f32)
            for g, f in zip(g711, f32):
                assert g == gr.encode_bytes(AudioSamples(f.as_slice() * np.float32(0.3)).to_i16_vec(), law)


def _launches(m, make, ids, seed=2):
    lib = N.lib()
    enc = m.infer_encoder_batch([ids], seeds=[seed])[0]
    w = make()
    st = SpeechStreamer(enc, 40, 3, warp=w)
    n0 = lib.sb200_launch_count()
    out = list(st)
    return out, lib.sb200_launch_count() - n0


def test_equivalences(voices):
    m = voices("medium")
    ids = m.phonemes_to_input_ids(LONG)
    # phi equal to the pitch ratio: the ratio stream's chunks, counts and launches
    a, na = _launches(m, lambda: ProsodyStream(m, 1.25, formant=1.25), ids)
    b, nb = _launches(m, lambda: ProsodyStream(m, 1.25), ids)
    assert _same(a, b) and na == nb
    # a neutral phi on a plain stream is the plain stream (stream_synthesis makes none)
    plain = list(m.stream_synthesis(LONG, 40, 3, seed=2))
    assert _same(list(m.stream_synthesis(LONG, 40, 3, seed=2, formant_ratio=1.0)), plain)
    assert _same(list(m.stream_synthesis(LONG, 40, 3, seed=2, formant_ratio=NAN)), plain)
    # a uniform contour with phi is the ratio stream with phi
    enc = m.infer_encoder_batch([ids], seeds=[2])[0]
    uni = list(SpeechStreamer(enc, 40, 3, warp=ProsodyStream(m, None, None, [1.25] * len(ids), enc, formant=1.0)))
    ratio = list(_streamer(m, ids, 2, 40, 3, warp=ProsodyStream(m, 1.25, formant=1.0)))
    assert _same(uni, ratio)
    # with phi that asks, each pass adds the formant region's staging, and its stage when it emits a hop
    c, nc = _launches(m, lambda: ProsodyStream(m, 1.25, formant=1.0), ids)
    passes = len(c)
    assert passes < nc - nb <= 2 * passes, (nc, nb, passes)


MIXED = [(LONG, dict(formant_ratio=1.2)), (LONG, dict()), (SHORT, dict(pitch=1.25, formant_ratio=1.0)),
         (LONG, dict(pitch=0.8, tempo=1.5, output_rate=16000, formant_ratio=1.0)), (LONG, dict(tempo=0.8)),
         (SHORT, dict(formant_ratio=0.8, encoding="mulaw", gain=0.5)), (LONG, dict(pitch=1.25)),
         (LONG, dict(output_rate=16000)), (SHORT, dict(pitch=1.25, formant_ratio=1.25))]


def test_stream_batch_mixes_formant_warped_and_plain_streams(voices):
    m = voices("medium")
    sb = StreamBatch(m, 40, 3)
    keys = [sb.add(ph, seed=10 + i, **kw) for i, (ph, kw) in enumerate(MIXED)]
    got = _drain(sb)
    for i, (ph, kw) in enumerate(MIXED):
        assert _same(got[keys[i]], list(m.stream_synthesis(ph, 40, 3, seed=10 + i, **kw))), (i, kw)
    # the streams without phi keep their passes and bits without the formant streams
    sb = StreamBatch(m, 40, 3)
    rest = [i for i, (_, kw) in enumerate(MIXED) if "formant_ratio" not in kw]
    keys2 = [sb.add(MIXED[i][0], seed=10 + i, **MIXED[i][1]) for i in rest]
    got2 = _drain(sb)
    for i, k2 in zip(rest, keys2):
        assert _same(got[keys[i]], got2[k2]), i


def test_realtime_batch_equals_synthesize_streamed(voices):
    m = voices("medium")
    synth = SonataSpeechSynthesizer(m)
    text = LONG + "\n" + SHORT + "\n" + LONG
    oc = AudioOutputConfig(None, 80, None, 30)
    for kw in (dict(formant_ratio=1.2), dict(pitch_ratio=1.25, formant_ratio=1.0, output_rate=16000)):
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
    for make, p in ((lambda mm: ProsodyStream(mm, formant=1.2), None), (lambda mm: ProsodyStream(mm, 1.25, formant=1.0),
                                                                      1.25)):
        w = make(m)
        out = [m.infer_decoder_batch([chunks[0]], fade=42, warps=[w], last=[False])[0]]
        with pytest.raises(OperationError, match="chunk 1: the prosody stream of chunk 0 appears twice"):
            m.infer_decoder_batch([chunks[1], chunks[1]], fade=42, warps=[w, w], last=[False, False])
        with pytest.raises(OperationError, match="chunk 0: the prosody stream was made for another voice"):
            m.infer_decoder_batch([chunks[1]], fade=42, warps=[make(voices("low"))])
        out.append(m.infer_decoder_batch([chunks[1]], fade=42, warps=[w], last=[False])[0])
        out.append(m.infer_decoder_batch([chunks[2]], fade=42, warps=[w], last=[True])[0])
        with pytest.raises(OperationError, match="chunk 0: the prosody stream has already been flushed"):
            m.infer_decoder_batch([chunks[2]], fade=42, warps=[w], last=[True])
        plain = m.infer_decoder_batch(chunks, fade=42, resamplers=[None] * 3)
        phi = 1.2 if p is None else 1.0
        assert _cat(out).tobytes() == debug_formant(_cat(plain), rate, phi, p).tobytes()
        assert w.last_formant_ms() > 0.0
    with pytest.raises(OperationError, match="asks for"):
        ProsodyStream(m, formant=1.0)
    with pytest.raises(OperationError, match="formant ratio 3.0"):
        ProsodyStream(m, 1.25, formant=3.0)


@pytest.mark.parametrize("rate,pitch", [(22050, 1.25), (22050, 1.5), (16000, 1.5)])
def test_formants_kept_through_a_pitch_stream(lib_built, rate, pitch):
    """A pitch stream with phi = 1 keeps the vowel's LPC formants within 10 %, as the batch stage does
    (test_formant_host), and moves F0 by the pitch.  (At 16 kHz and pitch 1.25 the 120 Hz vowel's F1 measures 11 %
    high, batch and stream alike: its harmonics 150 Hz apart leave the LPC fit few points near 700 Hz.)"""
    x = fr.vowel(rate)
    src = fr.lpc_formants(x, rate)
    lens = [1000] * (len(x) // 1000) + [len(x) % 1000]
    y, _ = debug_formant_stream(x, lens, rate, 1.0, pitch)
    assert y.tobytes() == debug_formant(x, rate, 1.0, pitch).tobytes()
    got = fr.lpc_formants(y, rate)
    assert len(got) == 3 and np.all(np.abs(got / src - 1.0) < 0.10), (src, got)
    f0 = fr.f0_from_harmonics(y, rate, 120.0 * pitch)
    assert abs(f0 / (pitch * fr.f0_from_harmonics(x, rate, 120.0)) - 1.0) < 0.01, f0
