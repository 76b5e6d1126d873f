"""GPU (-m gpu): pitch contours on realtime streams.

The contract: the concatenation of a contoured stream's chunks equals, bit for bit, sb200_debug_prosody_contour of the
concatenation of the chunks the same stream yields without a contour (after the device post-path), with n = 256 T_y and
ends = 256 C_i; with an output rate, sb200_debug_resample of that; with G.711, each chunk converted as the resampled
route converts its chunks.  A uniform contour is the ratio stream, a neutral one the plain stream, streams sharing a
pass equal themselves alone, and each id's delivered end is the batch path's."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import g711_reference as gr
import prosody_contour_reference as pcr
import prosody_contour_stream_reference as pcs
import prosody_stream_reference as psr
from test_prosody_contour_stream_host import TEMPOS, contours, question
from test_prosody_stream_gpu import LONG, SHORT, _cat, _drain, _plain, _same, debug_resample, voices
from sonata_b200 import OperationError, workload
from sonata_b200 import _native as N
from sonata_b200.core import AudioSamples
from sonata_b200.job import SynthesisJob
from sonata_b200.piper import ProsodyStream, SpeechStreamer, StreamBatch, _char_values_to_ids, _contour_value
from sonata_b200.synth import AudioOutputConfig, RealtimeBatch

pytestmark = pytest.mark.gpu
NAN = float("nan")
QUALITIES = ("x_low", "low", "medium", "high")

f32p = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
i64p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))


def _message(err):
    return C.string_at(err.message).decode() if err.message else ""


def debug_contour(x, rate, ends, ratios, tempo):
    """(y, offsets) of sb200_debug_prosody_contour over the whole buffer."""
    x = np.ascontiguousarray(x, np.float32)
    ends = np.ascontiguousarray(ends, np.int64)
    ratios = np.ascontiguousarray(ratios, np.float32)
    pl = pcr.plan(rate, len(x), ends, ratios, tempo)
    y = np.zeros(pl["n2"] + 1, np.float32)
    off = np.zeros(pl["F"] + 1, np.int32)
    err = N.sb200_error()
    rc = N.lib().sb200_debug_prosody_contour(0, f32p(x), x.size, rate, i64p(ends), f32p(ratios), len(ends),
                                             NAN if tempo is None else tempo, f32p(y), y.size,
                                             off.ctypes.data_as(C.POINTER(C.c_int32)), off.size, None, 0,
                                             C.byref(err))
    assert rc == 0, _message(err)
    return y[:pl["n2"]], off[:pl["F"]]


def debug_contour_stream(x, lens, rate, ends, ratios, tempo):
    """(y, per-chunk counts, offsets) of a fresh contoured stream fed x in chunks of lens."""
    x = np.ascontiguousarray(x, np.float32)
    lens = np.ascontiguousarray(lens, np.int64)
    ends = np.ascontiguousarray(ends, np.int64)
    ratios = np.ascontiguousarray(ratios, np.float32)
    pl = pcr.plan(rate, len(x), ends, ratios, tempo)
    y = np.zeros(pl["n2"] + 1, np.float32)
    got = np.zeros(len(lens), np.int64)
    off = np.zeros(pl["F"] + 1, np.int32)
    err = N.sb200_error()
    rc = N.lib().sb200_debug_prosody_contour_stream(0, f32p(x), i64p(lens), len(lens), rate, i64p(ends),
                                                    f32p(ratios), len(ends), NAN if tempo is None else tempo, f32p(y),
                                                    y.size, i64p(got), off.ctypes.data_as(C.POINTER(C.c_int32)),
                                                    off.size, C.byref(err))
    assert rc == 0, _message(err)
    return y[:pl["n2"]], got, off[:pl["F"]]


def constructed(kind, n, rate, seed):
    """Sweeps, silence and clipped runs."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / rate
    if kind == "sweep":
        f = 80 + 900 * t / max(t[-1], 1e-9)
        return (0.5 * np.sin(2 * np.pi * np.cumsum(f) / rate)).astype(np.float32)
    if kind == "silence_bursts":
        x = np.zeros(n, np.float32)
        for a in rng.integers(0, max(n - 3000, 1), 6):
            x[a:a + 2500] = 0.3 * rng.standard_normal(min(2500, n - a))
        return x
    x = 1.6 * np.sin(2 * np.pi * 150 * t) + 0.05 * rng.standard_normal(n)       # clipped by the quantiser: |x| > 1
    return x.astype(np.float32)


KINDS = ("sweep", "silence_bursts", "clipped")


@pytest.mark.parametrize("rate", (22050, 16000))
@pytest.mark.parametrize("tempo", TEMPOS)
@pytest.mark.parametrize("name", list(contours()))
def test_raw_push_equals_the_whole_signal(lib_built, rate, tempo, name):
    frames, ratios = contours()[name]
    cum = np.cumsum(frames)
    n, ends = 256 * max(int(cum[-1]), 1), 256 * cum
    if name == "all_zero" and tempo is None:
        pytest.skip("a neutral contour and no tempo is no stream (refused)")
    kind = KINDS[(list(contours()).index(name) + TEMPOS.index(tempo)) % len(KINDS)]
    x = constructed(kind, n, rate, seed=rate + n)
    want, want_off = debug_contour(x, rate, ends, ratios, tempo)
    for cname, lens in psr.chunkings(n, rate).items():
        y, got, off = debug_contour_stream(x, lens, rate, ends, ratios, tempo)
        np.testing.assert_array_equal(got, [r["emitted"] for r in pcs.stream(rate, n, ends, ratios, tempo, lens)],
                                      err_msg=cname)
        assert y.tobytes() == want.tobytes(), (kind, cname)
        np.testing.assert_array_equal(off, want_off, err_msg=cname)


def test_raw_push_single_samples(lib_built):
    rate = 16000
    frames = np.array([3, 1, 0, 2, 1, 4, 1])
    ratios = [0.5, 2.0, 1.3, 0.7, 2.0, 1.0, 0.6]
    cum = np.cumsum(frames)
    n, ends = 256 * int(cum[-1]), 256 * cum
    x = constructed("sweep", n, rate, 1)
    for tempo in (None, 2.0):
        want, _ = debug_contour(x, rate, ends, ratios, tempo)
        y, _, _ = debug_contour_stream(x, [1] * n, rate, ends, ratios, tempo)
        assert y.tobytes() == want.tobytes(), tempo


def _char_contour(phonemes, seed):
    """A per-character contour: a rise at the end, some characters at other ratios, some without one."""
    rng = np.random.default_rng(seed)
    c = list(rng.choice([0.8, 1.0, 1.25, 0.6, 1.7], len(phonemes)))
    c[len(c) - 6:] = [1.3] * 6
    c[0] = None
    return c


def _stream_inputs(m, phonemes, seed, cs, pad):
    """(enc, the plain chunks after the device post-path joined, ends, n) of the seeded sentence."""
    ids = m.phonemes_to_input_ids(phonemes)
    enc = m.infer_encoder_batch([ids], seeds=[seed])[0]
    plain = _cat(_plain(m, enc, cs, pad))
    return enc, plain, 256 * np.cumsum(enc.p_duration), 256 * enc.num_frames


def _id_contour(m, phonemes, char_contour):
    _, src = m.phonemes_to_input_ids_map(phonemes)
    return [NAN if v is None else v for v in _char_values_to_ids(char_contour, phonemes, src, 0, "pitch ratios",
                                                                   _contour_value)]


@pytest.mark.parametrize("quality", QUALITIES)
def test_stream_synthesis_equals_whole_on_every_voice(voices, quality):
    m = voices(quality)
    rate = m.audio_output_info().sample_rate
    cc = _char_contour(LONG, 5)
    ratios = _id_contour(m, LONG, cc)
    for cs, pad in ((55, 3), (4000, 3)):
        enc, plain, ends, n = _stream_inputs(m, LONG, 4, cs, pad)
        assert len(plain) == n
        for tempo in (None, 0.8):
            whole = debug_contour(plain, rate, ends, ratios, tempo)[0]
            st = m.stream_synthesis(LONG, cs, pad, seed=4, pitch_contour=cc, tempo=tempo)
            got = list(st)
            assert _cat(got).tobytes() == whole.tobytes(), (cs, tempo)
            assert st.bounds[-1] == len(whole)
            # at an output rate: the warped sentence resampled at once
            rs = list(m.stream_synthesis(LONG, cs, pad, seed=4, pitch_contour=cc, tempo=tempo, output_rate=48000))
            assert _cat(rs).tobytes() == debug_resample(whole, rate, 48000).tobytes(), (cs, tempo)
            # mu-law: each chunk is G.711 of to_i16_vec of the f32 chunk
            g = list(m.stream_synthesis(LONG, cs, pad, seed=4, pitch_contour=cc, tempo=tempo, encoding="mulaw"))
            assert len(g) == len(got)
            for a, b in zip(g, got):
                assert a == gr.encode_bytes(AudioSamples(b.as_slice()).to_i16_vec(), "mulaw")


@pytest.mark.parametrize("tempo", (None, 1.5, 0.5))
def test_uniform_is_the_ratio_stream_and_neutral_is_plain(voices, tempo):
    m = voices("medium")
    for ph in (LONG, SHORT):
        # uniform over every id (a per-character contour leaves bos and eos at 1)
        ids = m.phonemes_to_input_ids(ph)
        enc = m.infer_encoder_batch([ids], seeds=[2])[0]
        uni = list(SpeechStreamer(enc, 40, 3, warp=ProsodyStream(m, None, tempo, [1.25] * len(ids), enc)))
        enc = m.infer_encoder_batch([ids], seeds=[2])[0]
        ratio = list(SpeechStreamer(enc, 40, 3, warp=ProsodyStream(m, 1.25, tempo)))
        assert _same(uni, ratio), (ph, tempo)
        neutral = list(m.stream_synthesis(ph, 40, 3, seed=2, pitch_contour=[1.0, None] * (len(ph) // 2) +
                                          [NAN] * (len(ph) % 2), tempo=tempo))
        plain = list(m.stream_synthesis(ph, 40, 3, seed=2, tempo=tempo))
        assert _same(neutral, plain), (ph, tempo)


def test_stream_batch_mixes_contoured_ratio_and_plain_streams(voices):
    m = voices("medium")
    q = [1.0] * len(LONG)
    q[-8:] = question(8)
    kinds = [(LONG, dict(pitch_contour=_char_contour(LONG, 1))), (LONG, dict()), (SHORT, dict(pitch=0.8)),
             (LONG, dict(pitch_contour=q, tempo=1.5, output_rate=16000)),
             (SHORT, dict(pitch_contour=_char_contour(SHORT, 2), encoding="alaw", gain=0.5)),
             (LONG, dict(tempo=0.8)), (SHORT, dict(pitch_contour=[1.25] * len(SHORT)))]
    sb = StreamBatch(m, 40, 3)
    keys = [sb.add(ph, seed=20 + i, **kw) for i, (ph, kw) in enumerate(kinds)]
    # the same sentence added as ids, with its contour per id
    ids = m.phonemes_to_input_ids(LONG)
    kid = sb.add(ids, seed=20, pitch_contour=_id_contour(m, LONG, kinds[0][1]["pitch_contour"]))
    with pytest.raises(KeyError):
        sb.bounds(keys[0])
    got = {}
    for k, a in sb.step():                  # the step that encodes every stream: all bounds readable after it
        got.setdefault(k, []).append(a)
    bounds = [sb.bounds(k) for k in keys]
    for k, a in _drain(sb).items():
        got.setdefault(k, []).extend(a)
    for i, (ph, kw) in enumerate(kinds):
        st = m.stream_synthesis(ph, 40, 3, seed=20 + i, **kw)
        assert _same(got[keys[i]], list(st)), (i, kw)
        b = bounds[i]
        if st.bounds is None:
            assert b is None, i
        else:
            np.testing.assert_array_equal(b, st.bounds, err_msg=str(i))
    assert _same(got[kid], got[keys[0]])


@pytest.mark.parametrize("tempo", (None, 1.5))
def test_bounds_are_the_batch_paths(voices, tempo):
    m = voices("medium")
    rate = m.audio_output_info().sample_rate
    ids = list(workload.synthetic_ids(90, utt=11))
    rng = np.random.default_rng(11)
    contour = list(rng.choice([0.8, 1.0, 1.25, 1.6], len(ids)))
    job = SynthesisJob(m, [ids], seeds=[31], pitch_contours=[contour], tempos=[tempo])
    job.run()
    want = job.prosody_bounds()[0]
    n2 = len(job.fetch()[0].samples.as_slice())
    job.close()
    enc = m.infer_encoder_batch([ids], seeds=[31])[0]
    w = ProsodyStream(m, None, tempo, contour, enc)
    np.testing.assert_array_equal(w.bounds, want)
    assert want[-1] == n2
    for out_rate in (None, 16000, 48000):
        sb = StreamBatch(m, 55, 3)
        k = sb.add(ids, seed=31, pitch_contour=contour, tempo=tempo, output_rate=out_rate)
        got = _drain(sb)[k]
        up, down = (1, 1) if out_rate is None else (out_rate // np.gcd(rate, out_rate), rate // np.gcd(rate, out_rate))
        np.testing.assert_array_equal(sb.bounds(k), -((-want * up) // down))
        assert sb.bounds(k)[-1] == len(_cat(got)), out_rate


def test_creation_checks(voices):
    m = voices("medium")
    other = voices("low")
    ids = list(workload.synthetic_ids(40, utt=3))
    enc = m.infer_encoder_batch([ids], seeds=[5])[0]
    lib = N.lib()

    def create(model, latent, ratios, tempo=NAN):
        r = np.ascontiguousarray(ratios, np.float32)
        h, err = C.c_void_p(), N.sb200_error()
        rc = lib.sb200_prosody_stream_create_contour(model._h, latent._h, f32p(r), r.size, tempo, C.byref(h),
                                                     C.byref(err))
        if rc == 0:
            lib.sb200_prosody_stream_free(h)
        return rc, _message(err)
    good = [1.2] * len(ids)
    assert create(m, enc, good)[0] == 0
    rc, msg = create(m, enc, good[:-1])
    assert rc == 19 and "ratios for a latent of" in msg
    rc, msg = create(other, enc, good)
    assert rc == 19 and "not encoded by this voice" in msg
    bad = list(good)
    bad[5] = 2.5
    rc, msg = create(m, enc, bad)
    assert rc == 19 and "id 5" in msg
    rc, msg = create(m, enc, [1.0] * len(ids))
    assert rc == 19 and "ask for nothing" in msg
    assert create(m, enc, [1.0] * len(ids), 1.5)[0] == 0
    rc, msg = create(m, enc, good, 5.0)
    assert rc == 19 and "tempo ratio" in msg
    # bounds: a ratio stream has none
    w = ProsodyStream(m, 1.25)
    out, err = np.zeros(4, np.int64), N.sb200_error()
    assert lib.sb200_prosody_stream_bounds(w._h, i64p(out), 4, C.byref(err)) == 19
    assert "without a pitch contour" in _message(err)
    wc = ProsodyStream(m, None, None, good, enc)
    assert lib.sb200_prosody_stream_bounds(wc._h, i64p(out), 4, C.byref(err)) == 19       # too small
    with pytest.raises(OperationError, match="5 pitch ratios for 4 ids"):
        ProsodyStream(m, None, None, [1.2] * 5, m.infer_encoder_batch([ids[:4]], seeds=[1])[0])


def test_misuse_with_a_contoured_stream(voices):
    m = voices("medium")
    rate = m.audio_output_info().sample_rate
    ids = list(workload.synthetic_ids(150, utt=3))
    enc = m.infer_encoder_batch([ids], seeds=[5])[0]
    contour = list(np.random.default_rng(4).choice([0.7, 1.0, 1.4], len(ids)))
    # trimmed, the chunks cover frames [0, 37), [37, 77) and [77, T): the whole latent
    chunks = [(enc, 0, 40, 0, 3), (enc, 34, 80, 3, 3), (enc, 74, enc.num_frames, 3, 0)]
    w = ProsodyStream(m, None, None, contour, enc)
    out = [m.infer_decoder_batch([chunks[0]], fade=42, warps=[w], last=[False])[0]]
    with pytest.raises(OperationError, match="chunk 1: the prosody stream of chunk 0 appears twice"):
        m.infer_decoder_batch([chunks[1], chunks[1]], fade=42, warps=[w, w], last=[False, False])
    # a chunk that would end the stream before its n inputs, or go past them, fails (internal) before any device work,
    # and the stream is left as it was
    with pytest.raises(OperationError, match="internal: a contour prosody stream would end"):
        m.infer_decoder_batch([chunks[1]], fade=42, warps=[w], last=[True])
    with pytest.raises(OperationError, match="internal: a contour prosody stream would go on"):
        m.infer_decoder_batch([(enc, 0, enc.num_frames, 0, 0)], fade=0, warps=[w], last=[False])
    out.append(m.infer_decoder_batch([chunks[1]], fade=42, warps=[w], last=[False])[0])
    out.append(m.infer_decoder_batch([chunks[2]], fade=42, warps=[w], last=[True])[0])
    with pytest.raises(OperationError, match="chunk 0: the prosody stream has already been flushed"):
        m.infer_decoder_batch([chunks[2]], fade=42, warps=[w], last=[True])
    plain = m.infer_decoder_batch(chunks, fade=42, resamplers=[None] * 3)
    ends = 256 * np.cumsum(enc.p_duration)
    assert _cat(out).tobytes() == debug_contour(_cat(plain), rate, ends, contour, None)[0].tobytes()


def test_neutral_contour_with_a_tempo_has_bounds_on_every_entry_point(voices):
    """A given contour of 1 / NaN only with a tempo is a contoured stream whichever way it is made: the tempo stream's
    bits, and bounds."""
    m = voices("medium")
    ids = m.phonemes_to_input_ids(LONG)
    st = m.stream_synthesis(LONG, 40, 3, seed=6, pitch_contour=[1.0] * len(LONG), tempo=1.5)
    got = list(st)
    enc = m.infer_encoder_batch([ids], seeds=[6])[0]
    direct = ProsodyStream(m, None, 1.5, [1.0] * len(ids), enc)
    np.testing.assert_array_equal(st.bounds, direct.bounds)
    assert st.bounds[-1] == len(_cat(got))
    assert _same(got, list(m.stream_synthesis(LONG, 40, 3, seed=6, tempo=1.5)))
    sb = StreamBatch(m, 40, 3)
    k = sb.add(ids, seed=6, pitch_contour=[NAN] * len(ids), tempo=1.5)
    sb.step()
    np.testing.assert_array_equal(sb.bounds(k), direct.bounds)


def test_batches_keep_no_state_for_ended_streams(voices):
    """Bounds stay readable until the step after a stream's last chunk, and then the batch holds nothing for it: a
    long-running StreamBatch or RealtimeBatch does not grow with the sentences it has served."""
    m = voices("medium")
    sb = StreamBatch(m, 40, 3)
    kws = [dict(pitch_contour=[1.25] * len(SHORT)), dict(pitch_contour=_char_contour(LONG, 3)), dict(), dict(pitch=1.25),
           dict(pitch_contour=[1.1] * len(LONG)), dict(tempo=0.8)]
    keys = [sb.add(SHORT if i == 0 else LONG, seed=1 + i, **kw) for i, kw in enumerate(kws)]
    got, ended = {}, set()
    while len(sb):
        for k, a in sb.step():
            got.setdefault(k, []).append(a)
        for k in ended:                     # ended before this step: nothing kept
            with pytest.raises(KeyError):
                sb.bounds(k)
        for i, k in enumerate(keys):
            if k in sb or k in ended:
                continue
            # the step that returned its last chunk: its bounds are still readable
            b = sb.bounds(k)
            if "pitch_contour" in kws[i]:
                assert b[-1] == len(_cat(got[k])), i
            else:
                assert b is None, i
            ended.add(k)
        assert len(sb._retired) <= len(keys)
    assert ended == set(keys)
    sb.step()
    for k in keys:
        with pytest.raises(KeyError):
            sb.bounds(k)
    assert not sb._active and not sb._pending and not sb._retired
    rb = RealtimeBatch(m, 30, 3)
    for i in range(3):
        rb.add(LONG + "\n" + SHORT, AudioOutputConfig(None, None, None, None), seed=i)
    while len(rb):
        rb.step()
    rb.step()
    assert not rb._by_stream and not rb._streams._active and not rb._streams._retired
