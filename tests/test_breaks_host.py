"""Host tests of breaks (include/sonata_b200.h, sb200_speak_batch_ids_breaks): the numpy contract against a literal
per-sample reading of the header, the checks and their messages in Python and in the library, the per-character
mapping, alignments from the ends after the pauses, and the stream emission rule over random chunkings."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import break_reference as br
import sonata_b200
from sonata_b200 import _native as N, voicegen
from sonata_b200.core import Audio, OperationError
from sonata_b200.piper import (_VitsCommons, _alignment, _batch_options, _break_arrays, _breaks_ask,
                               _char_breaks_to_ids, _check, _stream_options, VitsStreamingModel)

NAN, INF = float("nan"), float("inf")


# ---------------------------------------------------------------------------------------------------- the contract
def literal(x, ends, ms, rate):
    """The header read sample by sample, in plain Python floats (IEEE double, each operation rounded)."""
    n2 = len(x)
    N_ = [int(np.floor(float(np.float32(v)) * rate / 1000.0 + 0.5)) if not (np.isnan(v) or v == 0) else 0 for v in ms]
    P, M = [], []
    for e, n in zip(ends, N_):
        if n == 0:
            continue
        if P and P[-1] == e:
            M[-1] += n
        else:
            P.append(int(e))
            M.append(n)
    F = rate // 200
    S = lambda t: t * t * (3.0 - 2.0 * t)
    D = [0]
    for m in M:
        D.append(D[-1] + m)
    out = [None] * (n2 + D[-1])
    for j in range(n2):
        h = 1.0
        for p in P:
            if p - F <= j < p:
                h = h * S((float(p - j) - 0.5) / F)
            if p <= j < p + F:
                h = h * S((float(j - p) + 0.5) / F)
        k = sum(1 for p in P if p <= j)
        out[j + D[k]] = np.float32(x[j]) * np.float32(h)
    for k, p in enumerate(P):
        for q in range(p + D[k], p + D[k + 1]):
            assert out[q] is None
            out[q] = np.float32(0.0)
    assert all(v is not None for v in out)
    return np.array(out, np.float32)


@pytest.mark.parametrize("rate", (22050, 16000))
def test_contract_matches_the_header_sample_by_sample(rate):
    rng = np.random.default_rng(rate)
    F = rate // 200
    x = rng.standard_normal(3000).astype(np.float32)
    cases = [
        # merged equal ends (an id with no samples between them), and a break that rounds to 0 samples
        ([0, 700, 700, 1500, 3000], [NAN, 10.0, 5.0, 0.01, NAN]),
        # breaks closer than 2F: overlapping fades
        ([900, 900 + F // 2, 900 + F + 3, 3000], [3.0, 2.0, 1.0, 0.0]),
        # breaks at 0 (after ids with no samples) and at n2 (trailing)
        ([0, 0, 1200, 3000], [4.0, 1.5, NAN, 7.0]),
        # every break rounds to 0 samples: nothing changes
        ([1000, 3000], [0.01, 0.02]),
        # ids with no samples everywhere
        ([0, 0, 0, 1, 1, 2999, 3000, 3000], [1.0, NAN, 2.0, 1.0, 0.0, 3.0, 1.0, 2.0]),
    ]
    for ends, ms in cases:
        want = literal(x, ends, ms, rate)
        got = br.apply(x, ends, ms, rate)
        assert got.tobytes() == want.tobytes(), (ends, ms)
        assert got.size == x.size + int(br.samples(ms, rate).sum())
        assert br.delivered_ends(ends, ms, rate)[-1] == got.size


def test_lengths_round_half_up_in_double():
    assert br.samples([1000.0], 22050)[0] == 22050
    assert br.samples([0.02267], 22050)[0] == 0            # 0.4999 samples
    assert br.samples([0.0227], 22050)[0] == 1             # 0.50054 samples
    assert br.samples([NAN, 0.0, 10000.0], 16000).tolist() == [0, 0, 160000]
    # the ms value is the f32 the library receives
    assert br.samples([np.float32(0.1)], 22050)[0] == int(np.floor(float(np.float32(0.1)) * 22050 / 1000 + 0.5))


def test_neutral_and_zero_breaks_keep_every_bit():
    x = np.random.default_rng(1).standard_normal(2000).astype(np.float32)
    assert br.apply(x, [1000, 2000], [NAN, 0.0], 22050).tobytes() == x.tobytes()
    assert br.apply(x, [1000, 2000], [0.01, 0.0], 22050).tobytes() == x.tobytes()


def test_pauses_are_silent_and_the_speech_around_them_fades():
    rate = 16000
    F = rate // 200
    x = np.ones(4000, np.float32)
    y = br.apply(x, [2000, 4000], [10.0, NAN], rate)              # 160 samples after sample 2000
    assert y.size == 4160
    assert np.all(y[2000:2160] == 0) and np.signbit(y[2000:2160]).sum() == 0
    assert np.all(y[:2000 - F] == 1) and np.all(y[2160 + F:] == 1)
    fade_out, fade_in = y[2000 - F:2000], y[2160:2160 + F]
    assert np.all(np.diff(fade_out) < 0) and np.all(np.diff(fade_in) > 0)
    assert fade_out.tobytes() == fade_in[::-1].tobytes()        # symmetric about the pause
    np.testing.assert_array_equal(br.delivered_ends([2000, 4000], [10.0, NAN], rate), [2160, 4160])


# ---------------------------------------------------------------------------------------------------- emission rule
@pytest.mark.parametrize("seed", range(6))
def test_stream_emission_over_random_chunkings(seed):
    """After each chunk the stage has emitted O(J) samples: the chunks join to the whole paused signal, and a chunk
    whose input reaches a break emits its zeros."""
    rng = np.random.default_rng(seed)
    rate = (22050, 16000)[seed % 2]
    n_ids = int(rng.integers(1, 40))
    ends = 256 * np.cumsum(rng.integers(0, 6, n_ids))
    n2 = max(int(ends[-1]), 256)
    ends[-1] = n2
    ms = rng.choice([NAN, 0.0, 5.0, 40.0, 0.01, 250.0], n_ids).astype(np.float32)
    x = rng.standard_normal(n2).astype(np.float32)
    whole = br.apply(x, ends, ms, rate)
    P, M = br.plan(ends, ms, rate)
    cuts = np.sort(rng.choice(np.arange(1, n2), size=min(n2 - 1, int(rng.integers(1, 30))), replace=False))
    parts, out = [], 0
    for a, b in zip(np.r_[0, cuts], np.r_[cuts, n2]):
        o = br.emitted(int(b), P, M)
        parts.append(whole[out:o])
        for p, m in zip(P, M):                               # a break the chunk's input reaches is emitted in it
            if a < p <= b:
                q = p + br.emitted(int(p), P, M) - p - m
                assert out <= q and q + m <= o
        out = o
    assert out == whole.size == n2 + int(M.sum())
    assert np.concatenate(parts).tobytes() == whole.tobytes()


# ---------------------------------------------------------------------------------------------------- Python checks
def test_python_checks_name_the_utterance_and_the_id():
    assert _break_arrays([3], None) is None
    assert _break_arrays([3, 2], [[NAN, 0.0, None], None]) is None
    img = _break_arrays([3, 2], [[250.0, None, 0], [10000, 0.5]])
    assert img.dtype == np.float32 and img[0] == 250 and np.isnan(img[1]) and img[3] == 10000
    cases = [([[0.0, 10001.0, 0.0]], "utterance 0, id 1: break 10001.0 ms is not a finite value in (0.0, 10000.0]"),
             ([[0.0, 0.0, INF]], "utterance 0, id 2: break inf ms"),
             ([[-5.0, 0.0, 0.0]], "utterance 0, id 0: break -5.0 ms"),
             ([[0.0, "long", 0.0]], "utterance 0, id 1: break 'long' is not a number"),
             ([[0.0, 0.0]], "utterance 0: 2 breaks for 3 ids")]
    for breaks, msg in cases:
        with pytest.raises(OperationError, match=re.escape(msg)):
            _break_arrays([3], breaks)
    with pytest.raises(OperationError, match=re.escape("stream 4, id 0: break -1.0 ms")):
        _break_arrays([1], [[-1.0]], ["stream 4"])
    assert not _breaks_ask(None, 22050) and not _breaks_ask(np.array([NAN, 0.02], np.float32), 22050)
    assert _breaks_ask(np.array([NAN, 0.0227], np.float32), 22050)


def test_batch_options_check_breaks_after_volume():
    o = _batch_options(None, 2, [2, 1], breaks=[[300.0, NAN], None])
    assert o.breaks is not None and o.breaks[0] == 300
    with pytest.raises(OperationError, match="utterance 1, id 0: volume"):
        _batch_options(None, 2, [2, 1], volume_contours=[None, [99.0]], breaks=[None, [-1.0]])
    with pytest.raises(OperationError, match="utterance 1, id 0: break"):
        _batch_options(None, 2, [2, 1], breaks=[None, [-1.0]])


def test_per_character_breaks_go_after_the_last_id():
    # ids: bos, (id, pad) per kept character, eos; src: the character of each id
    src = [-1, 0, 0, 1, 1, 3, 3, -1]                 # "ab~c": character 2 is dropped
    got = _char_breaks_to_ids([100.0, None, 50.0, 20.0], "ab~c", src, 0)
    # a's pause after a's pad (id 2), the dropped character's after b's pad (id 4), c's after its pad (id 6)
    assert np.isnan(got[0]) and got[2] == 100.0 and got[4] == 50.0 and got[6] == 20.0
    assert sum(not np.isnan(v) for v in got) == 3
    # a dropped first character goes after bos; breaks landing on one id add up
    got = _char_breaks_to_ids([30.0, None, 20.0, None], "~b~c", [-1, 1, 1, 3, 3, -1], 0)
    assert got[0] == 30.0 and got[2] == 20.0
    got = _char_breaks_to_ids([None, 5.0, 7.0, None], "ab~c", src, 0)
    assert got[4] == 12.0
    with pytest.raises(OperationError, match=re.escape("utterance 0, character 1: break -3.0 ms")):
        _char_breaks_to_ids([None, -3.0, None, None], "ab~c", src, 0)
    with pytest.raises(OperationError, match=re.escape("stream: 2 breaks for 4 characters")):
        _char_breaks_to_ids([1.0, 2.0], "ab~c", src, "stream")


class FakeModel:
    """Ids: bos 1, (ord(ch) % 50 + 3, pad 0) per character except '~' (dropped), eos 2; the f32 route records the
    options it is given and reports each id's end after the pauses before it."""

    def __init__(self):
        self.calls = []

    def phonemes_to_input_ids_map(self, ph):
        ids, src = [1], [-1]
        for c, ch in enumerate(ph):
            if ch != "~":
                ids += [ord(ch) % 50 + 3, 0]
                src += [c, c]
        return ids + [2], src + [-1]

    def _speak_ids(self, batches, o, frames=False):
        self.calls.append((batches, o))
        out, pos = [], 0
        for ids in batches:
            ends = 256 * np.arange(1, len(ids) + 1)
            bounds = None
            if o.breaks is not None:
                ms = o.breaks[pos:pos + len(ids)]
                bounds = br.delivered_ends(ends, ms, 22050)
            n = int(ends[-1] if bounds is None else bounds[-1])
            out.append((Audio(np.zeros(n, np.float32), 22050), np.ones(len(ids), np.int32), bounds))
            pos += len(ids)
        return out


def test_alignment_from_the_ends_after_the_pauses():
    fake = FakeModel()
    res = _VitsCommons.speak_batch_with_alignment(fake, ["ab~c", "xy"], breaks=[[100.0, None, 50.0, None], None])
    _, o = fake.calls[-1]
    assert o.breaks is not None
    (a0, al0), (a1, al1) = res
    # "ab~c": bos, a, b, c, eos; a's pause belongs to a, the dropped character's to b
    assert [e.phoneme for e in al0] == ["^", "a", "b", "c", "$"]
    pa, pb = br.samples([100.0], 22050)[0], br.samples([50.0], 22050)[0]
    assert [e.num_samples for e in al0] == [256, 512 + pa, 512 + pb, 512, 256]
    assert al0[0].start_sample == 0 and al0[-1].start_sample + al0[-1].num_samples == len(a0.samples.as_slice())
    # the utterance without breaks keeps the frame alignment
    assert [e.num_samples for e in al1] == [256, 512, 512, 256]
    # _alignment itself: each entry ends where its last id does, at an output rate at ceil(E' up / down)
    al = _alignment("ab", [-1, 0, 0, 1, 1, -1], [1] * 6, 3200, 2, 1, bounds=[256, 512, 700, 900, 1500, 1600])
    assert [(e.start_sample, e.num_samples) for e in al] == [(0, 512), (512, 888), (1400, 1600), (3000, 200)]


# ---------------------------------------------------------------------------------------------------- library checks
@pytest.fixture(scope="module")
def config_only(lib_built):
    p = voicegen.write_voice(voicegen.default_voice_dir(), "medium")
    m = sonata_b200.VitsStreamingModel(p, device=-1)       # config only: any device call fails differently
    yield m
    m.close()


def test_the_c_entry_points_refuse_before_any_device_work(config_only):
    lib = N.lib()
    ids = np.array([1, 5, 2, 1, 6, 7, 2], np.int64)
    offs = np.array([0, 3, 7], np.uint64)
    i64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))
    f32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    sz = lambda a: a.ctypes.data_as(C.POINTER(C.c_size_t))
    outs = (N.sb200_audio * 2)()

    def speak(bk):
        err = N.sb200_error()
        rc = lib.sb200_speak_batch_ids_breaks(config_only._h, i64(ids), sz(offs), 2, None, None, None, None, None,
                                              None, None, None, None, None, None, None, None, None, None, f32(bk), outs,
                                              None, None, None, None, C.byref(err))
        with pytest.raises(OperationError) as e:
            _check(rc, err)
        return str(e.value)
    for bad, msg in ((10001.0, "utterance 1, id 2: break 10001.000000 ms is not a finite value in (0, 10000]"),
                     (INF, "utterance 1, id 2: break inf ms"), (-INF, "utterance 1, id 2: break -inf ms"),
                     (-0.5, "utterance 1, id 2: break -0.500000 ms")):
        got = speak(np.array([6, NAN, 0, 0, 300, bad, 0], np.float32))
        assert msg in got, got
    # good breaks pass the checks and reach the job, which a config-only voice cannot run
    assert "break" not in speak(np.array([6, NAN, 0, 0, 300, 10000, 0], np.float32))
    # the debug hook checks its breaks before any device work
    x = np.zeros(10, np.float32)
    err, n_out = N.sb200_error(), C.c_int64()
    rc = lib.sb200_debug_breaks(0, f32(x), 10, i64(np.array([10], np.int64)), f32(np.array([-2.0], np.float32)), 1,
                                22050, f32(x), 10, C.byref(n_out), C.byref(err))
    with pytest.raises(OperationError, match=re.escape("id 0: break -2.000000 ms")):
        _check(rc, err)
    # and the paused length against 2^31 - 1
    ends = np.arange(1, 401, dtype=np.int64) * 0 + 10
    ms = np.full(400, 10000.0, np.float32)
    err = N.sb200_error()
    rc = lib.sb200_debug_breaks(0, f32(x), 10, i64(ends), f32(ms), 400, 600000, f32(x), 10, C.byref(n_out),
                                C.byref(err))
    with pytest.raises(OperationError, match=re.escape("passes 2^31 - 1")):
        _check(rc, err)


def test_stream_options_name_the_stream(config_only):
    with pytest.raises(OperationError, match=re.escape("stream 2, id 1: break 20000.0 ms")):
        _stream_options(config_only, "StreamBatch", 2, [1, 5, 2], breaks=[0.0, 20000.0, 0.0])
    with pytest.raises(OperationError, match=re.escape("stream: 2 breaks for 3 ids")):
        _stream_options(config_only, "stream_synthesis", None, [1, 5, 2], breaks=[0.0, 4.0])
    o = _stream_options(config_only, "stream_synthesis", None, [1, 5, 2], breaks=[0.0, 4.0, None])
    assert o.breaks == [0.0, 4.0, None]


def test_models_without_streaming_voices_refuse_by_name():
    class Other:
        pass
    with pytest.raises(OperationError, match="stream_synthesis cannot insert breaks"):
        VitsStreamingModel.stream_synthesis(Other(), "ab", 10, 3, breaks=[0.0, 0.0])
