"""GPU (-m gpu): target durations (include/sonata_b200.h, sb200_speak_batch_ids_fit and
sb200_encode_batch_ids_targets).

The hook and the synthesis path against tests/fit_reference.py exactly (u* and per-id counts, from the fetched w image,
on every voice and at the contract's edges); a fitted utterance against the same utterance with its fitted counts
fixed, alone and in a mixed batch, and through pitch, breaks, loudness, G.711 and FLAC; neutral tables; alignments;
streams fitted in their encoder pass; and StreamBatch neighbours."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import fit_reference as fr
from test_prosody_stream_gpu import LONG, SHORT, _cat, _drain, voices  # noqa: F401
from sonata_b200 import _native as N, workload
from sonata_b200.job import SynthesisJob
from sonata_b200.piper import SpeechStreamer, StreamBatch, rate_ratio

pytestmark = pytest.mark.gpu
NAN = float("nan")
QUALITIES = ("x_low", "low", "medium", "high")
f32p = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
i32p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))
i64p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))


def debug_fit(w, fixed, first, end, budget):
    w = np.ascontiguousarray(w, np.float32)
    fixed = np.ascontiguousarray(fixed, np.int32)
    first, end, budget = (np.ascontiguousarray(a, np.int64) for a in (first, end, budget))
    k = first.size
    factor, u, f = np.zeros(w.size, np.float32), np.zeros(max(k, 1), np.float32), np.zeros(max(k, 1), np.int64)
    err = N.sb200_error()
    rc = N.lib().sb200_debug_fit(0, f32p(w), w.size, i32p(fixed), i64p(first), i64p(end), i64p(budget), k,
                                 f32p(factor), f32p(u), i64p(f), C.byref(err))
    assert rc == 0, C.string_at(err.message).decode() if err.message else rc
    return factor, u[:k], f[:k]


def _bits(a):
    return np.asarray(a, np.float32).tobytes()


# ---------------------------------------------------------------------------------------------------- the hook
def test_hook_equals_the_contract(lib_built):
    rng = np.random.default_rng(7)
    for trial in range(40):
        n = int(rng.integers(1, 400))
        w = (rng.choice([0.0, 1e-30, 0.4, 1.0, 2.5, 6.0, 30.0], n) * rng.uniform(0.6, 1.4, n)).astype(np.float32)
        if trial % 7 == 0:
            w[rng.integers(0, n)] = np.inf
        fixed = np.where(rng.random(n) < 0.1, rng.integers(0, 12, n), -1)
        cuts = np.unique(rng.integers(0, n + 1, int(rng.integers(2, 8))))
        first, end = cuts[:-1], cuts[1:]
        nat = np.array([fr.frames(w[a:e], fixed[a:e], 1.0) for a, e in zip(first, end)])
        budget = (nat * rng.choice([0.3, 0.8, 1.0, 1.25, 3.0], nat.size)).astype(np.int64) + rng.integers(-2, 3, nat.size)
        factor, u, f = debug_fit(w, fixed, first, end, budget)
        want = np.ones(n, np.float32)
        for k, (a, e) in enumerate(zip(first, end)):
            ru, rf = fr.solve(w[a:e], fixed[a:e], int(budget[k]))
            assert _bits(u[k]) == _bits(ru) and f[k] == rf, (trial, k)
            if (fixed[a:e] < 0).any():
                want[a:e] = ru
        assert _bits(factor) == _bits(want), trial
    # plateaus: ten equal ids step together; a span over its target; one that 2 still fits
    w = np.full(10, 10.0, np.float32)
    _, u, f = debug_fit(w, np.full(10, -1), [0, 0, 0], [10, 10, 10], [75, 10, 10**6])
    assert f.tolist() == [70, 50, 200] and u[1] == 0.5 and u[2] == 2.0


# ---------------------------------------------------------------------------------------------------- the pass
def _targets_for(n_ids, nat_ms, kind):
    if kind == "short":
        return 0.8 * nat_ms
    if kind == "long":
        return 1.25 * nat_ms
    if kind == "words":                 # a span about every 4 ids, every other one asking
        spans = [(a, min(a + 3, n_ids - 1), 60.0 + 7 * (a % 5)) for a in range(0, n_ids, 4)]
        return [(a, b, ms if k % 2 == 0 else NAN) for k, (a, b, ms) in enumerate(spans)]
    if kind == "over":
        return [(1, n_ids - 2, 1.0)]
    if kind == "under":
        return [(0, n_ids - 1, 600000.0)]
    raise ValueError(kind)


KINDS = ("short", "long", "words", "over", "under")


@pytest.mark.parametrize("quality", QUALITIES)
def test_pass_equals_the_contract_from_the_fetched_w(voices, quality):
    m = voices(quality)
    rate = m.audio_output_info().sample_rate
    batches = [list(workload.synthetic_ids(n, utt=u)) for n, u in ((40, 1), (90, 2), (25, 3), (61, 4), (33, 5))]
    seeds = [11, 12, 13, 14, 15]
    plain = m.infer_batch_with_durations(batches, seeds=seeds)
    targets = [_targets_for(len(b), 1000.0 * len(a.samples.as_slice()) / rate, k)
               for b, (a, _), k in zip(batches, plain, KINDS)]
    job = SynthesisJob(m, batches, debug=True, seeds=seeds, target_durations=targets)
    try:
        job.run()
        frames = job.id_frames()
        rep = job.targets()
        names = {r["name"] for r in job.profile()}
        assert "fit" in names
        for b, ids in enumerate(batches):
            w = job.debug_fetch("fit.w", b).reshape(-1)
            t = targets[b]
            spans = [(0, len(ids), t)] if isinstance(t, float) else [(a, e + 1, ms) for a, e, ms in t]
            res, factor, c = fr.fit(w, np.full(len(ids), -1), spans, rate)
            inside = factor != 1
            for (u, L), (ru, rL) in zip(rep[b], res):
                assert _bits(u) == _bits(ru) and L == rL, (b, u, ru, L, rL)
            asked = np.zeros(len(ids), bool)
            for (a, e, ms) in spans:
                if not math.isnan(ms):
                    asked[a:e] = True
            assert (frames[b][asked] == c[asked]).all(), b
            # ids outside the spans keep their counts
            assert (frames[b][~asked] == plain[b][1][~asked]).all(), b
            for (a, e, ms), (u, L) in zip(spans, rep[b]):
                if math.isnan(ms):
                    continue
                T = fr.target_samples(ms, rate)
                assert L <= T or u == 0.5
                assert L == 256 * int(frames[b][a:e].sum())
            assert inside.sum() <= asked.sum()
    finally:
        job.close()


def test_fitted_equals_fixed_counts_alone_and_in_a_mixed_batch(voices):
    m = voices("medium")
    batches = [list(workload.synthetic_ids(n, utt=u)) for n, u in ((50, 1), (80, 2), (30, 3))]
    seeds = [5, 6, 7]
    targets = [1500.0, None, [(2, 20, 500.0), (30, 40, 300.0)]]
    fit = m.infer_batch_with_durations(batches, seeds=seeds, target_durations=targets)
    fixed = m.infer_batch_with_durations(batches, seeds=seeds, durations=[f for _, f in fit])
    for (a, fa), (b, fb) in zip(fit, fixed):
        assert (fa == fb).all() and a.samples.as_slice().tobytes() == b.samples.as_slice().tobytes()
    alone = m.infer_batch_with_durations([batches[2]], seeds=[7], target_durations=[targets[2]])
    assert alone[0][0].samples.as_slice().tobytes() == fit[2][0].samples.as_slice().tobytes()
    assert (alone[0][1] == fit[2][1]).all()


def test_neutral_tables_keep_every_bit_and_launch_nothing(voices):
    m = voices("low")
    batches = [list(workload.synthetic_ids(n, utt=u)) for n, u in ((40, 1), (70, 2))]
    ref = m.infer_batch_with_values(batches, seeds=[1, 2])
    for t in (None, [None, None], [NAN, [(0, 3, NAN)]]):
        got = m.infer_batch_with_values(batches, seeds=[1, 2], target_durations=t)
        assert all(a.samples.as_slice().tobytes() == b.samples.as_slice().tobytes() for a, b in zip(ref, got))
        job = SynthesisJob(m, batches, seeds=[1, 2], target_durations=t)
        try:
            job.run()
            assert "fit" not in {r["name"] for r in job.profile()}
        finally:
            job.close()


@pytest.mark.parametrize("out_rate", (None, 16000))
def test_alignment_spans_match_the_reported_length(voices, out_rate):
    m = voices("medium")
    rate = m.audio_output_info().sample_rate
    ph = LONG
    ids, src = m.phonemes_to_input_ids_map(ph)
    spans = [(0, 4, 400.0), (10, 20, 700.0)]
    (audio, al), = m.speak_batch_with_alignment([ph], seeds=[3], target_durations=[spans],
                                                output_rates=None if out_rate is None else [out_rate])
    job = SynthesisJob(m, [ids], seeds=[3], target_durations=[
        [(min(i for i, c in enumerate(src) if a <= c <= b), max(i for i, c in enumerate(src) if a <= c <= b), ms)
         for a, b, ms in spans]])
    try:
        job.run()
        rep = job.targets()[0]
    finally:
        job.close()
    up, down = rate_ratio(rate, out_rate)
    # alignment entries: bos, one per kept character, eos; their boundaries are ceil(E up / down)
    kept = sorted({int(c) for c in src if c >= 0})
    starts = {}
    for e, c in zip(al[1:-1], kept):
        starts[c] = (e.start_sample, e.start_sample + e.num_samples)
    for (a, b, ms), (u, L) in zip(spans, rep):
        cs = [c for c in kept if a <= c <= b]
        s0, s1 = starts[cs[0]][0], starts[cs[-1]][1]
        if (up, down) == (1, 1):
            assert s1 - s0 == L
        else:       # each boundary is ceil(E up / down)
            assert abs((s1 - s0) - L * up / down) < 1
        assert L <= fr.target_samples(ms, rate) or u == 0.5


def test_composes_as_fixed_counts(voices):
    m = voices("medium")
    batches = [list(workload.synthetic_ids(n, utt=u)) for n, u in ((60, 1), (45, 2))]
    seeds = [21, 22]
    targets = [1800.0, [(3, 30, 900.0)]]
    brk = [np.where(np.arange(len(batches[0])) % 9 == 8, 120.0, NAN).astype(np.float32), None]
    fit = m.infer_batch_with_durations(batches, seeds=seeds, target_durations=targets, breaks=brk)
    frames = [f for _, f in fit]
    kw = dict(seeds=seeds, pitches=[1.3, None], breaks=brk, loudness=[-20.0, -23.0])
    a = m.infer_batch_with_values(batches, target_durations=targets, **kw)
    b = m.infer_batch_with_durations(batches, durations=frames, **kw)
    assert all(x.samples.as_slice().tobytes() == y.samples.as_slice().tobytes() for x, (y, _) in zip(a, b))
    for route in ("g711", "flac"):
        kw2 = dict(seeds=seeds, breaks=brk, output_rates=[16000, None])
        if route == "g711":
            got = m.infer_batch_g711(batches, "mulaw", target_durations=targets, **kw2)
        else:
            got = m.infer_batch_flac(batches, target_durations=targets, **kw2)
        job = SynthesisJob(m, batches, **kw2)
        try:
            job.set_durations(frames=frames)
            job.run()
            want = job.fetch_g711("mulaw") if route == "g711" else job.fetch_flac()
        finally:
            job.close()
        assert got == want, route


# ---------------------------------------------------------------------------------------------------- streams
def test_stream_is_fitted_in_its_encoder_pass(voices):
    m = voices("medium")
    target = [(0, 10, 600.0), (20, 40, 900.0)]
    st = m.stream_synthesis(LONG, 55, 3, seed=9, target_duration=target)
    chunks = list(st)
    ids, src = m.phonemes_to_input_ids_map(LONG)
    enc_fit = m.infer_encoder_batch([ids], seeds=[9], target_durations=[[
        (min(i for i, c in enumerate(src) if a <= c <= b), max(i for i, c in enumerate(src) if a <= c <= b), ms)
        for a, b, ms in target]])[0]
    assert (st.enc.p_duration == enc_fit.p_duration).all()
    assert st.enc.fit == enc_fit.fit
    enc_fixed = m.infer_encoder_batch([ids], seeds=[9], durations=[enc_fit.p_duration])[0]
    assert (enc_fixed.p_duration == enc_fit.p_duration).all()
    want = list(SpeechStreamer(enc_fixed, 55, 3))
    assert _cat(chunks).tobytes() == _cat(want).tobytes()


def test_stream_batch_keeps_the_other_streams(voices):
    m = voices("medium")
    sb = StreamBatch(m, 40, 3)
    k0 = sb.add(LONG, seed=1)
    k1 = sb.add(SHORT, seed=2, target_duration=700.0)
    k2 = sb.add(LONG, seed=3, output_rate=16000)
    got = _drain(sb)
    sb2 = StreamBatch(m, 40, 3)
    j0 = sb2.add(LONG, seed=1)
    j2 = sb2.add(LONG, seed=3, output_rate=16000)
    ref = _drain(sb2)
    for k, j in ((k0, j0), (k2, j2)):
        assert len(got[k]) == len(ref[j])
        assert all(x.as_slice().tobytes() == y.as_slice().tobytes() for x, y in zip(got[k], ref[j]))
    alone = list(m.stream_synthesis(SHORT, 40, 3, seed=2, target_duration=700.0))
    assert _cat(got[k1]).tobytes() == _cat(alone).tobytes()
