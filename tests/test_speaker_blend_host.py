"""CPU: the host side of speaker blends -- the numpy contract (tests/blend_reference.py), the argument checks and their
messages at every Python surface and at the C entry point, the C image of a blend table, the CLI's flag and JSON field,
the blends' trip through `shard.Frontend` (gloo, world size 2), and the oracle's meaning of a blend pinned against a
live transformers VitsModel."""
import ctypes as C
import os
import re
import sys
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import blend_reference as br
import sonata_b200
from oracle import vits_oracle as vo
from sonata_b200 import PiperSynthesisConfig, _native as N, cli, voicegen
from sonata_b200.core import OperationError
from sonata_b200.piper import StreamBatch, _blend_arrays, _check
from sonata_b200.shard import Frontend
from sonata_b200.synth import RealtimeBatch, SonataSpeechSynthesizer


@pytest.fixture(scope="module")
def paths(lib_built):
    d = voicegen.default_voice_dir()
    return {"medium4": voicegen.write_voice(d, "medium", n_speakers=4), "medium": voicegen.write_voice(d, "medium")}


@pytest.fixture(scope="module")
def m4(paths):
    m = sonata_b200.VitsModel(paths["medium4"], device=-1)       # config only: any device call fails differently
    yield m
    m.close()


@pytest.fixture(scope="module")
def s4(paths):
    m = sonata_b200.VitsStreamingModel(paths["medium4"], device=-1)
    yield m
    m.close()


@pytest.fixture(scope="module")
def m1(paths):
    m = sonata_b200.VitsModel(paths["medium"], device=-1)
    yield m
    m.close()


# ---------------------------------------------------------------------------------------------------- the reference
def test_reference_canonical_form():
    s, w = br.canonical([(3, 0.25), (1, 0.0), (0, 0.75)])
    assert s.tolist() == [0, 3] and w.tolist() == [np.float32(0.75), np.float32(0.25)]
    s1, w1 = br.canonical([(2, 7.5)])
    assert s1.tolist() == [2] and w1.tolist() == [1.0]
    # reordered, zero weights added, scaled by a power of two: the same canonical form
    a = br.canonical([(1, 0.3), (2, 0.7)])
    for other in ([(2, 0.7), (1, 0.3)], [(2, 0.7), (0, 0.0), (1, 0.3)], [(1, 0.3 * 8), (2, 0.7 * 8)]):
        b = br.canonical([(k, np.float32(np.float32(u))) for k, u in other])
        assert a[0].tolist() == b[0].tolist() and a[1].tobytes() == b[1].tobytes(), other
    # w_i = (float)((double)u_i / U), U summed in double in canonical order
    u = [np.float32(0.1), np.float32(0.2), np.float32(0.3)]
    U = float(u[0]) + float(u[1]) + float(u[2])
    assert br.canonical([(5, u[2]), (0, u[0]), (2, u[1])])[1].tolist() == [np.float32(float(x) / U) for x in u]
    for bad in ([], [(1, 0.5), (1, 0.5)], [(0, -1.0)], [(0, float("nan"))], [(0, float("inf"))], [(0, 0.0), (1, 0.0)]):
        with pytest.raises(ValueError):
            br.canonical(bad)


def test_reference_fmaf_rounds_once():
    rng = np.random.default_rng(3)
    a = rng.standard_normal(20000).astype(np.float32)
    b = rng.standard_normal(20000).astype(np.float32) * np.float32(2.0) ** rng.integers(-30, 30, 20000).astype(np.float32)
    c = rng.standard_normal(20000).astype(np.float32)
    got = br._fmaf(a, b, c)
    for i in range(0, 20000, 37):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(exact))
        # the nearest f32 to the exact value (ties to even): compare against both neighbours exactly
        cands = [lo, np.nextafter(lo, np.float32(np.inf)), np.nextafter(lo, np.float32(-np.inf))]
        best = min(cands, key=lambda x: (abs(Fraction(float(x)) - exact), int(np.float32(x).view(np.int32)) & 1))
        assert got[i] == best, (a[i], b[i], c[i])


def test_reference_g_is_within_its_bound():
    rng = np.random.default_rng(5)
    E = rng.standard_normal((6, 256)).astype(np.float32)
    for pairs in ([(1, 0.7), (4, 0.3)], [(0, 1.0), (2, 2.0), (5, 3.0)], [(k, 1.0) for k in range(6)]):
        s, w = br.canonical(pairs)
        g = br.blend_g(E, s, w)
        g64, bound = br.blend_g64(E, s, w)
        assert np.all(np.abs(g.astype(np.float64) - g64) <= bound)
    s, w = br.canonical([(3, 5.0)])
    assert np.array_equal(br.blend_g(E, s, w), E[3])


# ---------------------------------------------------------------------------------------------------- the C image
def test_blend_image_round_trips(m4):
    s, w, o = _blend_arrays(m4, [{"speaker_2": 0.7, 0: 0.3}, None, {3: 1}, {1: 0.0, "speaker_3": 2.5}], 4)
    assert s.dtype == np.int64 and w.dtype == np.float32 and o.dtype == np.uint64
    assert o.tolist() == [0, 2, 2, 3, 5]
    assert s.tolist() == [2, 0, 3, 1, 3]
    assert w.tolist() == [np.float32(0.7), np.float32(0.3), 1.0, 0.0, 2.5]
    assert _blend_arrays(m4, None, 3) == (None, None, None)
    assert _blend_arrays(m4, [None, None], 2) == (None, None, None)
    words = Frontend(group=None, pin=False, model=m4, run_local=lambda *a, **k: [])._encode_blends(
        [{"speaker_2": 0.7, 0: 0.3}, None, {3: 1}], 3)
    back, used = Frontend._decode_blends(words, 3)
    assert used == words.size
    assert back == [{2: float(np.float32(0.7)), 0: float(np.float32(0.3))}, None, {3: 1.0}]


# ---------------------------------------------------------------------------------------------------- refusals
BAD = [  # blend, what the message says
    ({9: 1.0}, "No speaker was found with the given id `9`"),
    ({"nobody": 1.0}, "No speaker was found with the name `nobody`"),
    ({1: 0.5, "speaker_1": 0.5}, "speaker 1 appears more than once"),
    ({2: -0.5}, "weight -0.5 of speaker 2"),
    ({2: float("nan")}, "weight nan of speaker 2"),
    ({2: float("inf")}, "weight inf of speaker 2"),
    ({2: 1e39}, "weight 1e\\+39 of speaker 2"),          # finite in double, infinite in f32
    ({0: 0.0, 3: 0.0}, "every weight is zero"),
    ({}, "the blend is empty"),
    ({2.5: 1.0}, "speaker 2.5 is neither an id nor a name"),
    ({True: 1.0}, "neither an id nor a name"),
    ({2: "0.5"}, "weight '0.5' of speaker 2 is not a number"),
    ([(1, 0.5)], "is not a mapping"),
]


@pytest.mark.parametrize("blend,msg", BAD)
def test_bad_blends_are_refused_by_name_at_every_batch_surface(m4, blend, msg):
    good = {"speaker_0": 0.5, 3: 0.5}
    ids = [[1, 5, 2], [1, 6, 2], [1, 7, 2]]
    blends = [good, None, blend]
    calls = [lambda: m4.infer_batch_with_values(ids, speaker_blends=blends),
             lambda: m4.infer_batch_with_durations(ids, speaker_blends=blends),
             lambda: m4.speak_batch(["ab", "cd", "ef"], speaker_blends=blends),
             lambda: m4.speak_batch_with_alignment(["ab", "cd", "ef"], speaker_blends=blends),
             lambda: m4.infer_batch_g711(ids, "mulaw", speaker_blends=blends),
             lambda: m4.speak_batch_g711(["ab", "cd", "ef"], "alaw", speaker_blends=blends),
             lambda: m4.infer_batch_flac(ids, speaker_blends=blends),
             lambda: m4.speak_batch_flac(["ab", "cd", "ef"], speaker_blends=blends)]
    from sonata_b200.job import SynthesisJob
    calls.append(lambda: SynthesisJob(m4, ids, speaker_blends=blends))
    for call in calls:
        with pytest.raises(OperationError, match="utterance 2: speaker blend: .*" + msg):
            call()


@pytest.mark.parametrize("blend,msg", BAD[:9])
def test_bad_blends_are_refused_by_name_on_streams(s4, blend, msg):
    with pytest.raises(OperationError, match="stream: speaker blend: .*" + msg):
        s4.stream_synthesis("ab", 44, 2, speaker_blend=blend)
    with pytest.raises(OperationError, match="utterance 1: speaker blend: .*" + msg):
        s4.infer_encoder_batch([[1, 5, 2], [1, 6, 2]], speaker_blends=[None, blend])
    sb = StreamBatch(s4, 44, 2)
    sb.add([1, 5, 2], speaker_blend={1: 1.0})
    with pytest.raises(OperationError, match="stream 1: speaker blend: .*" + msg):
        sb.add([1, 6, 2], speaker_blend=blend)
    assert len(sb) == 1                                   # refused at add: nothing was queued
    rb = RealtimeBatch(s4, 44, 2)
    with pytest.raises(OperationError, match="request 0: speaker blend: .*" + msg):
        rb.add("ab", speaker_blend=blend)
    assert len(rb) == 0
    syn = SonataSpeechSynthesizer(s4)
    for mode in (syn.synthesize_lazy, syn.synthesize_parallel, syn.synthesize_streamed):
        with pytest.raises(OperationError, match="request: speaker blend: .*" + msg):
            next(iter(mode("ab", speaker_blend=blend)))
    for mode in (lambda: syn.synthesize_to_file(os.devnull, "ab", speaker_blend=blend),
                 lambda: syn.synthesize_flac("ab", speaker_blend=blend),
                 lambda: next(iter(syn.synthesize_lazy("ab", encoding="mulaw", speaker_blend=blend)))):
        with pytest.raises(OperationError, match="request: speaker blend: .*" + msg):
            mode()


def test_a_single_speaker_voice_refuses_every_blend(m1):
    with pytest.raises(OperationError, match="utterance 0: speaker blend: the voice has a single speaker"):
        m1.infer_batch_with_values([[1, 5, 2]], speaker_blends=[{0: 1.0}])
    assert _blend_arrays(m1, [None], 1) == (None, None, None)


def test_the_c_entry_point_refuses_before_any_device_work(m4, m1):
    lib = N.lib()
    ids = np.array([1, 5, 2, 1, 6, 2], np.int64)
    offs = np.array([0, 3, 6], np.uint64)
    i64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))
    f32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    sz = lambda a: a.ctypes.data_as(C.POINTER(C.c_size_t))
    outs = (N.sb200_audio * 2)()
    cases = [([1, 1], [0.5, 0.5], "utterance 1: speaker blend: speaker 1 appears more than once"),
             ([7], [1.0], "utterance 1: speaker blend: No speaker was found with the given id `7`"),
             ([2], [-1.0], "utterance 1: speaker blend: the weight -1.0+ of speaker 2 is not a finite number >= 0"),
             ([2], [float("nan")], "utterance 1: speaker blend: the weight nan of speaker 2"),
             ([2, 3], [0.0, 0.0], "utterance 1: speaker blend: every weight is zero")]
    for spk, w, msg in cases:
        s = np.array(spk, np.int64)
        wt = np.array(w, np.float32)
        bo = np.array([0, 0, len(spk)], np.uint64)
        err = N.sb200_error()
        rc = lib.sb200_speak_batch_ids_blends(m4._h, i64(ids), sz(offs), 2, None, None, None, None, None, None, None,
                                              None, None, None, None, i64(s), f32(wt), sz(bo), outs, None, None, None,
                                              None, C.byref(err))
        with pytest.raises(OperationError) as e:
            _check(rc, err)
        assert re.search(msg, str(e.value)), str(e.value)
    s, wt, bo = np.array([0], np.int64), np.array([1.0], np.float32), np.array([0, 1, 1], np.uint64)
    err = N.sb200_error()
    rc = lib.sb200_speak_batch_ids_blends(m1._h, i64(ids), sz(offs), 2, None, None, None, None, None, None, None, None,
                                          None, None, None, i64(s), f32(wt), sz(bo), outs, None, None, None, None,
                                          C.byref(err))
    with pytest.raises(OperationError, match="utterance 0: speaker blend: the voice has a single speaker"):
        _check(rc, err)


# ---------------------------------------------------------------------------------------------------- CLI
def test_cli_flag_and_json_field_parse():
    assert cli.parse_speaker_blend("speaker_3=0.7,speaker_12=0.3") == {"speaker_3": 0.7, "speaker_12": 0.3}
    assert cli.parse_speaker_blend("3=0.7, 12 = 0.3") == {3: 0.7, 12: 0.3}
    assert cli.speaker_blend_of({"speaker_3": 0.7, "12": 0.3}) == {"speaker_3": 0.7, 12: 0.3}
    assert cli.speaker_blend_of(None) is None
    args = cli.build_parser().parse_args(["v.onnx.json", "--speaker-blend", "speaker_1=1,2=3"])
    assert cli.speaker_blend_of(args.speaker_blend) == {"speaker_1": 1.0, 2: 3.0}
    for bad in ("speaker_3", "=0.5", "speaker_3=abc"):
        with pytest.raises(OperationError, match="speaker blend"):
            cli.parse_speaker_blend(bad)
    with pytest.raises(OperationError, match="speaker blend"):
        cli.speaker_blend_of([1, 2])


def test_cli_request_refuses_a_bad_blend_in_every_mode(s4):
    syn = SonataSpeechSynthesizer(s4)
    cfg = PiperSynthesisConfig()
    for mode in ("lazy", "parallel", "realtime"):
        req = {"text": "ab", "mode": mode, "speaker_blend": {"speaker_1": 0.5, "9": 0.5}}
        with pytest.raises(OperationError, match="No speaker was found with the given id `9`"):
            cli.process_request(syn, cfg, req, None, out=open(os.devnull, "wb"))


# ---------------------------------------------------------------------------------------------------- Frontend
def _gloo_worker_blends(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from sonata_b200 import shard, workload
    ok = True
    seen = {}

    def fake(ids_list, dst, cap, fmt, **kw):
        waves = [np.repeat(ids.astype(np.float32), 2) for ids in ids_list]
        seen.update(kw)
        seen["ids"] = [ids.copy() for ids in ids_list]
        if dst is not None:
            dst[:] = np.concatenate(waves)
        return [len(w) for w in waves]

    fe = shard.Frontend(group=None, pin=False, run_local=fake)
    for rnd, lens in enumerate(([5, 17, 3, 9, 12, 1, 8], [3, 3, 300000, 3, 3, 3])):
        n = len(lens)
        batches = [workload.synthetic_ids(k, utt=10 * rnd + i) for i, k in enumerate(lens)]
        blends = [None if i % 3 == 0 else {i % 4: 0.25 * i, (i + 1) % 4: 1.0 / 3.0} for i in range(n)]
        seeds = [None if i % 2 else 1000 + i for i in range(n)] if rnd == 0 else None
        seen.clear()
        out = fe.synthesize(batches if rank == 0 else None, seeds=seeds if rank == 0 else None,
                            speaker_blends=blends if rank == 0 else None)
        mine = np.nonzero(fe.last_table[0] == rank)[0]
        want = [None if blends[i] is None else {k: float(np.float32(u)) for k, u in blends[i].items()} for i in mine]
        ok = ok and seen.get("speaker_blends") == want
        ok = ok and (rnd != 0 or seen.get("seeds") == [seeds[i] for i in mine])
        ok = ok and all(np.array_equal(a, batches[i]) for a, i in zip(seen["ids"], mine))
        if rank == 0:
            ok = ok and all(np.array_equal(o, np.repeat(b.astype(np.float32), 2)) for o, b in zip(out, batches))
        del out
    seen.clear()
    fe.synthesize([workload.synthetic_ids(4), workload.synthetic_ids(6)] if rank == 0 else None,
                  speaker_blends=[None, None] if rank == 0 else None)
    ok = ok and "speaker_blends" not in seen              # no blend given: the hook is called without them
    fe.close()
    dist.barrier()
    q.put((rank, bool(ok)))
    dist.destroy_process_group()


def test_frontend_blends_reach_the_owning_rank_gloo_world2():
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker_blends, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(240)
        assert p.exitcode == 0
    assert sorted(q.get(timeout=5) for _ in range(2)) == [(0, True), (1, True)]


def test_frontend_without_blends_broadcasts_todays_block():
    fe = Frontend(group=None, pin=False, run_local=lambda *a, **k: [])
    assert fe._encode_blends(None, 3) is None and fe._encode_blends([None, None, None], 3) is None


# ---------------------------------------------------------------------------------------------------- oracle pin
def test_blend_conditioning_against_live_transformers_run():
    """The 3-speaker high voice with a 4th embedding row holding the float64 blend 0.7 E[0] + 0.3 E[2]: transformers'
    VitsModel speaking as that row and the oracle fed the same g agree within TOL_ORACLE, on the stochastic and the
    deterministic paths."""
    pytest.importorskip("transformers")
    import hf_reference as hf
    from test_hf_pin import TOL_ORACLE
    a = voicegen.ARCH["high"]
    T = dict(voicegen.make_tensors("high", n_speakers=3))
    E = np.asarray(T["emb_g.weight"], np.float64)
    s, w = br.canonical([(0, 0.7), (2, 0.3)])
    g64 = sum(float(wi) * E[si] for si, wi in zip(s, w))
    T["emb_g.weight"] = np.concatenate([np.asarray(T["emb_g.weight"]), g64[None].astype(np.float32)], 0)
    m = hf.load_piper_tensors(hf.build_hf_model(a, n_speakers=4), T, a)
    W = vo.to_torch(T)
    ids = vo.synthetic_ids(16, utt=11)
    outs = {}
    for sid, scales, seed in ((3, (0.667, 1.0, 0.8), 2), (3, (0.0, 1.0, 0.0), 0), (0, (0.0, 1.0, 0.0), 0),
                              (2, (0.0, 1.0, 0.0), 0)):
        wav, ew, ez = hf.hf_infer(m, ids, *scales, seed=seed, speaker_id=sid)
        got = vo.infer(W, ids, list(scales), eps_w=ew[None] if scales[2] else None, eps_z=ez[None] if scales[0] else None,
                       sid=sid).numpy()
        assert got.shape == wav.shape, (sid, got.shape, wav.shape)
        assert float(np.abs(got - wav).max()) < TOL_ORACLE, sid
        outs[(sid, scales[0])] = wav
    for other in (0, 2):            # the blend is neither of its speakers
        x, y = outs[(3, 0.0)], outs[(other, 0.0)]
        assert x.shape != y.shape or float(np.abs(x - y).max()) > 1e-2
