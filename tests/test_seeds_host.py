"""Per-utterance noise seeds without a GPU: the host restatement of the keyed draws (tests/noise_reference.py) against
Random123's Philox4x32-10 known answers and N(0, 1), and the argument checks of every `seeds=` entry point, which run
before any device work."""
import json
import os
import sys

import numpy as np
import pytest
from scipy import stats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import noise_reference as nr
import sonata_b200
from sonata_b200 import OperationError
from sonata_b200.job import SynthesisJob
from sonata_b200.piper import StreamBatch, VitsStreamingModel, _seed_arrays


# ---------------------------------------------------------------- Philox4x32-10 known answers (Random123 kat_vectors)
@pytest.mark.parametrize("ctr, key, want", [
    ([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
    ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
    ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
     [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]),
])
def test_philox_known_answers(ctr, key, want):
    got = nr.philox4x32_10(np.array([ctr], np.uint32), np.array(key, np.uint32))
    assert [int(x) for x in got[0]] == want


def test_seeded_counter_layout():
    """Quad q of a seeded tensor is counter (q, q >> 32, tag, 0) under key (seed, seed >> 32)."""
    seed = 0x0123456789ABCDEF
    bits = nr.seeded_bits(seed, 1, 3, 192)
    for q in (0, 1, 143):
        one = nr.philox4x32_10(np.array([[q, 0, 1, 0]], np.uint32), np.array([0x89ABCDEF, 0x01234567], np.uint32))
        assert np.array_equal(bits[q], one[0])
    # prefix stability: the first frames do not depend on how many follow
    assert np.array_equal(nr.eps_z(seed, 5, 192), nr.eps_z(seed, 9, 192)[:5])
    assert np.array_equal(nr.eps_w(seed, 7), nr.eps_w(seed, 8)[:7])


# ---------------------------------------------------------------- distribution of the restated draws
N_DRAWS = 1 << 20


@pytest.mark.parametrize("seed", [0, 1, 2**64 - 1, 0x5eed5eed])
@pytest.mark.parametrize("tag", [0, 1])
def test_seeded_draws_are_standard_normal(seed, tag):
    x = nr.seeded_normals(seed, tag, N_DRAWS // 4, 4).reshape(-1)
    n = x.size
    assert abs(x.mean()) < 5 / np.sqrt(n)
    assert abs(x.var() - 1.0) < 5 * np.sqrt(2.0 / n)
    assert stats.kstest(x, "norm").pvalue > 1e-3


@pytest.mark.parametrize("seed", [0, 41, 2**63])
def test_neighbouring_seeds_and_streams_are_uncorrelated(seed):
    rows = N_DRAWS // 192
    a = nr.eps_z(seed, rows, 192).reshape(-1)
    b = nr.eps_z((seed + 1) % 2**64, rows, 192).reshape(-1)
    w = nr.eps_w(seed, a.size // 2).reshape(-1)
    lim = 5 / np.sqrt(a.size)
    assert abs(np.corrcoef(a, b)[0, 1]) < lim
    assert abs(np.corrcoef(a, w)[0, 1]) < lim


# ---------------------------------------------------------------- argument checks
def test_seed_arrays_pack_and_flag():
    assert _seed_arrays(None, 3) == (None, None)
    assert _seed_arrays([None, None], 2) == (None, None)        # no seed: the call without seeds
    v, f = _seed_arrays([5, None, 2**64 - 1], 3)
    assert v.dtype == np.uint64 and f.dtype == np.int32
    assert [int(x) for x in v] == [5, 0, 2**64 - 1] and list(f) == [1, 0, 1]
    v, f = _seed_arrays(np.array([3, 4], np.uint64), 2)
    assert [int(x) for x in v] == [3, 4] and list(f) == [1, 1]


@pytest.mark.parametrize("seeds, msg", [
    ([1], "1 entries for 2 utterances"),
    ([1, -1], "utterance 1: noise seed -1 is not in"),
    ([2**64, 1], "utterance 0: noise seed 18446744073709551616 is not in"),
    ([1.0, 1], "utterance 0: noise seed 1.0 is not an integer"),
    ([True, 1], "utterance 0: noise seed True is not an integer"),
    ([None, "7"], "utterance 1: noise seed '7' is not an integer"),
    (7, "expected one entry"),
])
def test_seed_argument_errors(seeds, msg):
    with pytest.raises(OperationError, match=msg):
        _seed_arrays(seeds, 2)


@pytest.fixture(scope="module")
def config_only(voice_paths, tmp_path_factory):
    cfg = json.load(open(voice_paths["medium"], encoding="utf-8"))
    d = tmp_path_factory.mktemp("seeds")
    plain, streaming = d / "plain.onnx.json", d / "streaming.onnx.json"
    plain.write_text(json.dumps(cfg), encoding="utf-8")
    cfg["streaming"] = True
    streaming.write_text(json.dumps(cfg), encoding="utf-8")
    m = sonata_b200.VitsModel(str(plain), device=-1)
    s = VitsStreamingModel(str(streaming), device=-1)
    yield m, s
    m.close()
    s.close()


def test_every_seeds_entry_point_checks_before_the_device(config_only):
    m, s = config_only
    bad = [3, -2]
    ids = [[1, 5, 2], [1, 6, 2]]
    calls = [
        lambda: m.infer_batch_with_values(ids, seeds=bad),
        lambda: m.speak_batch(["at", "ta"], seeds=bad),
        lambda: m.infer_batch_with_durations(ids, seeds=bad),
        lambda: m.speak_batch_with_alignment(["at", "ta"], seeds=bad),
        lambda: s.infer_encoder_batch(ids, seeds=bad),
        lambda: SynthesisJob(m, ids, seeds=bad),
    ]
    for call in calls:
        with pytest.raises(OperationError, match="utterance 1: noise seed -2"):
            call()
    with pytest.raises(OperationError, match="utterance 0: noise seed -1"):
        s.stream_synthesis("at", 45, 3, seed=-1)
    with pytest.raises(OperationError, match="noise seed 'x' is not an integer"):
        StreamBatch(s, 45, 3).add([1, 5, 2], seed="x")
    # good seeds reach the library, which has no CPU path
    with pytest.raises(OperationError, match="no CPU path"):
        m.infer_batch_with_values(ids, seeds=[3, None])
    with pytest.raises(OperationError, match="no CPU path"):
        s.infer_encoder_batch(ids, seeds=[None, 2**64 - 1])


# ---------------------------------------------------------------- frontends
def test_sentence_seed_wraps_and_checks():
    from sonata_b200.synth import sentence_seed
    assert sentence_seed(None, 3) is None
    assert [sentence_seed(2**64 - 2, i) for i in range(3)] == [2**64 - 2, 2**64 - 1, 0]
    with pytest.raises(OperationError, match="noise seed -1"):
        sentence_seed(-1, 0)


def test_seed_words_round_trip():
    from sonata_b200.shard import Frontend
    seeds = [None, 0, 2**64 - 1, 2**63, 12345]
    words = Frontend._encode_seeds(seeds, 5)
    assert words.dtype == np.int64 and words.shape == (10,)
    assert Frontend._decode_seeds(words) == seeds
    with pytest.raises(OperationError, match="utterance 1"):
        Frontend._encode_seeds([1, 2**64], 2)


def _gloo_worker_seeds(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from sonata_b200 import shard, workload
    ok = True
    seen = {}

    def fake(ids_list, dst, cap, fmt, **kw):     # 2 samples per id; remembers what arrived
        waves = [np.repeat(ids.astype(np.float32), 2) for ids in ids_list]
        seen.update(kw)
        seen["ids"] = [ids.copy() for ids in ids_list]
        if dst is not None:
            dst[:] = np.concatenate(waves)
        return [len(w) for w in waves]

    fe = shard.Frontend(group=None, pin=False, run_local=fake)
    # round 2 has more than 2^18 int64 words: its seeds travel in the second broadcast block
    for rnd, lens in enumerate(([5, 17, 3, 9, 12, 1, 8], [3, 3, 300000, 3, 3, 3])):
        batches = [workload.synthetic_ids(n, utt=10 * rnd + i) for i, n in enumerate(lens)]
        seeds = [None if i % 3 == 1 else (2**64 - 1 - i if i % 2 else i * 1000) for i in range(len(lens))]
        cfgs = [sonata_b200.PiperSynthesisConfig(None, 0.1 * i, 1.0, 0.8) for i in range(len(lens))] if rnd else None
        seen.clear()
        out = fe.synthesize(batches if rank == 0 else None, configs=cfgs if rank == 0 else None,
                            seeds=seeds if rank == 0 else None)
        mine = np.nonzero(fe.last_table[0] == rank)[0]
        ok = ok and seen.get("seeds") == [seeds[i] for i in mine]
        ok = ok and (cfgs is None) == ("configs" not in seen)
        ok = ok and all(np.array_equal(a, batches[i]) for a, i in zip(seen["ids"], mine))
        if rank == 0:
            ok = ok and all(np.array_equal(o, np.repeat(b.astype(np.float32), 2)) for o, b in zip(out, batches))
        del out
    seen.clear()
    fe.synthesize([workload.synthetic_ids(4), workload.synthetic_ids(6)] if rank == 0 else None)
    ok = ok and "seeds" not in seen                      # no seeds given: the hook is called without them
    fe.close()
    dist.barrier()
    q.put((rank, bool(ok)))
    dist.destroy_process_group()


def test_frontend_seeds_reach_the_owning_rank_gloo_world2():
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker_seeds, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(240)
        assert p.exitcode == 0
    assert sorted(q.get(timeout=5) for _ in range(2)) == [(0, True), (1, True)]


class _FakeSynth:
    def __init__(self):
        self.calls = []
        self.model = self

    def set_fallback_synthesis_config(self, cfg):
        pass

    def synthesize_lazy(self, text, oc, seed=None):
        self.calls.append(("lazy", seed))
        return iter([])

    def synthesize_parallel(self, text, oc, seed=None):
        self.calls.append(("parallel", seed))
        return iter([])

    def synthesize_streamed(self, text, oc, cs, cp, seed=None):
        self.calls.append(("realtime", seed))
        return iter([])

    def synthesize_to_file(self, path, text, oc, seed=None):
        self.calls.append(("file", seed))


def test_cli_reads_the_seed_field_and_flag(monkeypatch, tmp_path):
    import io
    from sonata_b200 import cli
    assert cli.build_parser().parse_args(["v.json", "--seed", "18446744073709551615"]).seed == 2**64 - 1
    assert cli.build_parser().parse_args(["v.json"]).seed is None
    fake = _FakeSynth()
    default = sonata_b200.PiperSynthesisConfig()
    for mode in ("lazy", "parallel", "realtime"):
        cli.process_request(fake, default, {"text": "a", "mode": mode, "seed": 9}, None, out=io.BytesIO())
    cli.process_request(fake, default, {"text": "a", "seed": 4}, str(tmp_path / "o.wav"))
    cli.process_request(fake, default, {"text": "a"}, None, out=io.BytesIO())
    assert fake.calls == [("lazy", 9), ("parallel", 9), ("realtime", 9), ("file", 4), ("lazy", None)]
    # stdin requests: the flag is the default, a request's own field wins
    monkeypatch.setattr(cli, "from_config_path", lambda path, device: _Closable())
    monkeypatch.setattr(cli, "SonataSpeechSynthesizer", lambda model: fake)
    monkeypatch.setattr(sys, "stdin", io.StringIO('{"text": "a"}\n{"text": "b", "seed": 2}\n'))
    monkeypatch.setattr(sys, "stdout", type("O", (), {"buffer": io.BytesIO()})())
    fake.calls.clear()
    assert cli.main(["v.json", "--seed", "7"]) == 0
    assert fake.calls == [("lazy", 7), ("lazy", 2)]


class _Closable:
    def get_default_synthesis_config(self):
        return sonata_b200.PiperSynthesisConfig()

    def close(self):
        pass
