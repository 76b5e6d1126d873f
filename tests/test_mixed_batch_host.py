"""CPU: the host side of per-utterance synthesis configs -- Python argument checks and the configs' trip through
`shard.Frontend` (gloo, world size 2).  The C entry points are covered by test_host's header / export check."""
import os

import numpy as np
import pytest

import sonata_b200
from sonata_b200 import PiperSynthesisConfig
from sonata_b200.core import OperationError
from sonata_b200.piper import _config_array
from sonata_b200.shard import Frontend


def test_config_array_checks_its_arguments():
    assert _config_array(None, 3) is None
    arr = _config_array([PiperSynthesisConfig(None, 0.5, 1.25, 0.0), PiperSynthesisConfig(3, 0.667, 1.0, 0.8)], 2)
    assert (arr[0].has_speaker, arr[0].speaker, arr[0].noise_scale, arr[0].length_scale, arr[0].noise_w) == (0, 0, 0.5, 1.25, 0.0)
    assert (arr[1].has_speaker, arr[1].speaker) == (1, 3)
    with pytest.raises(OperationError, match="2 configs for 3 utterances"):
        _config_array([PiperSynthesisConfig()] * 2, 3)
    with pytest.raises(OperationError, match="utterance 1"):
        _config_array([PiperSynthesisConfig(), {"speaker": 1}], 2)


def test_model_entry_points_check_lengths_before_any_device_work(voice_paths):
    m = sonata_b200.VitsModel(voice_paths["medium"], device=-1)      # config only: a device call would fail differently
    with pytest.raises(OperationError, match="1 configs for 2 utterances"):
        m.infer_batch_with_values([[1, 5, 2], [1, 6, 2]], [PiperSynthesisConfig()])
    with pytest.raises(OperationError, match="3 configs for 1 utterances"):
        m.speak_batch(["ab"], [PiperSynthesisConfig()] * 3)
    with pytest.raises(OperationError, match="1 configs for 0 utterances"):
        m.speak_batch([], [PiperSynthesisConfig()])
    assert m.speak_batch([], []) == []
    m.close()


def test_config_image_round_trips():
    cfgs = [PiperSynthesisConfig(None, 0.667, 1.0, 0.8), PiperSynthesisConfig(31, 0.1 + 0.2, 1e-7, 0.0),
            PiperSynthesisConfig(0, -0.0, 3.5, 1.0 / 3.0)]
    words = Frontend._encode_configs(cfgs)
    assert words.dtype == np.int64 and words.shape == (12,)
    back = Frontend._decode_configs(words)
    assert back == cfgs and np.signbit(back[2].noise_scale)


def _gloo_worker_configs(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from sonata_b200 import shard, workload
    ok = True
    seen = {}

    def fake(ids_list, dst, cap, fmt, configs=None):     # 2 samples per id; remembers what arrived
        waves = [np.repeat(ids.astype(np.float32), 2) for ids in ids_list]
        seen["configs"] = configs
        seen["ids"] = [ids.copy() for ids in ids_list]
        if dst is not None:
            dst[:] = np.concatenate(waves)
        return [len(w) for w in waves]

    def legacy(ids_list, dst, cap, fmt):                  # a hook written before configs existed
        waves = [np.repeat(ids.astype(np.float32), 2) for ids in ids_list]
        if dst is not None:
            dst[:] = np.concatenate(waves)
        return [len(w) for w in waves]

    fe = shard.Frontend(group=None, pin=False, run_local=fake)
    # round 2 has more than 2^18 int64 words: its configs travel in the second broadcast block
    for rnd, lens in enumerate(([5, 17, 3, 9, 12, 1, 8], [3, 3, 300000, 3, 3, 3])):
        batches = [workload.synthetic_ids(n, utt=10 * rnd + i) for i, n in enumerate(lens)]
        cfgs = [PiperSynthesisConfig(None if i % 3 == 0 else i, 0.1 * i, 1.0 + 0.01 * i, 0.8 - 0.05 * i)
                for i in range(len(lens))]
        out = fe.synthesize(batches if rank == 0 else None, configs=cfgs if rank == 0 else None)
        owner = fe.last_table[0]
        mine = np.nonzero(owner == rank)[0]
        ok = ok and seen["configs"] == [cfgs[i] for i in mine]                    # owning rank, utterance order
        ok = ok and all(np.array_equal(a, batches[i]) for a, i in zip(seen["ids"], mine))
        if rank == 0:
            ok = ok and all(np.array_equal(o, np.repeat(b.astype(np.float32), 2)) for o, b in zip(out, batches))
        del out
    fe.synthesize([workload.synthetic_ids(4), workload.synthetic_ids(6)] if rank == 0 else None)
    ok = ok and seen["configs"] is None                   # no configs given: the hook is called without them
    fe.close()
    fe = shard.Frontend(group=None, pin=False, run_local=legacy)
    out = fe.synthesize([workload.synthetic_ids(4), workload.synthetic_ids(6)] if rank == 0 else None)
    ok = ok and (rank != 0 or len(out) == 2)
    del out
    fe.close()
    dist.barrier()
    q.put((rank, bool(ok)))
    dist.destroy_process_group()


def test_frontend_configs_reach_the_owning_rank_gloo_world2():
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker_configs, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(240)
        assert p.exitcode == 0
    assert sorted(q.get(timeout=5) for _ in range(2)) == [(0, True), (1, True)]
