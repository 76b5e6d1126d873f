"""CPU: host-side logic that mirrors the reference's Rust around `session.run`, the C ABI surface,
the weight container and the N>1 sharding plumbing (gloo, world_size 2)."""
import ctypes
import os
import sys
import re

import numpy as np
import pytest

import sonata_b200
from sonata_b200 import AudioSamples, Audio, AdaptiveMelChunker, PiperSynthesisConfig, _native, svw, voicegen
from sonata_b200.core import FailedToLoadResource, OperationError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------- C ABI
def test_library_exports_every_declared_symbol(lib_built):
    hdr = open(os.path.join(ROOT, "include", "sonata_b200.h")).read()
    declared = set(re.findall(r"\b(sb200_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 38
    for name in sorted(declared):
        assert hasattr(lib_built, name), f"{name} declared in include/sonata_b200.h but not exported"
        assert name in _native.SIGNATURES, f"{name} has no ctypes signature"
    assert lib_built.sb200_version().startswith(b"sonata_b200")


def test_struct_layouts_match_header():
    assert ctypes.sizeof(_native.sb200_error) == 16
    assert ctypes.sizeof(_native.sb200_audio) == 24
    assert ctypes.sizeof(_native.sb200_synth_config) == 24
    assert ctypes.sizeof(_native.sb200_audio_info) == 12
    assert ctypes.sizeof(_native.sb200_region_stat) == 64
    assert ctypes.sizeof(_native.sb200_chunk_capture) == 64


# ---------------------------------------------------------------- config / id mapping (piper/src/lib.rs:112-250)
@pytest.fixture(scope="module")
def cfg_model(voice_paths):
    m = sonata_b200.VitsModel(voice_paths["medium"], device=-1)
    yield m
    m.close()


def test_phonemes_to_input_ids(cfg_model):
    # [bos] + (id, pad)* + [eos]; unknown chars dropped silently (:243); 2N+2 ids
    ids = cfg_model.phonemes_to_input_ids("ab")
    assert ids[0] == 1 and ids[-1] == 2 and ids[2] == 0 and ids[4] == 0 and len(ids) == 6
    assert cfg_model.phonemes_to_input_ids("") == [1, 2]
    assert cfg_model.phonemes_to_input_ids("a\U0001F600b") == ids          # emoji not in the map
    ipa = cfg_model.phonemes_to_input_ids("tˈɛst.")                        # golden string of espeak-phonemizer tests
    assert len(ipa) == 2 * 6 + 2 and all(x == 0 for x in ipa[2:-1:2])


def test_config_queries(cfg_model):
    ai = cfg_model.audio_output_info()
    assert (ai.sample_rate, ai.num_channels, ai.sample_width) == (22050, 1, 2)      # :282-288
    assert cfg_model.get_language() == "en_US"
    assert cfg_model.properties() == {"quality": "medium"}
    d = cfg_model.get_default_synthesis_config()
    assert d.speaker == 0 and abs(d.noise_scale - 0.667) < 1e-6 and d.length_scale == 1.0      # :444-451
    assert cfg_model.get_fallback_synthesis_config().speaker is None                           # :54-59
    cfg_model.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.1, 1.5, 0.2))
    f = cfg_model.get_fallback_synthesis_config()
    assert abs(f.noise_scale - 0.1) < 1e-7 and abs(f.length_scale - 1.5) < 1e-7 and abs(f.noise_w - 0.2) < 1e-7
    with pytest.raises(OperationError, match="No speaker was found"):                          # :224-227
        cfg_model.set_fallback_synthesis_config(PiperSynthesisConfig(7, 0.1, 1.0, 0.2))
    with pytest.raises(OperationError, match="Invalid configuration"):
        cfg_model.set_fallback_synthesis_config({"noise_scale": 1})
    assert not cfg_model.supports_streaming_output()
    with pytest.raises(OperationError, match="Streaming synthesis is not supported"):
        cfg_model.stream_synthesis("a", 72, 3)


def test_load_errors(tmp_path, voice_paths):
    with pytest.raises(FailedToLoadResource, match="Faild to load model config"):
        sonata_b200.from_config_path(str(tmp_path / "missing.onnx.json"), device=-1)
    bad = tmp_path / "bad.onnx.json"
    bad.write_text("{not json")
    with pytest.raises(FailedToLoadResource, match="Faild to parse model config"):
        sonata_b200.from_config_path(str(bad), device=-1)
    # no GPU / config-only handle: synthesis must fail loudly, never fall back
    m = sonata_b200.VitsModel(voice_paths["medium"], device=-1)
    with pytest.raises(OperationError, match="no CPU path"):
        m.infer_with_values([1, 5, 0, 2])
    m.close()


# ---------------------------------------------------------------- audio-ops mirror (samples.rs)
def test_to_i16_known_answers():
    assert AudioSamples([]).to_i16_vec().size == 0
    assert AudioSamples([0.0, 0.0, 0.0]).as_wave_bytes() == b"\0" * 6           # eps guard, samples.rs:68
    v = AudioSamples([0.5, -0.25, 0.125]).to_i16_vec()
    assert v.tolist() == [32767, -16383, 8191]                                  # peak-normalised, truncating cast
    v = AudioSamples([-1.0, 1.0]).to_i16_vec()
    assert v.tolist() == [-32767, 32767]
    assert AudioSamples([0.5, -0.25]).as_wave_bytes() == np.array([32767, -16383], "<i2").tobytes()


def test_crossfade_and_audio():
    a = AudioSamples(np.ones(100, np.float32))
    a.crossfade(42)
    s = a.as_slice()
    assert s[0] == 0.0 and s[-1] == 0.0 and abs(s[41] - 1.0) < 1e-6 and s[50] == 1.0
    assert abs(s[1] - np.sin(np.float32(1 / 41) * np.pi / 2)) < 1e-6 and s[1] == s[-2]
    b = AudioSamples(np.ones(10, np.float32))
    b.crossfade(42)                                                             # clamps to len/2
    assert b.as_slice()[4] == 1.0 and b.as_slice()[0] == 0.0
    au = Audio(np.zeros(22050, np.float32), 22050, 250.0)
    assert abs(au.duration_ms() - 1000.0) < 1e-6 and abs(au.real_time_factor() - 0.25) < 1e-9
    assert Audio([], 22050, 3.0).real_time_factor() == 0.0


# ---------------------------------------------------------------- streaming chunk scheduler (piper/src/lib.rs:860-913)
def test_adaptive_mel_chunker_worked_example():
    ch = list(AdaptiveMelChunker(774, 72, 3))
    assert [c[0] for c in ch] == [(0, 75), (69, 222), (216, 441), (435, None)]
    assert [c[1] for c in ch] == [(0, -768), (768, -768), (768, -768), (768, None)]
    # emitted frames are contiguous: 0-72, 72-219, 219-438, 438-774
    covered, pos = 0, 0
    for (m0, m1), (a0, a1) in ch:
        m1 = 774 if m1 is None else m1
        n = (m1 - m0) * 256 - a0 - (0 if a1 is None else -a1)
        assert m0 * 256 + a0 == pos
        pos += n
    assert pos == 774 * 256


@pytest.mark.parametrize("cs,pad", [(72, 3), (100, 3), (55, 3), (45, 3)])
@pytest.mark.parametrize("frames", [100, 150, 151, 774, 3078])
def test_adaptive_mel_chunker_covers_everything(cs, pad, frames):
    pos = 0
    for (m0, m1), (a0, a1) in AdaptiveMelChunker(frames, cs, pad):
        m1e = frames if m1 is None else m1
        assert 0 <= m0 < m1e <= frames
        assert m0 * 256 + a0 == pos
        pos = m1e * 256 + (0 if a1 is None else a1)
    assert pos == frames * 256


# ---------------------------------------------------------------- weight container
def test_svw_roundtrip(tmp_path):
    from collections import OrderedDict
    t = OrderedDict(a=np.arange(7, dtype=np.float32).reshape(7), b=np.arange(6, dtype=np.int32).reshape(2, 3),
                    c=np.float32(3.5).reshape(()))
    p = tmp_path / "t.svw"
    svw.write_svw(p, t)
    r = svw.read_svw(p)
    assert list(r) == ["a", "b", "c"]
    for k in t:
        assert r[k].dtype == t[k].dtype and np.array_equal(r[k], t[k])


def test_voicegen_deterministic_and_calibrated():
    a = voicegen.make_tensors("medium")
    b = voicegen.make_tensors("medium")
    assert all(np.array_equal(a[k], b[k]) for k in a)
    n = sum(v.size for k, v in a.items() if not k.startswith("hp."))
    assert 15.0e6 < n < 16.5e6                      # en_US-lessac-medium is 15.8 M parameters (SURVEY §8d)
    assert voicegen.load_gains("medium") and voicegen.load_gains("high")


# ---------------------------------------------------------------- sharding (SURVEY §8e) on gloo, world_size 2
def test_lpt_partition_balanced():
    from sonata_b200.shard import lpt_partition
    from sonata_b200.workload import mixed_lengths
    lens = mixed_lengths(1024)
    parts = lpt_partition(lens.tolist(), 8)
    assert sorted(i for p in parts for i in p) == list(range(1024))
    loads = [int(lens[p].sum()) for p in parts]
    assert max(loads) - min(loads) <= int(lens.max())
    assert lpt_partition([3, 3, 3, 3], 2) == [[0, 2], [1, 3]]


def _gloo_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from sonata_b200 import shard, workload
    lens = [5, 17, 3, 9, 12, 1, 8]
    batches = [workload.synthetic_ids(n, utt=i) for i, n in enumerate(lens)]

    def fake_synth(mine):        # deterministic stand-in for the CUDA pass: 4 samples per id
        return [np.repeat(ids.astype(np.float32), 4) * 0.5 for ids in mine]

    out = shard.sharded_synthesize(batches if rank == 0 else None, fake_synth)
    if rank == 0:
        ok = all(np.array_equal(o, np.repeat(b.astype(np.float32), 4) * 0.5) for o, b in zip(out, batches))
        q.put(bool(ok) and len(out) == len(batches))
    dist.barrier()
    dist.destroy_process_group()


def _gloo_worker_frontend(rank, world, port, q):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from sonata_b200 import shard, workload
    ok = True
    for pcm16 in (False, True):
        def fake(ids_list, dst, cap, fmt, pcm16=pcm16):       # deterministic stand-in for the CUDA pass: 3 samples per id
            waves = [(np.repeat(ids.astype(np.float32), 3) % 100).astype(np.int16 if pcm16 else np.float32) for ids in ids_list]
            if dst is not None:
                flat = np.concatenate(waves)
                assert flat.nbytes == cap and fmt == (1 if pcm16 else 0)
                dst[:] = flat
            return [len(w) for w in waves]
        fe = shard.Frontend(group=None, pcm16=pcm16, pin=False, run_local=fake)
        for rnd, lens in enumerate(([5, 17, 3, 9, 12, 1, 8], [40, 2], [3, 3, 3, 3, 3, 3, 3, 3, 400000])):   # round 3 grows the segment
            batches = [workload.synthetic_ids(n, utt=10 * rnd + i) for i, n in enumerate(lens)]
            out = fe.synthesize(batches if rank == 0 else None)
            if rank == 0:
                dt = np.int16 if pcm16 else np.float32
                ok = ok and len(out) == len(batches) and all(
                    o.dtype == dt and np.array_equal(o, (np.repeat(b.astype(np.float32), 3) % 100).astype(dt)) for o, b in zip(out, batches))
                owner, samples = fe.last_table
                ok = ok and sorted(set(owner.tolist())) == [0, 1] and samples.tolist() == [3 * len(b) for b in batches]
            else:
                ok = ok and out is None
            del out
        ok = ok and fe.synthesize([workload.synthetic_ids(4)] if rank == 0 else None, device_only=True) is None
        fe.close()
    dist.barrier()
    if rank == 0:
        q.put(bool(ok))
    dist.destroy_process_group()


def test_frontend_shared_segment_gloo_world2():
    """`shard.Frontend`: rank 0 broadcasts the ids, every rank writes its waveforms (f32 or i16) into its slice of one
    shared host segment, rank 0 reads them in utterance order; the segment grows on demand and is reused."""
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker_frontend, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(180)
        assert p.exitcode == 0
    assert q.get(timeout=5) is True


def test_sharded_synthesize_gloo_world2():
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    assert q.get(timeout=5) is True


def test_c5_length_buckets_and_completion_stats():
    """SURVEY §8d C5 scheduling helpers (tools/bench_c5.py): longest-first buckets, latency percentiles."""
    from sonata_b200 import workload
    n = workload.mixed_lengths(1024)
    assert n.shape == (1024,) and n.min() >= 64 and n.max() <= 512
    assert np.array_equal(n, workload.mixed_lengths(1024))                 # seeded
    b = workload.length_buckets(n, 32)
    assert len(b) == 32 and all(len(x) == 32 for x in b)
    flat = [i for x in b for i in x]
    assert sorted(flat) == list(range(1024))
    mx = [max(n[i] for i in x) for x in b]; mn = [min(n[i] for i in x) for x in b]
    assert all(mn[k] >= mx[k + 1] for k in range(len(b) - 1))              # longest first, non-overlapping ranges
    assert workload.length_buckets([5, 9, 7], 2) == [[1, 2], [0]]
    p50, p99, agg = workload.completion_stats([[0, 1], [2]], [1.0, 3.0], [4.0, 2.0])
    assert p50 == 1.0 and abs(p99 - 2.96) < 1e-9 and agg == 2.0
    assert workload.completion_stats([], [], []) == (0.0, 0.0, 0.0)


def test_tensor_core_emulation_primitives():
    """tools/emu_tc_accuracy.py (round-2 planning): operand rounding matches torch's bf16 cast, the truncating fp32
    conversion never rounds away from zero, and flushing the accumulator reduces the error of a long contraction."""
    import torch
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import emu_tc_accuracy as emu
    rng = np.random.default_rng(3)
    x = (rng.standard_normal(4096) * np.exp(rng.uniform(-20, 20, 4096))).astype(np.float32)
    assert np.array_equal(emu.round_to_bits(x, 8), torch.from_numpy(x).to(torch.bfloat16).to(torch.float32).numpy())
    hi = emu.round_to_bits(x, 11)
    assert np.all(np.abs(hi - x) <= np.abs(x) * 2.0 ** -11) and np.all((hi.view(np.uint32) & 0x1FFF) == 0)
    v = rng.standard_normal(2048) * 1e3
    rz = emu.to_f32(v, "rz").astype(np.float64)
    assert np.all(np.abs(rz) <= np.abs(v)) and np.all(np.abs(rz - v) <= np.abs(v) * 2.0 ** -23)
    a = rng.standard_normal((16, 1024)).astype(np.float32)
    b = (rng.standard_normal((1024, 8)) / 32).astype(np.float32)
    ref = a.astype(np.float64) @ b.astype(np.float64)
    plain = np.abs(emu.emulate(a, b, "tf32", "rz", 0) - ref).max()
    chunked = np.abs(emu.emulate(a, b, "tf32", "rz", 8) - ref).max()
    assert chunked < plain and chunked < 5e-6
