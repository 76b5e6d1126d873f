"""Utterance-level sharding across the GPUs of one box (SURVEY §8(e)).

Utterances are independent (the reference already treats sentences as independent tasks,
synth/src/lib.rs:316-320), so the path shards with NO data-path collective: the only exchanges are
the scatter of ids from rank 0 and the collection of waveforms at rank 0, done with torch.distributed (NCCL over
NVLink on GPUs; gloo in the CPU tests).  Weights are replicated.  `Frontend` is the production path (ids broadcast,
results through a page-locked host segment shared by the ranks); `scatter_ids` / `gather_waveforms` keep the plain
NCCL scatter / gather into rank 0's HBM for comparison.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch
import torch.distributed as dist


def lpt_partition(costs: Sequence[float], world: int) -> List[List[int]]:
    """Longest-processing-time greedy: sort by cost descending, give each to the least loaded rank.
    Cost ~ T_x (frames ~ 3 T_x).  Returns, per rank, utterance indices in ascending order."""
    import heapq
    order = sorted(range(len(costs)), key=lambda i: (-costs[i], i))
    heap = [(0.0, r) for r in range(world)]           # (load, rank): ties go to the lowest rank
    parts: List[List[int]] = [[] for _ in range(world)]
    for i in order:
        load, r = heapq.heappop(heap)
        parts[r].append(i)
        heapq.heappush(heap, (load + costs[i], r))
    return [sorted(p) for p in parts]


def _dev(group=None) -> torch.device:
    return torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else torch.device("cpu")


def scatter_ids(batches: Optional[Sequence[np.ndarray]], group=None) -> List[np.ndarray]:
    """Rank 0 passes the full list of id sequences; every rank returns its own shard (LPT).
    Also returns nothing else: global indices are recovered by gather_waveforms."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    dev = _dev(group)
    if rank == 0:
        lens = np.array([len(b) for b in batches], dtype=np.int64)
        parts = lpt_partition(lens.tolist(), world)
        owner = np.zeros(len(batches), dtype=np.int64)
        for r, p in enumerate(parts):
            owner[p] = r
        meta = torch.tensor([len(batches)], dtype=torch.int64, device=dev)
    else:
        meta = torch.zeros(1, dtype=torch.int64, device=dev)
    dist.broadcast(meta, 0, group=group)
    n = int(meta.item())
    table = torch.zeros(2, n, dtype=torch.int64, device=dev)
    if rank == 0:
        table[0] = torch.from_numpy(lens).to(dev)
        table[1] = torch.from_numpy(owner).to(dev)
    dist.broadcast(table, 0, group=group)
    lens_all = table[0].cpu().numpy()
    owner_all = table[1].cpu().numpy()
    mine = np.nonzero(owner_all == rank)[0]
    per_rank_tot = [int(lens_all[owner_all == r].sum()) for r in range(world)]
    cap = max(max(per_rank_tot), 1)
    recv = torch.zeros(cap, dtype=torch.int64, device=dev)
    if rank == 0:
        sl = []
        for r in range(world):
            buf = torch.zeros(cap, dtype=torch.int64)
            idx = np.nonzero(owner_all == r)[0]
            if len(idx):
                buf[:per_rank_tot[r]] = torch.from_numpy(np.concatenate([np.asarray(batches[i], dtype=np.int64) for i in idx]))
            sl.append(buf.to(dev))
        dist.scatter(recv, sl, src=0, group=group)
    else:
        dist.scatter(recv, None, src=0, group=group)
    flat = recv.cpu().numpy()
    out, o = [], 0
    for i in mine:
        out.append(flat[o:o + int(lens_all[i])].copy())
        o += int(lens_all[i])
    scatter_ids.last = {"mine": mine, "owner": owner_all, "n": n}
    return out


def gather_waveforms(local_wave: torch.Tensor, local_lens: Sequence[int], group=None, to_host: bool = True):
    """`local_wave`: this rank's utterances concatenated (device tensor for NCCL, 1-D float32);
    `local_lens`: samples per local utterance.  Rank 0 returns the waveforms in GLOBAL utterance order."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    dev = _dev(group)
    info = scatter_ids.last
    n, owner, mine = info["n"], info["owner"], info["mine"]
    lens = torch.zeros(n, dtype=torch.int64, device=dev)
    if len(mine):
        lens[torch.from_numpy(mine).to(dev)] = torch.tensor(list(local_lens), dtype=torch.int64, device=dev)
    dist.all_reduce(lens, group=group)
    lens_all = lens.cpu().numpy()
    tot = [int(lens_all[owner == r].sum()) for r in range(world)]
    cap = max(max(tot), 1)
    send = torch.zeros(cap, dtype=torch.float32, device=dev)
    send[:tot[rank]] = local_wave[:tot[rank]].to(dev)
    if rank == 0:
        gl = [torch.empty(cap, dtype=torch.float32, device=dev) for _ in range(world)]
        dist.gather(send, gl, dst=0, group=group)
        if not to_host:          # device-resident result: per-rank buffers + the tables to slice them
            return gl, owner, lens_all
        out: List[Optional[np.ndarray]] = [None] * n
        for r in range(world):
            flat = gl[r].cpu().numpy()
            o = 0
            for i in np.nonzero(owner == r)[0]:
                out[i] = flat[o:o + int(lens_all[i])].copy()
                o += int(lens_all[i])
        return out  # type: ignore[return-value]
    dist.gather(send, None, dst=0, group=group)
    return None


class SharedSegment:
    """A host memory segment mapped by every rank of the box (file-backed MAP_SHARED mapping on a RAM filesystem when
    one has room, else the temp directory), optionally page-locked through the library (`sb200_host_register`) so
    device->host copies into it are DMA transfers.  Grown on demand; the name travels over the process group."""

    def __init__(self, group=None, pin: bool = True):
        self.group, self.pin = group, pin
        self.path, self.mm, self.cap, self._fd = None, None, 0, None
        self._reg_ptr, self._np = None, None

    @staticmethod
    def _pick_dir(nbytes: int) -> str:
        import tempfile
        for d in ("/dev/shm", tempfile.gettempdir()):
            try:
                st = os.statvfs(d)
                if st.f_bavail * st.f_frsize > nbytes + (64 << 20):
                    return d
            except OSError:
                continue
        return tempfile.gettempdir()

    def ensure(self, nbytes: int) -> None:
        """collective: every rank calls with the same `nbytes`"""
        if nbytes <= self.cap:
            return
        import mmap
        rank = dist.get_rank(self.group)
        self.close()
        cap = max(int(nbytes * 1.25), 1 << 20)
        cap = (cap + 4095) & ~4095
        name = [None]
        if rank == 0:
            import tempfile
            fd, path = tempfile.mkstemp(prefix="sb200_seg_", dir=self._pick_dir(cap))
            os.ftruncate(fd, cap)
            name[0] = path
            self._fd = fd
        dist.broadcast_object_list(name, src=0, group=self.group)
        self.path = name[0]
        if rank != 0:
            self._fd = os.open(self.path, os.O_RDWR)
        self.mm = mmap.mmap(self._fd, cap, mmap.MAP_SHARED, mmap.PROT_READ | mmap.PROT_WRITE)
        self._np = np.frombuffer(self.mm, dtype=np.uint8)
        self.cap = cap
        if self.pin:
            try:
                from . import _native as N
                lib = N.lib()
                if int(lib.sb200_device_count()) > 0:
                    err = N.sb200_error()
                    if int(lib.sb200_host_register(self._np.ctypes.data, cap, C.byref(err))) == 0:
                        self._reg_ptr = self._np.ctypes.data
                    elif err.message:
                        lib.sb200_string_free(err.message)     # copies still work, through pageable memory
            except ImportError:
                pass
        dist.barrier(group=self.group)
        if rank == 0:
            os.unlink(self.path)          # every rank holds its mapping; the name is no longer needed

    @property
    def address(self) -> int:
        return self._np.ctypes.data

    def view(self, offset: int, nbytes: int, dtype) -> np.ndarray:
        return self._np[offset:offset + nbytes].view(dtype)

    def close(self) -> None:
        if self.mm is None:
            return
        if self._reg_ptr is not None:
            from . import _native as N
            N.lib().sb200_host_unregister(self._reg_ptr)
            self._reg_ptr = None
        self._np = None
        try:
            self.mm.close()
        except BufferError:
            pass                                   # views handed out earlier are still alive
        if self._fd is not None:
            os.close(self._fd)
        self.mm, self.cap, self._fd = None, 0, None


class Frontend:
    """ONE frontend process (rank 0) serving a batch of utterances on every GPU of the box: the multi-GPU form of
    `SonataSpeechStreamParallel::new` (synth/src/lib.rs:314-325: fan the sentences out, collect every result).

      rank 0 : ids of all utterances  --NCCL broadcast (ids + LPT owner table, ~1 MB)-->  every rank
      rank r : its shard as ONE batched pass on its GPU (weights replicated)
      all    : per-utterance sample counts  --NCCL all-reduce (n int64)-->  exact layout of the result segment
      rank r : device -> host copy of its waveforms straight into ITS SLICE of a page-locked host segment shared by
               all ranks -- N PCIe links in parallel instead of funnelling every GPU's audio through rank 0
               (NCCL gather + one copy)
      rank 0 : after a barrier, reads every waveform from the same pages (zero-copy numpy views)

    `pcm16=True` delivers peak-normalised i16 PCM converted on the device (`to_i16_vec`, samples.rs:51-75): what
    libsonata's callback receives, at half the device->host bytes.  Every device / host buffer is allocated once and
    reused; the collectives carry only ids, per-utterance configs and length tables.  `run_local(ids_list, dst, capacity,
    fmt)` is the per-rank synthesis hook (default: the CUDA job of `model`), called with `configs=` (the shard's configs in
    its utterance order) only when the caller gave configs, and `seeds=` likewise; the gloo tests pass a deterministic
    stand-in."""

    def __init__(self, model=None, group=None, pcm16: bool = False, pin: bool = True, run_local: Optional[Callable] = None):
        self.model, self.group, self.pcm16 = model, group, pcm16
        self.seg = SharedSegment(group, pin)
        self.run_local = run_local
        self._payload = None           # device buffer for the id broadcast (first block)
        self._host = None              # page-locked host staging of the same
        self._big = None               # device buffer for inputs beyond the first block
        self._lens = None              # device / page-locked host buffers for the sample-count all-reduce
        self._lens_h = None
        self.last_device_ms = 0.0
        self.last_table = None
        self.collect_profile = False   # keep the per-region device times of the last local pass (bench.py)
        self.last_profile = []

    # -- collective plumbing ----------------------------------------------------------------------------------------
    FIRST_BLOCK = 1 << 18      # int64 elements (2 MB) of the first broadcast: [n, total, has, lens, owner, ids ...,
    #                            configs: 4 words per utterance when has & 1, seeds: 2 words per utterance when has & 2]

    @staticmethod
    def _encode_configs(configs) -> np.ndarray:
        """int64 image of per-utterance PiperSynthesisConfigs: speaker (-1 for None), then the bits of noise_scale,
        length_scale and noise_w as float64 (exact for any Python float)."""
        out = np.empty((len(configs), 4), dtype=np.int64)
        out[:, 0] = [-1 if c.speaker is None else int(c.speaker) for c in configs]
        out[:, 1:] = np.array([[c.noise_scale, c.length_scale, c.noise_w] for c in configs],
                              dtype=np.float64).reshape(-1, 3).view(np.int64)
        return out.reshape(-1)

    @staticmethod
    def _decode_configs(words: np.ndarray) -> list:
        from .piper import PiperSynthesisConfig
        w = words.reshape(-1, 4)
        f = np.ascontiguousarray(w[:, 1:]).view(np.float64)
        return [PiperSynthesisConfig(None if s < 0 else int(s), float(a), float(b), float(c))
                for s, (a, b, c) in zip(w[:, 0].tolist(), f.tolist())]

    @staticmethod
    def _encode_seeds(seeds, n: int) -> np.ndarray:
        """int64 image of per-utterance noise seeds: [seeded flag, the seed's 64 bits] per utterance."""
        from .piper import _seed_arrays
        vals, flags = _seed_arrays(seeds, n)
        out = np.zeros((n, 2), dtype=np.int64)
        if vals is not None:
            out[:, 0] = flags
            out[:, 1] = vals.view(np.int64)
        return out.reshape(-1)

    @staticmethod
    def _decode_seeds(words: np.ndarray) -> list:
        w = np.ascontiguousarray(words.reshape(-1, 2))
        vals = w[:, 1].view(np.uint64)
        return [int(v) if f else None for f, v in zip(w[:, 0].tolist(), vals.tolist())]

    def _bcast_ids(self, batches, configs=None, seeds=None):
        """ONE broadcast of a fixed-size block carries the header and (for up to ~260k ids) everything else, the
        per-utterance configs included; a second broadcast follows only for larger inputs.  Host staging buffers are
        page-locked and reused.  Seeds, when given, follow the configs; without them the block is what it always was."""
        rank, world = dist.get_rank(self.group), dist.get_world_size(self.group)
        dev = _dev(self.group)
        fb = self.FIRST_BLOCK
        if self._payload is None:
            self._payload = torch.empty(fb, dtype=torch.int64, device=dev)
            pin = dev.type == "cuda"
            self._host = torch.empty(fb, dtype=torch.int64, pin_memory=pin)
        total = 0
        if rank == 0:
            lens = np.fromiter((len(b) for b in batches), dtype=np.int64, count=len(batches))
            owner = np.zeros(len(batches), dtype=np.int64)
            for r, p in enumerate(lpt_partition(lens.tolist(), world)):
                owner[p] = r
            n0 = len(batches)
            ids_end = 3 + 2 * n0 + int(lens.sum())
            seed_words = None if seeds is None else self._encode_seeds(seeds, n0)
            cfg_end = ids_end + (4 * n0 if configs is not None else 0)
            total = cfg_end + (0 if seed_words is None else seed_words.size)
            if self._host.numel() < total:
                self._host = torch.empty(int(total * 1.5), dtype=torch.int64, pin_memory=self._host.is_pinned())
            h = self._host.numpy()
            h[0], h[1], h[2] = n0, total, (configs is not None) | (2 if seed_words is not None else 0)
            h[3:3 + n0] = lens
            h[3 + n0:3 + 2 * n0] = owner
            np.concatenate([np.asarray(b, dtype=np.int64) for b in batches], out=h[3 + 2 * n0:ids_end])
            if configs is not None:
                h[ids_end:cfg_end] = self._encode_configs(configs)
            if seed_words is not None:
                h[cfg_end:total] = seed_words
            self._payload.copy_(self._host[:fb], non_blocking=True)
        dist.broadcast(self._payload, 0, group=self.group)
        if rank != 0:
            self._host[:fb].copy_(self._payload, non_blocking=True)
            if dev.type == "cuda":
                torch.cuda.current_stream().synchronize()
            total = int(self._host[1])
        if total > fb:                                   # rare: more than one block of ids
            total_t = total
            if self._big is None or self._big.numel() < total_t - fb:
                self._big = torch.empty(int((total_t - fb) * 1.5), dtype=torch.int64, device=dev)
            rest = self._big[:total_t - fb]
            if rank == 0:
                rest.copy_(self._host[fb:total_t])
            dist.broadcast(rest, 0, group=self.group)
            if rank != 0:
                if self._host.numel() < total_t:
                    nh = torch.empty(int(total_t * 1.5), dtype=torch.int64, pin_memory=self._host.is_pinned())
                    nh[:fb] = self._host[:fb]
                    self._host = nh
                self._host[fb:total_t].copy_(rest)
                if dev.type == "cuda":
                    torch.cuda.current_stream().synchronize()
        flat = self._host.numpy()
        n = int(flat[0])
        lens, owner = flat[3:3 + n], flat[3 + n:3 + 2 * n].copy()
        offs = 3 + 2 * n + np.concatenate([[0], np.cumsum(lens)])
        mine = np.nonzero(owner == rank)[0]
        my_cfgs = my_seeds = None
        end = offs[-1]
        if flat[2] & 1:
            words = flat[end:end + 4 * n].reshape(n, 4)
            my_cfgs = self._decode_configs(words[mine])
            end += 4 * n
        if flat[2] & 2:
            my_seeds = self._decode_seeds(flat[end:end + 2 * n].reshape(n, 2)[mine])
        return n, owner, mine, [flat[offs[i]:offs[i + 1]].copy() for i in mine], my_cfgs, my_seeds

    def synthesize(self, batches: Optional[Sequence[np.ndarray]], device_only: bool = False,
                   configs: Optional[Sequence] = None, seeds: Optional[Sequence] = None):
        """Collective.  Rank 0 passes every utterance's ids and gets the waveforms back in utterance order (views into
        the shared segment, valid until the next call); the other ranks pass None and get None.
        `device_only`: stop after the passes (results stay in each GPU's memory): the device-resident timing of bench.py.
        `configs` (rank 0): one PiperSynthesisConfig per utterance; they travel with the ids and each rank runs its
        shard with its utterances' configs.  None: the voice's fallback config everywhere.
        `seeds` (rank 0): one noise seed (int in [0, 2**64) or None) per utterance, as for
        VitsModel.infer_batch_with_values; a seeded utterance's samples do not depend on the rank or shard it lands on."""
        rank, world = dist.get_rank(self.group), dist.get_world_size(self.group)
        dev = _dev(self.group)
        if rank == 0 and configs is not None and len(configs) != len(batches):
            from .core import OperationError
            raise OperationError(f"Invalid configuration for Vits Model: {len(configs)} configs for {len(batches)} utterances")
        if rank == 0 and seeds is not None:
            from .piper import _seed_arrays
            _seed_arrays(seeds, len(batches))           # argument errors before any collective
        n, owner, mine, my_ids, my_cfgs, my_seeds = self._bcast_ids(batches, configs, seeds)
        extra = {} if my_cfgs is None else {"configs": my_cfgs}
        if my_seeds is not None:
            extra["seeds"] = my_seeds
        bps = 2 if self.pcm16 else 4
        fmt = 1 if self.pcm16 else 0
        # two-step because the layout of the segment depends on every rank's frame counts: run first (waveforms stay on
        # the device), exchange the counts, then copy out.  The job stays alive in between.
        job = None
        if self.run_local is None and self.model is not None:
            from .job import SynthesisJob
            samples_local = []
            if my_ids:
                job = SynthesisJob(self.model, my_ids, configs=my_cfgs, seeds=my_seeds)
                self.last_device_ms = job.run()
                samples_local = job.lengths()[1]
                if self.collect_profile:
                    self.last_profile = job.profile()
        else:
            samples_local = self.run_local(my_ids, None, 0, fmt, **extra) if my_ids else []
        if self._lens is None or self._lens.numel() < n:
            cap = max(n, 1024)
            self._lens = torch.zeros(cap, dtype=torch.int64, device=dev)
            self._lens_h = torch.zeros(cap, dtype=torch.int64, pin_memory=dev.type == "cuda")
        lh = self._lens_h.numpy()
        lh[:n] = 0
        if len(mine):
            lh[mine] = np.asarray(samples_local, dtype=np.int64)
        lens_t = self._lens[:n]
        lens_t.copy_(self._lens_h[:n], non_blocking=True)
        dist.all_reduce(lens_t, group=self.group)
        self._lens_h[:n].copy_(lens_t, non_blocking=True)
        if dev.type == "cuda":
            torch.cuda.current_stream().synchronize()
        samples = lh[:n].copy()
        self.last_table = (owner, samples)
        if device_only:
            if job is not None:
                job.close()
            return None
        order = [i for r in range(world) for i in np.nonzero(owner == r)[0]]      # rank-major: a rank's slice is contiguous
        offs = np.zeros(n, dtype=np.int64)
        pos = 0
        for i in order:
            offs[i] = pos
            pos += int(samples[i]) * bps
        self.seg.ensure(max(pos, 1))
        my_bytes = int(samples[mine].sum()) * bps if len(mine) else 0
        if my_bytes:
            start = int(offs[mine[0]])
            if job is not None:
                job.copy_out(self.seg.address + start, my_bytes, fmt)
            else:
                self.run_local(my_ids, self.seg.view(start, my_bytes, np.int16 if self.pcm16 else np.float32), my_bytes, fmt,
                               **extra)
        if job is not None:
            job.close()
        dist.barrier(group=self.group)
        if rank != 0:
            return None
        dt = np.int16 if self.pcm16 else np.float32
        return [self.seg.view(int(offs[i]), int(samples[i]) * bps, dt) for i in range(n)]

    def close(self):
        self.seg.close()


def sharded_synthesize(batches: Optional[Sequence[np.ndarray]], synth: Callable[[List[np.ndarray]], List[np.ndarray]],
                       group=None) -> Optional[List[np.ndarray]]:
    """scatter -> local synthesis (`synth`: list of id arrays -> list of float32 waveforms) -> gather."""
    mine = scatter_ids(batches, group)
    waves = synth(mine) if mine else []
    dev = _dev(group)
    if waves:
        local = torch.from_numpy(np.concatenate(waves)).to(dev)
    else:
        local = torch.zeros(0, dtype=torch.float32, device=dev)
    return gather_waveforms(local, [len(w) for w in waves], group)

