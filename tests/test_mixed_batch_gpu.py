"""GPU (-m gpu): one batch whose utterances have different speakers and synthesis scales.

Every utterance of a mixed batch must come out bit for bit as the same utterance run alone with its config as the
voice's fallback config (noise injected, so the Philox draws' batch position plays no part); uniform configs must give
the bits of a job that never set any; and a mixed batch must match the oracle run per utterance with its own sid and
scales."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import sonata_b200
from oracle import vits_oracle as vo
from sonata_b200 import PiperSynthesisConfig, OperationError, voicegen, workload
from sonata_b200.job import SynthesisJob

pytestmark = pytest.mark.gpu

LENS = [1, 7, 64, 65, 130, 513, 33, 200, 2, 97, 300, 16]
SPEAKERS = [0, 3, 1, 3, None, 2, 0, None, 1, 2, 3, 0]
LENGTH_SCALES = (0.7, 1.0, 1.3)
NOISE_W = (0.0, 0.8)
NOISE_SCALES = (0.0, 0.667)
CAPTURES = ("logw", "z_p", "z")


def _ids(n, utt):
    return workload.synthetic_ids(n // 2 + 1, utt=utt)[:n]


def _configs(n_speakers):
    out = []
    for b in range(len(LENS)):
        s = SPEAKERS[b]
        spk = None if (s is None or n_speakers <= 1) else s % n_speakers
        out.append(PiperSynthesisConfig(spk, NOISE_SCALES[(b // 2) % 2], LENGTH_SCALES[b % 3], NOISE_W[b % 2]))
    return out


@pytest.fixture(scope="module")
def voices(lib_built):
    d = voicegen.default_voice_dir()
    paths = {"medium4": voicegen.write_voice(d, "medium", n_speakers=4),
             "high3": voicegen.write_voice(d, "high", n_speakers=3),
             "x_low3": voicegen.write_voice(d, "x_low", n_speakers=3),
             "medium": voicegen.write_voice(d, "medium")}
    ms = {}

    def get(name):
        if name not in ms:
            ms[name] = sonata_b200.from_config_path(paths[name], device=0)
        return ms[name]
    get.paths = paths
    yield get
    for m in ms.values():
        m.close()


def _results(job, b):
    r = {"wav": job.fetch()[b].samples.as_slice().copy(), "cum": job.durations(b)}
    for name in CAPTURES:
        r[name] = job.debug_fetch(name, b)
    return r


QUALITY = {"medium4": "medium", "high3": "high", "x_low3": "x_low", "medium": "medium"}


def _noise(m, quality, batches, configs, seed=7):
    """eps_w per utterance; eps_z sized from a first pass (frame counts do not depend on noise_scale)."""
    rng = np.random.default_rng(seed)
    eps_w = [rng.standard_normal((len(ids), 2)).astype(np.float32) for ids in batches]
    job = SynthesisJob(m, batches, eps_w, None, configs=configs)
    job.run()
    frames = job.lengths()[0]
    job.close()
    inter = voicegen.ARCH[quality]["inter"]
    eps_z = [rng.standard_normal((f, inter)).astype(np.float32) for f in frames]
    return eps_w, eps_z


def _set_fallback(m, cfg):
    """The fallback config a single-utterance call needs to match `cfg` inside a batch: setting a fallback without a
    speaker keeps the previous speaker (piper/src/lib.rs:215-231), while a batch entry without one means speaker 0."""
    if cfg.speaker is None and m.get_speakers():
        cfg = PiperSynthesisConfig(0, cfg.noise_scale, cfg.length_scale, cfg.noise_w)
    m.set_fallback_synthesis_config(cfg)


def _alone(m, ids, cfg, ew, ez):
    _set_fallback(m, cfg)
    job = SynthesisJob(m, [ids], [ew], [ez], debug=True)
    job.run()
    r = _results(job, 0)
    r["i16"] = job.fetch_i16()[0]
    job.close()
    return r


def _check_mixed_equals_alone(m, quality, n_speakers):
    batches = [_ids(n, 40 + i) for i, n in enumerate(LENS)]
    configs = _configs(n_speakers)
    saved = m.get_fallback_synthesis_config()
    eps_w, eps_z = _noise(m, quality, batches, configs)
    job = SynthesisJob(m, batches, eps_w, eps_z, debug=True, configs=configs)
    job.run()
    i16 = job.fetch_i16()
    try:
        for b, ids in enumerate(batches):
            got = _results(job, b)
            ref = _alone(m, ids, configs[b], eps_w[b], eps_z[b])
            for k in ("wav", "cum") + CAPTURES:
                assert got[k].shape == ref[k].shape and np.array_equal(got[k], ref[k]), (b, k, configs[b])
            assert np.array_equal(i16[b], ref["i16"]), (b, "i16")
    finally:
        job.close()
        m.set_fallback_synthesis_config(saved)
    # the speakers are really different (a mixed batch is not quietly one speaker)
    if n_speakers > 1:
        ids = batches[6]
        outs = []
        for s in (0, 1):
            cfg = PiperSynthesisConfig(s, 0.0, 1.0, 0.0)
            outs.append(m.infer_batch_with_values([ids], [cfg])[0].samples.as_slice().copy())
        assert outs[0].shape != outs[1].shape or float(np.abs(outs[0] - outs[1]).max()) > 1e-3


@pytest.mark.parametrize("voice,backend", [("medium4", 1), ("medium4", 0), ("medium4", 2), ("high3", 1), ("high3", 0),
                                           ("x_low3", 1), ("x_low3", 0)])
def test_mixed_batch_equals_each_utterance_alone(voices, voice, backend):
    m = voices(voice)
    m.set_backend(backend)
    try:
        _check_mixed_equals_alone(m, QUALITY[voice], int(voice[-1]))
    finally:
        m.set_backend(1)


@pytest.mark.parametrize("voice", ["medium4", "medium"])
def test_uniform_configs_give_todays_bits(voices, voice):
    """set_configs with the fallback config for everyone == never calling it == NULL; on a single-speaker voice only the
    scales can vary."""
    m = voices(voice)
    batches = [_ids(n, 70 + i) for i, n in enumerate(LENS[:6])]
    fb = PiperSynthesisConfig(2 if voice == "medium4" else None, 0.667, 1.1, 0.8)
    m.set_fallback_synthesis_config(fb)
    # Philox draws depend on the call, so the three runs share injected noise
    eps_w, eps_z = _noise(m, QUALITY[voice], batches, [fb] * len(batches), seed=3)
    runs = []
    for how in ("none", "all", "null"):
        job = SynthesisJob(m, batches, eps_w, eps_z, debug=True)
        if how == "all":
            job.set_configs([fb] * len(batches))
        elif how == "null":
            job.set_configs([PiperSynthesisConfig(None, 0.0, 1.0, 0.0)] * len(batches))
            job.set_configs(None)
        job.run()
        runs.append([_results(job, b) for b in range(len(batches))])
        job.close()
    for r in runs[1:]:
        for b in range(len(batches)):
            for k in runs[0][b]:
                assert np.array_equal(r[b][k], runs[0][b][k]), (voice, b, k)
    # single-speaker voice: mixed scales against each utterance alone (Philox noise off: deterministic scales only
    # differ in length_scale; noise_w / noise_scale vary with injected eps_w)
    if voice == "medium":
        cfgs = [PiperSynthesisConfig(None, 0.0, LENGTH_SCALES[b % 3], NOISE_W[b % 2]) for b in range(len(batches))]
        job = SynthesisJob(m, batches, eps_w, None, debug=True, configs=cfgs)
        job.run()
        for b, ids in enumerate(batches):
            _set_fallback(m, cfgs[b])
            alone = SynthesisJob(m, [ids], [eps_w[b]], None, debug=True)
            alone.run()
            assert np.array_equal(_results(job, b)["wav"], _results(alone, 0)["wav"]), b
            alone.close()
        job.close()
    m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.667, 1.0, 0.8))


# (utterance seed, oracle frames) per utterance: every duration >= 1e-3 from the ceil() cliff in the fp32 oracle and its
# fp64 shadow under that utterance's own speaker, scales and eps_w (screened like tests/screen_margin.py)
ORACLE_CASE = [  # phonemes, speaker, length_scale, noise_w, noise_scale, seed, frames
    (14, 3, 0.8, 0.8, 0.667, 100, 83), (30, 0, 1.0, 0.0, 0.667, 110, 225), (9, None, 1.25, 0.8, 0.0, 120, 84),
    (41, 1, 1.0, 0.8, 0.667, 130, 281), (22, 3, 0.8, 0.0, 0.0, 140, 138), (17, 2, 1.25, 0.8, 0.667, 150, 155)]
MARGIN = 1e-3


@pytest.mark.parametrize("backend", [1, 0])
def test_mixed_batch_against_oracle(voices, backend):
    from test_gpu_parity import TOL_LOGW_MAX, TOL_STAGE, TOL_WAV
    m = voices("medium4")
    m.set_backend(backend)
    W = vo.to_torch(voicegen.make_tensors("medium", n_speakers=4))
    a = vo.arch_of(W)
    batches, configs, eps_w, eps_z, refs = [], [], [], [], []
    for b, (n, spk, ls, nw, nsc, seed, frames) in enumerate(ORACLE_CASE):
        ids = vo.synthetic_ids(n, utt=seed)
        ew = np.random.default_rng(500 + b).standard_normal((len(ids), 2)).astype(np.float32)
        ez = torch.randn(1, a["inter"], frames, generator=torch.Generator().manual_seed(900 + b))
        st = {}
        vo.infer(W, ids, [nsc, ls, nw], eps_w=torch.from_numpy(ew.T.copy()).view(1, 2, -1), eps_z=ez, stages=st, sid=spk)
        w = st["w"].view(-1).double()
        fr = w - torch.floor(w)
        assert float(torch.minimum(fr, 1 - fr).min()) >= MARGIN and st["y_len"] == frames, ("screening is stale", b)
        batches.append(ids); configs.append(PiperSynthesisConfig(spk, nsc, ls, nw)); refs.append(st)
        eps_w.append(ew); eps_z.append(ez[0].T.contiguous().numpy())
    job = SynthesisJob(m, batches, eps_w, eps_z, debug=True, configs=configs)
    job.run()
    frames_got = job.lengths()[0]
    wavs = job.fetch()
    tm = lambda t: t[0].T.numpy()
    try:
        for b, st in enumerate(refs):
            ref_cum = np.cumsum(st["w_ceil"].view(-1).numpy()).astype(np.int64)
            assert np.array_equal(job.durations(b).astype(np.int64), ref_cum) and frames_got[b] == st["y_len"], b
            pairs = [("x", job.debug_fetch("x", b), tm(st["x"]), TOL_STAGE),
                     ("stats", job.debug_fetch("stats", b), np.concatenate([tm(st["m_p"]), tm(st["logs_p"])], 1), TOL_STAGE),
                     ("logw", job.debug_fetch("logw", b), tm(st["logw"]), TOL_LOGW_MAX),
                     ("z_p", job.debug_fetch("z_p", b), tm(st["z_p"]), TOL_STAGE),
                     ("z", job.debug_fetch("z", b), tm(st["z"]), TOL_STAGE),
                     ("dec.pre", job.debug_fetch("dec.pre", b), tm(st["dec.pre"]), TOL_STAGE)]
            for i in range(len(a["up_rates"])):
                pairs.append((f"dec.mrf{i}", job.debug_fetch(f"dec.mrf{i}", b), tm(st[f"dec.mrf{i}"]), TOL_STAGE))
            pairs.append(("wav", wavs[b].samples.as_slice(), st["wav"].view(-1).numpy(), TOL_WAV))
            for name, got, ref, tol in pairs:
                assert got.shape == ref.shape, (b, name)
                err = float(np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64)).max())
                assert err < tol, (b, name, err)
    finally:
        job.close()
        m.set_backend(1)


def test_bad_configs_raise_and_leave_the_job_as_it_was(voices):
    m = voices("medium4")
    batches = [_ids(n, 90 + i) for i, n in enumerate((20, 31, 12))]
    good = [PiperSynthesisConfig(1, 0.0, 1.0, 0.0), PiperSynthesisConfig(3, 0.0, 0.9, 0.0),
            PiperSynthesisConfig(None, 0.0, 1.2, 0.0)]
    job = SynthesisJob(m, batches, configs=good)
    job.run()
    before = [a.samples.as_slice().copy() for a in job.fetch()]
    with pytest.raises(OperationError, match="utterance 2"):
        job.set_configs(good[:2] + [PiperSynthesisConfig(4, 0.0, 1.0, 0.0)])
    with pytest.raises(OperationError):
        job.set_configs(good[:2])
    job.run()
    after = [a.samples.as_slice().copy() for a in job.fetch()]
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
    job.close()
    with pytest.raises(OperationError, match="utterance 1"):
        m.infer_batch_with_values(batches[:2], [good[0], PiperSynthesisConfig(7, 0.0, 1.0, 0.0)])
    single = voices("medium")
    single.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.0, 1.0, 0.0))
    job = SynthesisJob(single, batches[:1])
    job.run()
    before = job.fetch()[0].samples.as_slice().copy()
    with pytest.raises(OperationError, match="utterance 0"):
        job.set_configs([PiperSynthesisConfig(0, 0.0, 1.0, 0.0)])
    job.run()
    assert np.array_equal(job.fetch()[0].samples.as_slice(), before)
    job.close()


def test_streaming_decoder_runs_on_the_one_slot_path(voices):
    """encode + ONE decode_chunk over the whole latent == a job of that utterance with speaker 3 (chunks with overlap
    see different zero padding at their edges, so only the whole-latent chunk is compared bit for bit)."""
    m = voices("medium4")
    ids = _ids(57, 5)
    cfg = PiperSynthesisConfig(3, 0.0, 1.0, 0.0)
    m.set_fallback_synthesis_config(cfg)
    try:
        job = SynthesisJob(m, [ids])
        job.run()
        ref = job.fetch()[0].samples.as_slice().copy()
        job.close()
        sm = sonata_b200.VitsStreamingModel(voices.paths["medium4"], device=0)
        sm.set_fallback_synthesis_config(cfg)
        enc = sm.infer_encoder(ids)
        got = enc.infer_decoder(0, enc.num_frames).as_slice()
        assert got.shape == ref.shape and np.array_equal(got, ref)
        del enc
        sm.close()
    finally:
        m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.667, 1.0, 0.8))


def test_frontend_world1_carries_configs(voices):
    """shard.Frontend on one rank (gloo, the GPU pass behind it): per-utterance configs give the alone results."""
    import socket
    import torch.distributed as dist
    from sonata_b200 import shard
    m = voices("medium4")
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        batches = [_ids(n, 120 + i) for i, n in enumerate((25, 60, 9, 140))]
        cfgs = [PiperSynthesisConfig(s, 0.0, ls, 0.0) for s, ls in ((3, 1.0), (None, 0.8), (1, 1.3), (2, 1.0))]
        fe = shard.Frontend(model=m, pin=False)
        out = fe.synthesize(batches, configs=cfgs)
        for ids, cfg, o in zip(batches, cfgs, out):
            _set_fallback(m, cfg)
            ref = m.infer_with_values(ids).samples.as_slice()
            assert o.shape == ref.shape and np.array_equal(o, ref)
        del out
        fe.close()
    finally:
        dist.destroy_process_group()
        m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.667, 1.0, 0.8))
