"""GPU (-m gpu): which attention kernel an utterance runs on, and that the choice never depends on its batch.

On the default backend an utterance of at most 1280 ids (96- or 48-wide heads, SB200_ATT_SIMT unset) runs its attention
on the tensor cores: two 3xTF32 grouped GEMMs around attn_softmax_kernel.  Every other utterance runs on the fp32
CUDA-core attention_kernel.  The route is the utterance's own, so a batch whose utterances lie on both sides of 1280
ids runs both kernels in every layer, and each utterance gets the bits it gets alone (DESIGN.md section 4).

* A mixed batch, in both orders, against each utterance alone, bit for bit: every layer's attention, x, stats, logw,
  the durations, z and the waveform, on the medium voice, x_low (48-wide heads) and the 4-speaker medium voice with
  the speakers mixed.  Also on backend 0 and with SB200_ATT_SIMT=1, where every utterance is on attention_kernel and
  the launch is sized by the batch's longest utterance (its shared-memory row width and its grid).
* The same through infer_batch_with_values, infer_encoder_batch and StreamBatch.
* attention_kernel's length limit per head width: the longest utterance it takes runs and is held to float64; one
  more id is refused when the job is created, alone or in a batch, with an error that names the utterance.
* The enc region launches what it launched before the route became per utterance: 3 attention launches per layer on
  the tensor cores, 1 on attention_kernel, 4 when the batch has both routes."""
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import att_reference as ar  # noqa: E402
import sonata_b200  # noqa: E402
from sonata_b200 import (PiperSynthesisConfig, SpeechStreamer, StreamBatch, VitsStreamingModel, voicegen,  # noqa: E402
                         workload)
from sonata_b200.job import SynthesisJob  # noqa: E402

pytestmark = pytest.mark.gpu

TC_MAX = 1280                     # the longest utterance the tensor-core attention takes (softmax rows in registers)
# Lengths on both sides of TC_MAX and far from it; 2000 ids sizes the fp32 launch past every other utterance.
MIXED = (33, 1281, 1, 640, 1280, 2000, 257)
# name -> (backend, SB200_ATT_SIMT set)
CONFIGS = {"b1": (1, False), "b1_fp32att": (1, True), "b0": (0, False)}
# name -> (voicegen quality, speakers)
VOICES = {"medium": ("medium", 1), "x_low": ("x_low", 1), "medium4": ("medium", 4)}


@pytest.fixture(scope="module")
def voices(lib_built):
    d = voicegen.default_voice_dir()
    paths = {name: voicegen.write_voice(d, q, n_speakers=n) if n > 1 else voicegen.write_voice(d, q)
             for name, (q, n) in VOICES.items()}
    ms = {}

    def get(name, streaming=False):
        key = (name, streaming)
        if key not in ms:
            ms[key] = (VitsStreamingModel(paths[name], device=0) if streaming
                       else sonata_b200.from_config_path(paths[name], device=0))
        return ms[key]
    yield get
    for m in ms.values():
        m.close()


def _ids(n, utt):
    return [int(i) for i in workload.synthetic_ids(n // 2 + 1, utt=utt)[:n]]


def _cfg(speaker):
    return PiperSynthesisConfig(speaker, 0.0, 1.0, 0.0)


def _route(backend, simt, monkeypatch):
    if simt:
        monkeypatch.setenv("SB200_ATT_SIMT", "1")
    else:
        monkeypatch.delenv("SB200_ATT_SIMT", raising=False)


def _frames(cum):
    return np.diff(np.concatenate([[0], np.asarray(cum, dtype=np.int64)]))


def _results(m, batch, cfgs, layers):
    """Per utterance of one debug job: every enc.{l}.att, x, stats, logw, durations, z and the waveform."""
    job = SynthesisJob(m, batch, debug=True, configs=cfgs)
    try:
        job.run()
        wav = [a.samples.as_slice().copy() for a in job.fetch()]
        out = []
        for b in range(len(batch)):
            r = {f"enc.{l}.att": job.debug_fetch(f"enc.{l}.att", b) for l in range(layers)}
            r.update({k: job.debug_fetch(k, b) for k in ("x", "stats", "logw", "z")})
            r["durations"], r["wav"] = job.durations(b), wav[b]
            out.append(r)
        return out
    finally:
        job.close()


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("voice", list(VOICES))
def test_mixed_batch_equals_each_alone(voices, voice, config, monkeypatch):
    """MIXED and MIXED reversed as one job each, against every utterance alone: every compared output bit for bit.
    Alone, an utterance of at most 1280 ids runs on the tensor cores (backend 1) and the others on attention_kernel
    with a launch sized by themselves; in the batch the same holds per utterance."""
    m = voices(voice)
    backend, simt = CONFIGS[config]
    n_spk = VOICES[voice][1]
    layers = voicegen.ARCH[VOICES[voice][0]]["layers"]
    ids = [_ids(n, 700 + i) for i, n in enumerate(MIXED)]
    cfgs = [_cfg(i % n_spk if n_spk > 1 else None) for i in range(len(MIXED))]
    _route(backend, simt, monkeypatch)
    m.set_backend(backend)
    try:
        alone = [_results(m, [ids[b]], [cfgs[b]], layers)[0] for b in range(len(ids))]
        for order in (list(range(len(ids))), list(reversed(range(len(ids))))):
            got = _results(m, [ids[b] for b in order], [cfgs[b] for b in order], layers)
            for g, b in zip(got, order):
                for k, want in alone[b].items():
                    assert g[k].shape == want.shape, (voice, config, MIXED[b], order[0], k, g[k].shape, want.shape)
                    assert np.array_equal(g[k], want), (voice, config, MIXED[b], order[0], k,
                                                        float(np.abs(g[k] - want).max()))
                assert (_frames(g["durations"]) >= 1).all() and np.isfinite(g["wav"]).all(), (voice, config, MIXED[b])
    finally:
        m.set_backend(1)
        monkeypatch.delenv("SB200_ATT_SIMT", raising=False)


def test_batched_entry_points_equal_each_alone(voices):
    """infer_batch_with_values, infer_encoder_batch (z through its whole decode, and p_duration) and a StreamBatch
    that admits a 1500-id stream in the same step as short ones, each against its one-utterance counterpart."""
    m = voices("medium")
    m.set_fallback_synthesis_config(_cfg(None))
    lens = (40, 1500, 7, 1280, 300)
    batch = [_ids(n, 760 + i) for i, n in enumerate(lens)]
    together = m.infer_batch_with_values(batch)
    for b, ids in enumerate(batch):
        alone = m.infer_with_values(ids).samples.as_slice()
        assert np.array_equal(together[b].samples.as_slice(), alone), ("infer_batch_with_values", lens[b])

    s = voices("medium", streaming=True)
    s.set_fallback_synthesis_config(_cfg(None))
    encs = s.infer_encoder_batch(batch)
    for b, ids in enumerate(batch):
        ref = s.infer_encoder(ids)
        assert encs[b].num_frames == ref.num_frames, ("infer_encoder_batch", lens[b])
        assert np.array_equal(encs[b].p_duration, ref.p_duration), ("infer_encoder_batch", lens[b])
        assert np.array_equal(encs[b].infer_decoder().as_slice(), ref.infer_decoder().as_slice()), lens[b]

    cs, pad = 150, 3
    sb = StreamBatch(s, cs, pad)
    keys = [sb.add(ids) for ids in batch]                        # one encoder pass for all five streams
    got = {k: [] for k in keys}
    while len(sb):
        for k, a in sb.step():
            got[k].append(a.as_slice().copy())
    for k, ids, n in zip(keys, batch, lens):
        exp = [a.as_slice().copy() for a in SpeechStreamer(s.infer_encoder(ids), cs, pad)]   # stream_synthesis
        assert len(got[k]) == len(exp) and all(np.array_equal(g, e) for g, e in zip(got[k], exp)), ("StreamBatch", n)
    assert len(got[keys[1]]) > 1                                  # the 1500-id stream is chunked, not one-shot


def _att_smem_bytes(T, D):
    """attention_kernel's dynamic shared memory (kernels_misc.cu attention_smem_bytes): 16 query rows of Q, of scores
    over tpad = round_up(T, 4) keys, of relative logits (32 wide) and the row sums, and four partial outputs."""
    tpad = (T + 3) // 4 * 4
    return 4 * (16 * D + 16 * tpad + 16 * 32 + 16 + 4 * 16 * D)


SMEM_LIMIT = 220 * 1024           # what job creation allows attention_kernel (engine.cu create_job)


@pytest.mark.parametrize("voice,limit", [("medium", 3004), ("x_low", 3244)])
def test_fp32_attention_length_limit(voices, voice, limit):
    """The longest utterance job creation accepts is the longest whose attention_kernel launch fits SMEM_LIMIT:
    4 (16 D + 16 round_up(T, 4) + 528 + 64 D) bytes <= 220 KB gives T <= 3004 for 96-wide heads (medium, high) and
    T <= 3244 for 48-wide heads (x_low).  That utterance runs: its layer-0 attention within fp32_att_bound of the
    float64 attention of the kernel's own Q / K / V, durations >= 1 and a finite waveform.  One more id is refused when
    the job is created, alone or in a batch, with an error naming the utterance's index and length; the voice's next
    job still runs."""
    m = voices(voice)
    m.set_fallback_synthesis_config(_cfg(None))
    a = voicegen.ARCH[voice]
    H, heads, D = a["hidden"], a["heads"], a["hidden"] // a["heads"]
    assert _att_smem_bytes(limit, D) <= SMEM_LIMIT < _att_smem_bytes(limit + 1, D)
    assert max(T for T in range(1, 4000) if _att_smem_bytes(T, D) <= SMEM_LIMIT) == limit

    ids = _ids(limit, 790)
    job = SynthesisJob(m, [ids], debug=True)
    try:
        job.run()
        qkv = job.debug_fetch("qkv0", 0)
        att = job.debug_fetch("att0", 0)
        with pytest.raises(sonata_b200.OperationError):
            job.debug_fetch("p0", 0)                               # a job wholly on attention_kernel has no p0
        frames = _frames(job.durations(0))
        wav = job.fetch()[0].samples.as_slice()
    finally:
        job.close()
    relk, relv = ar.rel_embeddings(voicegen.make_tensors(voice), 0)
    _, ref = ar.attention(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], relk, relv, heads)
    err, scale = float(np.abs(att - ref).max()), float(np.abs(ref).max())
    print(f"\n{voice} T={limit}: fp32 attention max|err| {err:.3g}, max|ref| {scale:.3g}, "
          f"{err / (2.0 ** -24 * scale):.1f} ulp of max|ref|, bound {ar.fp32_att_bound(limit, scale):.3g}")
    assert err <= ar.fp32_att_bound(limit, scale), (err, ar.fp32_att_bound(limit, scale))
    assert (frames >= 1).all() and len(frames) == limit
    assert wav.size == 256 * int(frames.sum()) and np.isfinite(wav).all()

    over = _ids(limit + 1, 791)
    for batch, b in (([over], 0), ([_ids(20, 792), over, _ids(5, 793)], 1)):
        with pytest.raises(sonata_b200.OperationError, match=rf"too long.*utterance {b}\D.*\b{limit + 1} ids"):
            SynthesisJob(m, batch)
    short = _ids(20, 792)
    assert np.array_equal(m.infer_with_values(short).samples.as_slice(),
                          m.infer_batch_with_values([short, ids])[0].samples.as_slice())


# Launches of the enc region on backend 1 before the route became per utterance, for a batch wholly on one side of
# 1280 ids: the embedding, per layer the q/k/v, o, ffn1 and ffn2 convs, two LayerNorms and the attention (3 launches on
# the tensor cores: two GEMMs and the softmax; 1 on attention_kernel), and the stats projection.
ENC_LAUNCHES = {"tc": 2 + 6 * (6 + 3), "fp32": 2 + 6 * (6 + 1)}


@pytest.mark.parametrize("voice", ["medium", "x_low"])
def test_attention_launches_per_layer(voices, voice):
    """A batch wholly at or below 1280 ids, or wholly above, launches what it launched before; a batch with both routes
    launches both attentions in every layer (4 per layer)."""
    m = voices(voice)
    m.set_fallback_synthesis_config(_cfg(None))
    layers = voicegen.ARCH[voice]["layers"]
    assert layers == 6
    want = {"tc": ENC_LAUNCHES["tc"], "fp32": ENC_LAUNCHES["fp32"], "mixed": 2 + layers * (6 + 4)}
    for name, lens in (("tc", (33, 1280, 1)), ("fp32", (1281, 2000)), ("mixed", (33, 2000, 1280))):
        job = SynthesisJob(m, [_ids(n, 800 + i) for i, n in enumerate(lens)])
        try:
            job.run()
            enc = {p["name"]: p for p in job.profile()}["enc"]
        finally:
            job.close()
        assert enc["launches"] == want[name], (voice, name, enc["launches"], want[name])


def test_refusal_names_the_utterance_in_every_entry_point(voices):
    """The length check runs when any job is created: a batch call and an encoder batch refuse an overlong utterance
    with the same error, and the voice runs its next job."""
    m = voices("medium")
    m.set_fallback_synthesis_config(_cfg(None))
    over = _ids(3005, 795)
    pat = re.compile(r"too long.*utterance 2\D.*\b3005 ids")
    with pytest.raises(sonata_b200.OperationError, match=pat):
        m.infer_batch_with_values([_ids(9, 796), _ids(4, 797), over])
    s = voices("medium", streaming=True)
    with pytest.raises(sonata_b200.OperationError, match=pat):
        s.infer_encoder_batch([_ids(9, 796), _ids(4, 797), over])
    assert m.infer_with_values(_ids(9, 796)).samples.as_slice().size > 0
