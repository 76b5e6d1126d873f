"""CPU: the float64 text-encoder restatement (tests/enc_reference.py) against the oracle, its torch emulations against the
numpy models they restate, and its bounds against emulated kernel mistakes on real voice stages."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import att_reference as ar  # noqa: E402
import enc_reference as er  # noqa: E402
from oracle import vits_oracle as vo  # noqa: E402
from sonata_b200 import voicegen, workload  # noqa: E402

_T = {}


def _tensors(q):
    if q not in _T:
        _T[q] = voicegen.make_tensors(q)
    return _T[q]


def _ids(n, utt):
    return workload.synthetic_ids(n // 2 + 1, utt=utt)[:n]


def test_emulations_match_the_numpy_models():
    """enc_reference's torch emulate / fma_chain / simt_pv agree bit for bit with tools/emu_tc_accuracy.emulate /
    fp32_fma and att_reference.simt_pv (the models the bounds are stated in)."""
    import emu_tc_accuracy as emu
    rng = np.random.default_rng(5)
    x = rng.standard_normal((45, 192)).astype(np.float32)
    w = (rng.standard_normal((192, 40)) / 14).astype(np.float32)
    xt, wt = torch.from_numpy(x), torch.from_numpy(w)
    for chunk in (8, 12, 0):
        for prods in (("hh", "lh", "hl"), ("hh",), ("hh", "lh")):
            a = er.emulate(xt, wt, chunk, prods).numpy()
            b = emu.emulate(x, w, "tf32", "rz", chunk, prods)
            assert np.array_equal(a, b), (chunk, prods, float(np.abs(a - b).max()))
    assert np.array_equal(er.fma_chain(xt, wt).numpy(), emu.fp32_fma(x, w))
    p = rng.random((37, 70)).astype(np.float32)
    v = rng.standard_normal((70, 48)).astype(np.float32)
    assert np.array_equal(er.simt_pv(torch.from_numpy(p), torch.from_numpy(v)).numpy(), ar.simt_pv(p, v))


@pytest.mark.parametrize("quality", ["medium", "high", "x_low"])
@pytest.mark.parametrize("n", [7, 150])
def test_reference_matches_oracle(quality, n):
    """The chain from the ids in float64 matches the oracle's text_encoder run in float64 within 1e-9 (relative to the
    stage's max |ref|) at enc.emb, every layer's output, m_p and logs_p; the float32 chain (the backend-0 yardstick)
    matches the float32 oracle within float32 error."""
    t = _tensors(quality)
    a = er.arch(t)
    ids = _ids(n, 70 + n)
    I = a["inter"]
    for dt, mode, tol in ((torch.float64, "f64", 1e-9), (torch.float32, "f32", 2e-5)):
        W = vo.to_torch(t, dtype=dt)
        st = {}
        x, m_p, logs_p = vo.text_encoder(W, torch.as_tensor(np.asarray(ids))[None], vo.arch_of(W), stages=st)
        res = er.run_chain(t, ids, er.Arith(mode))
        tm = lambda v: v[0].T.double().numpy()
        pairs = [("enc.emb", st["enc.emb"])] + [(f"enc.{i}.ln2", st[f"enc.layer{i}"]) for i in range(a["layers"])]
        pairs += [("m_p", m_p), ("logs_p", logs_p)]
        for name, ref in pairs:
            got = res["stats"][:, :I] if name == "m_p" else res["stats"][:, I:] if name == "logs_p" else res[name]
            got, ref = er._np(got), tm(ref)
            assert got.shape == ref.shape, (name, got.shape, ref.shape)
            e = float(np.abs(got - ref).max()) / float(np.abs(ref).max())
            assert e < tol, (quality, n, mode, name, e)


# --------------------------------------------------------------------------- bounds against emulated mistakes
CATCH = 3.0             # every emulated mistake lands at least this far above its bound
LAYER = 2               # a middle layer: its attention sees post-LayerNorm inputs
_CHAINS = {}


def _chain(quality, n, utt):
    key = (quality, n, utt)
    if key not in _CHAINS:
        _CHAINS[key] = er.run_chain(_tensors(quality), _ids(n, utt), er.Arith("f64"))
    return _CHAINS[key]


def _stage(t, name):
    return next(s for s in er.stages(t) if s[0] == name)


def _ratio(t, caps, name, mutated, backends=(1, 0)):
    """Smallest ratio, over the backends' bounds, of the mutated stage's error to the bound of stage `name`."""
    _, src, kind, fn = _stage(t, name)
    x = er.inputs(src, caps)
    ref = fn(x, er.Arith("f64"))
    got = fn(x, mutated)
    rs = []
    for be in backends:
        yard = fn(x, er.Arith("emu" if (kind == "conv" and be == 1) else "f32"))
        rs.append(er.stage_check(kind, got, ref, yard, be)[2])
    return min(rs)


# (stage, mutated arithmetic, backends whose bound must catch it); stages of layer LAYER of the medium voice.
# Not here: a LayerNorm taking the variance in one pass, E[x^2] - mean^2 in fp32 (Arith ln_var="onepass").  The
# encoder's LayerNorm inputs have means small beside their spread, so the cancellation costs little: it lands at 0.2x
# the LN bound, inside it, and no bound that the two-pass kernel passes with 2x margin could catch it.
MISTAKES = {
    "conv_tf one TF32 product": (f"enc.{LAYER}.ffn2", er.Arith("emu", products=("hh",)), (1,)),
    "conv_tf two of three split products": (f"enc.{LAYER}.ffn2", er.Arith("emu", products=("hh", "lh")), (1,)),
    "conv_tf without the chunk flush": (f"enc.{LAYER}.ffn2", er.Arith("emu", no_flush=True), (1,)),
    "FFN padding left 0, right 2": (f"enc.{LAYER}.ffn1", er.Arith("f64", ffn_pad=(0, 2)), (1, 0)),
    "LayerNorm eps 1e-6": (f"enc.{LAYER}.ln1", er.Arith("f32", ln_eps=1e-6), (1,)),
    "LayerNorm unbiased variance": (f"enc.{LAYER}.ln2", er.Arith("f32", ln_var="unbiased"), (1,)),
    "relative window 3": (f"enc.{LAYER}.att", er.Arith("f64", window=3), (1,)),
    "emb_rel_v band term dropped on the last row": (f"enc.{LAYER}.att", er.Arith("f64", drop_relv_last=True), (1,)),
    "zero-filled keys inside the softmax sum": (f"enc.{LAYER}.att", er.Arith("f64", zero_keys=True), (1,)),
    "layer l with layer l-1's relative embeddings": (f"enc.{LAYER}.att", er.Arith("f64", rel_layer=LAYER - 1), (1,)),
    "stats halves swapped": ("stats", er.Arith("f64", swap_stats=True), (1, 0)),
}


@pytest.mark.parametrize("mistake", list(MISTAKES))
def test_bounds_catch_emulated_mistakes(mistake):
    """Each plausible kernel mistake, emulated on the host on a real medium-voice stage (the float64 chain of a 45-id
    utterance standing in for the captures), lands at least CATCH times above the stage's bound."""
    t = _tensors("medium")
    name, mutated, backends = MISTAKES[mistake]
    r = _ratio(t, _chain("medium", 45, 9), name, mutated, backends)
    print(f"{mistake:48s} {name:14s} {r:10.1f}x the bound")
    assert r >= CATCH, (mistake, r)


@pytest.mark.parametrize("stage", ["ffn1", "ffn2"])
def test_bounds_catch_a_neighbour_row_at_the_segment_edge(stage):
    """The k = 3 FFN conv reading the neighbouring utterance's edge row instead of the zero gap row, at either end."""
    t = _tensors("medium")
    caps, other = _chain("medium", 45, 9), _chain("medium", 30, 11)
    _, src, _, _ = _stage(t, f"enc.{LAYER}.{stage}")
    nb = er._np(other[src])
    zero = np.zeros(nb.shape[1])
    for edge in ((nb[-1], zero), (zero, nb[0])):
        r = _ratio(t, caps, f"enc.{LAYER}.{stage}", er.Arith("f64", edge_rows=edge))
        print(f"neighbour row {stage} {'before' if edge[1] is zero else 'after':6s} {r:10.1f}x the bound")
        assert r >= CATCH, (stage, r)
