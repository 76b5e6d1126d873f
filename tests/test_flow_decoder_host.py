"""CPU: tests/dec_reference.py against the oracle's flow_reverse / decoder, and its bounds against plausible kernel
mistakes emulated on the host.  Runs without a device (the float64 reference moves to the GPU when one is present)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import dec_reference as dr  # noqa: E402
from oracle import vits_oracle as vo  # noqa: E402
from sonata_b200 import voicegen  # noqa: E402

# (quality, speakers, sid)
VOICES = {"medium": ("medium", 1, None), "high": ("high", 1, None), "x_low": ("x_low", 1, None),
          "medium_spk4_sid2": ("medium", 4, 2)}
_CACHE = {}


def _oracle(voice, n_ph=14, utt=5, dtype=torch.float32):
    """Tensors, sid and the oracle's stages (engine layout, float64 numpy) of one zero-noise utterance."""
    key = (voice, n_ph, utt, dtype)
    if key not in _CACHE:
        quality, nspk, sid = VOICES[voice]
        t = voicegen.make_tensors(quality, n_speakers=nspk)
        st = {}
        vo.infer(vo.to_torch(t, dtype=dtype), vo.synthetic_ids(n_ph, utt=utt), [0.0, 1.0, 0.0], stages=st, sid=sid)
        a = dr.arch(t)
        out = {}
        for name, v in st.items():
            if not torch.is_tensor(v) or v.dim() != 3:
                continue
            x = v[0].T.to(torch.float64).numpy()
            if name.startswith("flow."):            # after an odd number of couplings the engine keeps z reversed
                if (a["flow_n"] - int(name.split(".")[1])) % 2 == 1:
                    x = x[:, ::-1]
            out[name] = np.ascontiguousarray(x)
        out["wav"] = st["wav"][0].T.to(torch.float64).numpy()
        _CACHE[key] = (t, sid, out)
    return _CACHE[key]


@pytest.mark.parametrize("voice", list(VOICES))
def test_reference_matches_oracle(voice):
    """The float64 chain from the oracle's z_p matches the oracle run in float64 (to_torch(dtype=float64)) to 1e-9
    relative at every stage, and the fp32 oracle within fp32 error: 1e-4 of the stage's max |ref| (the oracle's fp32
    chain compounds; measured <= 2e-6).  Each stage from the fp32 oracle's own stage input agrees with it to 2e-6."""
    t, sid, o32 = _oracle(voice)
    _, _, o64 = _oracle(voice, dtype=torch.float64)
    ref = dr.run_chain(t, o64["z_p"], dr.Arith("f64"), sid)
    for name, _, _ in dr.stages(t, sid):
        r = dr._np(ref[name])
        scale = max(1.0, float(np.abs(r).max()))
        assert r.shape == o64[name].shape, (name, r.shape, o64[name].shape)
        e64 = float(np.abs(r - o64[name]).max())
        e32 = float(np.abs(r - o32[name]).max())
        assert e64 <= 1e-9 * scale, (voice, name, e64)
        assert e32 <= 1e-4 * scale, (voice, name, e32)
    for name, src, fn in dr.stages(t, sid):
        x = o32["z" if src == "z" else src]
        r = dr._np(fn(x, dr.Arith("f64")))
        assert np.abs(r - o32[name]).max() <= 2e-6 * max(1.0, float(np.abs(r).max())), (voice, name)


def _ratio(t, sid, stage, x, **mut):
    """Largest tile ratio of the mutated emulation's error to the stage's bound (tc_bound of the unmutated emulation)."""
    fn = {n: f for n, _, f in dr.stages(t, sid)}[stage]
    ref, emu = fn(x, dr.Arith("f64")), fn(x, dr.Arith("emu"))
    bad = fn(x, dr.Arith("emu", **mut))
    mult = dr.tc_mult(t, stage)
    assert dr.tc_check(emu, ref, emu, mult)[2] <= 1 / mult + 1e-12
    return dr.tc_check(bad, ref, emu, mult)[2]


@pytest.mark.parametrize("voice", ["medium", "high"])
def test_bound_catches_tc_mistakes(voice):
    """Each emulated mistake lands at least 3x above the bf16x2 bound on some tile of the stage it breaks, with the
    oracle's own stage inputs: a dropped hi*lo product in one conv of a ResBlock, bf16-only (no lo) input on each tile's
    halo rows, one ConvTranspose phase's taps shifted by a row, the MRF's 1/3 rounded to bf16."""
    t, sid, o = _oracle(voice)
    a = dr.arch(t)
    last = len(a["up_rates"]) - 1
    conv = "convs.1" if a["resblock"] == 2 else "convs2.1"
    ratios = {
        "drop_hilo": _ratio(t, sid, f"dec.mrf{last}", o[f"dec.up{last}"], drop_hilo=f"dec.resblocks.{3 * last + 1}.{conv}"),
        "halo_hi": _ratio(t, sid, "dec.mrf0", o["dec.up0"], halo_hi=True),
        "up_shift": _ratio(t, sid, "dec.up1", o["dec.mrf0"], up_shift=(1, 3)),
        "mrf_third_bf16": _ratio(t, sid, "dec.mrf1", o["dec.up1"], mrf_scale=float(torch.tensor(1 / 3).bfloat16())),
    }
    t, sid, o = _oracle(voice, n_ph=60, utt=3)          # > 128 frames: the flow's k = 5 convs have interior halos
    assert o["z_p"].shape[0] > dr.TILE
    ratios["halo_hi_flow"] = _ratio(t, sid, "flow.3", o["z_p"], halo_hi=True)
    print(voice, {k: f"{v:.3g}" for k, v in ratios.items()})
    assert all(v >= 3 for v in ratios.values()), ratios


def test_bound_catches_wrong_speaker_bias():
    """The wrong speaker's conv_pre bias on one 128-frame granule lands at least 3x above the dec.pre bound."""
    t, sid, o = _oracle("medium_spk4_sid2", n_ph=60, utt=3)
    assert o["z"].shape[0] > 2 * dr.TILE
    wrong = np.asarray(t["dec.conv_pre.bias"], np.float64) + dr.cond_vector(t, "dec.cond", 1)
    r = _ratio(t, sid, "dec.pre", o["z"], bias_rows=(1, torch.from_numpy(wrong)))
    assert r >= 3, r


def test_bound_catches_xlow_padding_weight():
    """2^-12 weights in the zero padding of x_low's widened coupling pre (the first target channel read into every hidden
    channel) land at least 3x above the bound of every coupling layer."""
    t, sid, o = _oracle("x_low", n_ph=60, utt=3)
    src = "z_p"
    for f in (3, 2, 1, 0):
        r = _ratio(t, sid, f"flow.{f}", o[src], pad_weight=2.0 ** -12)
        assert r >= 3, (f, r)
        src = f"flow.{f}"


def _decoder_chain(t, z):
    """The float64 decoder stages from z (dec.pre .. wav) on the CPU, as numpy."""
    ar = dr.Arith("f64")
    ar.dev = torch.device("cpu")           # one deterministic device, so equal inputs give equal bits
    res = {"z": ar.t(z)}
    for name, src, fn in dr.stages(t):
        if not name.startswith("flow."):
            res[name] = fn(res[src], ar)
    return {k: dr._np(v) for k, v in res.items()}


@pytest.mark.parametrize("voice", ["x_low", "high"])
def test_chunk_halo_bounds_the_receptive_field(voice):
    """dec_reference.chunk_halo against the float64 chain: z is changed outside a slice [lo, hi) of a 64-frame window,
    and every row of every stage that chunk_halo calls interior to the slice keeps its bits; the row just past the halo
    on either side (one row less of halo) changes at every stage, so the halo is also no larger than it must be.  The
    changed rows are BIG times larger than z: the farthest rows reach a stage through one edge tap of every conv on the
    way, and at z's own scale that contribution falls below float64 rounding by the high voice's dec.mrf3."""
    BIG = 1e12
    t = voicegen.make_tensors(voice)
    a = dr.arch(t)
    halo = dr.chunk_halo(t)
    lo, hi, n = 16, 48, 64
    rng = np.random.default_rng(11)
    z = rng.standard_normal((n, a["inter"]))
    z2 = z.copy()
    z2[:lo] = BIG * rng.standard_normal((lo, a["inter"]))
    z2[hi:] = BIG * rng.standard_normal((n - hi, a["inter"]))
    r1, r2 = _decoder_chain(t, z), _decoder_chain(t, z2)
    assert set(halo) == set(r1)
    for name, (left, right) in halo.items():
        U = r1[name].shape[0] // n
        i0, i1 = lo * U + left, hi * U - right
        assert i0 < i1, (voice, name, left, right)
        assert np.array_equal(r1[name][i0:i1], r2[name][i0:i1]), (voice, name)
        if name != "z":
            assert not np.array_equal(r1[name][i0 - 1], r2[name][i0 - 1]), (voice, name, "left")
            assert not np.array_equal(r1[name][i1], r2[name][i1]), (voice, name, "right")


@pytest.mark.parametrize("voice", ["medium", "high"])
def test_bound_catches_conv_post_edge_tap(voice):
    """conv_post dropping the taps that cross a 512-row block edge lands at least 3x above the fp32-class waveform bound."""
    t, sid, o = _oracle(voice)
    x = o[f"dec.mrf{len(dr.arch(t)['up_rates']) - 1}"]
    assert x.shape[0] > 2 * dr.POST_BLOCK
    ref, f32 = dr.dec_post(t, x, dr.Arith("f64")), dr.dec_post(t, x, dr.Arith("f32"))
    bad = dr.dec_post(t, x, dr.Arith("f64", post_edge=True))
    assert dr.f32_check(f32, ref, f32)[2] <= 1 / dr.F32_MULT
    r = dr.f32_check(bad, ref, f32)[2]
    assert r >= 3, r
