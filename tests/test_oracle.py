"""CPU: the oracle against its committed golden vectors and against independent restatements of
the pieces whose upstream definition is a different formula (dense generate_path matmul, naive
relative attention, forward spline, dense ConvTranspose)."""
import glob
import math
import os
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import vits_oracle as vo
from sonata_b200 import voicegen

GOLD = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz")))


def _crc(t):
    c = 0
    for k in sorted(t):
        c = zlib.crc32(np.ascontiguousarray(t[k]).tobytes(), c)
    return c


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p) for p in GOLD])
def test_oracle_reproduces_golden(path, oracle_weights):
    g = np.load(path)
    q = os.path.basename(path).split("_")[0]
    assert _crc(voicegen.make_tensors(q)) == int(g["weights_crc"]), "synthetic voice generator drifted"
    W = oracle_weights(q)
    st = {}
    ew = g["eps_w"].T[None] if "eps_w" in g else None
    ez = g["eps_z"].T[None] if "eps_z" in g else None
    wav = vo.infer(W, g["ids"], g["scales"], eps_w=None if ew is None else torch.from_numpy(ew.copy()),
                   eps_z=None if ez is None else torch.from_numpy(ez.copy()), stages=st)
    assert st["y_len"] == int(g["y_len"])
    assert np.array_equal(np.cumsum(st["w_ceil"].view(-1).numpy()).astype(np.int32), g["cum"])
    assert wav.numel() == 256 * int(g["y_len"])          # hop pinned at piper/src/lib.rs:910
    assert float(np.abs(wav.numpy() - g["wav"]).max()) < 2e-5


def test_fp64_shadow_close(oracle_weights):
    t = voicegen.make_tensors("medium")
    W32, W64 = oracle_weights("medium"), vo.to_torch(t, torch.float64)
    ids = vo.synthetic_ids(10, utt=11)
    s32, s64 = {}, {}
    w32 = vo.infer(W32, ids, [0, 1, 0], stages=s32)
    w64 = vo.infer(W64, ids, [0, 1, 0], stages=s64)
    assert torch.equal(s32["w_ceil"].double(), s64["w_ceil"])
    assert float((w32.double() - w64).abs().max()) < 2e-5


def test_expand_equals_dense_generate_path():
    """commons.generate_path + attn^T matmul (the reference graph's dense form) == our gather."""
    torch.manual_seed(0)
    T, C = 13, 6
    w_ceil = torch.randint(0, 5, (1, 1, T)).float()
    y_len = int(max(w_ceil.sum().item(), 1))
    m_p, logs_p = torch.randn(1, C, T), torch.randn(1, C, T)
    cum = torch.cumsum(w_ceil.view(-1), 0)
    j = torch.arange(y_len)
    path = (j[None, :] < cum[:, None]).float()            # sequence_mask(cum_duration, t_y)  [T, y]
    path = path - F.pad(path, [0, 0, 1, 0])[:-1]          # path - shifted path
    dense = torch.matmul(path.T, m_p[0].T).T[None]        # attn^T . m_p
    got, _ = vo.expand(m_p, logs_p, w_ceil, y_len, None, 0.0)
    assert torch.allclose(got, dense, atol=1e-6)


def test_relative_attention_matches_naive():
    a = dict(hidden=8, heads=2, window=2)
    torch.manual_seed(1)
    W = {}
    p = "x."
    for c in ("conv_q", "conv_k", "conv_v", "conv_o"):
        W[p + c + ".weight"] = torch.randn(8, 8, 1) * 0.3
        W[p + c + ".bias"] = torch.randn(8) * 0.1
    W[p + "emb_rel_k"] = torch.randn(1, 5, 4)
    W[p + "emb_rel_v"] = torch.randn(1, 5, 4)
    for T in (1, 2, 3, 7):
        x = torch.randn(1, 8, T)
        got = vo._mha(W, p, x, a)
        q = F.conv1d(x, W[p + "conv_q.weight"], W[p + "conv_q.bias"])[0].view(2, 4, T)
        k = F.conv1d(x, W[p + "conv_k.weight"], W[p + "conv_k.bias"])[0].view(2, 4, T)
        v = F.conv1d(x, W[p + "conv_v.weight"], W[p + "conv_v.bias"])[0].view(2, 4, T)
        out = torch.zeros(2, 4, T)
        for h in range(2):
            for i in range(T):
                qi = q[h, :, i] / 2.0
                s = torch.stack([qi @ k[h, :, j] + (qi @ W[p + "emb_rel_k"][0, j - i + 2] if abs(j - i) <= 2 else 0.0)
                                 for j in range(T)])
                pr = torch.softmax(s, 0)
                o = sum(pr[j] * v[h, :, j] for j in range(T))
                o = o + sum(pr[j] * W[p + "emb_rel_v"][0, j - i + 2] for j in range(T) if abs(j - i) <= 2)
                out[h, :, i] = o
        ref = F.conv1d(out.view(1, 8, T), W[p + "conv_o.weight"], W[p + "conv_o.bias"])
        assert torch.allclose(got, ref, atol=1e-5), T


@pytest.mark.parametrize("n", [7, 300])
def test_attention_reference_matches_oracle_mha(n):
    """tests/att_reference.py (the fp64 reference the CUDA attention is held to) against the oracle's `_mha` on layer 0
    of the medium voice: the band-by-band restatement and the oracle's rel_to_abs / abs_to_rel reshapes must agree, so
    they cannot share a misreading of the relative-position indexing.  conv_o is applied to the reference in float64."""
    import att_reference as ar
    t = voicegen.make_tensors("medium")
    a = voicegen.ARCH["medium"]
    ids = vo.synthetic_ids(n // 2, utt=4)[:n]
    x0, (q, k, v) = ar.project_qkv(t, 0, ids)
    relk, relv = ar.rel_embeddings(t, 0)
    Ps, out = ar.attention(q, k, v, relk, relv, a["heads"])
    assert all(np.allclose(P.sum(1), 1.0, rtol=0, atol=1e-12) for P in Ps)
    p = "enc_p.encoder.attn_layers.0."
    wo = np.asarray(t[p + "conv_o.weight"], dtype=np.float64)[:, :, 0]
    got = out @ wo.T + np.asarray(t[p + "conv_o.bias"], dtype=np.float64)
    W64 = vo.to_torch(t, torch.float64)
    ref = vo._mha(W64, p, torch.from_numpy(x0.T[None].copy()), a)[0].T.numpy()
    assert got.shape == ref.shape == (n, a["hidden"])
    assert float(np.abs(got - ref).max()) < 1e-10 * max(1.0, float(np.abs(ref).max()))


def test_pv_emulation_places_degraded_splits_above_attention_bound():
    """The accuracy bound of the tensor-core attention (att_reference.ATT_MULT x the fp32 kernel's error + a floor) is
    tight enough to catch a degraded P.V contraction.  CPU emulation (tools/emu_tc_accuracy.py model) of head 0 of
    layer 0 at T = 1280 keys, the longest utterance the tensor-core attention takes, with the fp32 kernel's summation
    order standing in for the fp32 kernel: the 3xTF32 chunk-flushed contraction lands below the bound; a single TF32
    MMA, two of the three split products, and the accumulation without the chunk flush each land above it.  Emulated
    (max |err|, |P.V| <= 2.3): fp32 kernel order 5.3e-6 (5.3e-6 measured on an H100 at T = 1280), 3xTF32 flushed
    1.8e-6, bound 1.5e-5; 1xTF32 1.3e-3, 2 products 8.3e-4, no flush 2.6e-5."""
    import att_reference as ar
    t = voicegen.make_tensors("medium")
    ids = vo.synthetic_ids(640, utt=9)[:1280]
    _, (q, k, v) = ar.project_qkv(t, 0, ids)
    relk, relv = ar.rel_embeddings(t, 0)
    D = q.shape[1] // voicegen.ARCH["medium"]["heads"]
    P, _ = ar.attention_head(q[:, :D], k[:, :D], v[:, :D], relk, relv)
    V = v[:, :D].astype(np.float32)
    e = ar.emulated_pv_errors(P, V)
    bound = ar.ATT_MULT * e["fp32_simt"] + ar.ATT_FLOOR * float(np.abs(P @ V).max())
    print({key: f"{val:.2e}" for key, val in e.items()}, f"bound {bound:.2e}", f"max|P.V| {float(np.abs(P @ V).max()):.2f}")
    assert e["3xtf32"] <= bound, (e, bound)
    for degraded in ("1xtf32", "2_products", "no_flush"):
        assert e[degraded] > bound, (degraded, e, bound)


@pytest.mark.parametrize("nspk,sid,n", [(1, None, 41), (4, 3, 300)])
def test_dp_reference_matches_oracle_sdp_reverse(nspk, sid, n):
    """tests/dp_reference.py (the float64 restatement the CUDA duration predictor is held to) against the oracle's
    `sdp_reverse` in float64, on the medium voice and the 4-speaker medium voice at sid 3, noise_w 0.8: dp.g, every
    flow's output and logw.  The oracle flips z between the flows; the reference keeps the columns fixed."""
    import dp_reference as dr
    t = voicegen.make_tensors("medium", n_speakers=nspk)
    W64 = vo.to_torch(t, torch.float64)
    a = vo.arch_of(W64)
    ids = vo.synthetic_ids(n // 2, utt=6)[:n]
    x64, _, _ = vo.text_encoder(W64, torch.as_tensor(ids).view(1, -1), a)
    eps = np.random.default_rng(2).standard_normal((n, 2))
    st = {}
    logw = vo.sdp_reverse(W64, x64, torch.from_numpy(eps.T[None].copy()), 0.8, a, stages=st,
                          g=vo.speaker_embedding(W64, sid))[0, 0].numpy()
    g = dr.dp_cond(t, x64[0].T.numpy(), sid)
    z = eps * 0.8
    for s in range(3):
        h29 = dr.flow_h29(t, s, dr.flow_h(t, s, z, g))
        uw, uh, ud = h29[:, :10] / np.sqrt(a["hidden"]), h29[:, 10:20] / np.sqrt(a["hidden"]), h29[:, 20:29]
        tc = dr.flow_cols(s)[1]
        z = z.copy()
        z[:, tc] = dr.rqs_inverse(z[:, tc], uw, uh, ud)
        ora = st[f"dp.flow{dr.FLOWS[s]}"][0].T.numpy()
        assert float(np.abs((z[:, ::-1] if s % 2 == 0 else z) - ora).max()) < 1e-10, s
    m0 = float(W64["dp.flows.0.m"].reshape(-1)[0])
    logs0 = float(W64["dp.flows.0.logs"].reshape(-1)[0])
    assert float(np.abs(dr.ea_inverse(z[:, 0], m0, logs0) - logw).max()) < 1e-10


def test_dp_bound_catches_degraded_variants(oracle_weights):
    """The bound of the duration predictor's DDSConv stages (dp_reference.DP_MULT x the fp32 oracle's error + DP_FLOOR)
    is tight enough to catch a degraded kernel.  On flow 0's DDSConv of a 201-id utterance (noise_w 0.8), float32
    emulations with a tanh GELU, LN eps 1e-6, or a 1x1 on one TF32 product each land above it, and the correct float32
    chain below it.  A single-pass variance only loses accuracy where |mean| >> std, which this predictor's LN inputs
    are not: it is shown above the bound on flow 0's first LN input rows shifted by 64 (LN removes a common offset
    exactly)."""
    import dp_reference as dr
    t = voicegen.make_tensors("medium")
    W32, W64 = oracle_weights("medium"), vo.to_torch(t, torch.float64)
    a = vo.arch_of(W64)
    ids = vo.synthetic_ids(100, utt=5)
    x = vo.text_encoder(W64, torch.as_tensor(ids).view(1, -1), a)[0][0].T.numpy().astype(np.float32)
    g = dr.dp_cond(t, x).astype(np.float32)
    z = (np.random.default_rng(0).standard_normal((len(ids), 2)) * 0.8).astype(np.float32)
    ref = dr.flow_h(t, 0, z, g)
    p = "dp.flows.7."
    zc = torch.from_numpy(z[:, 1].copy()).view(1, 1, -1)
    h32 = vo._dds(W32, p + "convs.", vo._conv(W32, p + "pre", zc), a, g=torch.from_numpy(g.T[None].copy()))[0].T.numpy()
    bound = dr.DP_MULT * float(np.abs(h32 - ref).max()) + dr.DP_FLOOR
    err = {k: float(np.abs(dr.flow_h(t, 0, z, g, np.float32, **v) - ref).max())
           for k, v in (("fp32", {}), ("tanh_gelu", dict(tanh=True)), ("ln_eps_1e-6", dict(eps=1e-6)),
                        ("one_tf32_1x1", dict(one_tf32=True)))}
    y = dr.depthwise(dr.flow_pre(t, 0, z, g), t[p + "convs.convs_sep.0.weight"], t[p + "convs.convs_sep.0.bias"], 1)
    y = (y + 64.0).astype(np.float32)
    gm, bt = t[p + "convs.norms_1.0.gamma"], t[p + "convs.norms_1.0.beta"]
    ln_ref = dr.layer_norm(y.astype(np.float64), gm, bt)
    ln_bound = dr.DP_MULT * float(np.abs(dr.layer_norm(y, gm, bt, np.float32) - ln_ref).max()) + dr.DP_FLOOR
    err["one_pass_var"] = float(np.abs(dr.layer_norm(y, gm, bt, np.float32, one_pass=True) - ln_ref).max())
    print({k: f"{v:.2e}" for k, v in err.items()}, f"bound {bound:.2e}", f"LN bound {ln_bound:.2e}")
    assert err["fp32"] <= bound, (err, bound)
    for k in ("tanh_gelu", "ln_eps_1e-6", "one_tf32_1x1"):
        assert err[k] > bound, (k, err, bound)
    assert err["one_pass_var"] > ln_bound, (err, ln_bound)


def test_spline_bound_catches_wrong_splines():
    """The element-wise bound of the spline kernel (dp_reference.spline_error_bound) is tight enough to catch a wrong
    spline: on every edge parameter set and input of the kernel test, the kernel's arithmetic emulated on the host with
    d_k and d_{k+1} swapped, or with 1.9 delta for 2 delta in e, lands above it (by a factor of 40 or more), and the
    correct arithmetic (contracted or not) lies within it."""
    import dp_reference as dr
    rng = np.random.default_rng(7)
    worst = {}
    for name, uw, uh, ud in dr.edge_params(rng):
        _, _, ch = dr.spline_fp32(np.zeros(1, np.float32), uw[None], uh[None], ud[None])
        y = dr.edge_inputs(ch[0])
        y = y[(y >= -5) & (y <= 5)]
        p = [np.repeat(a[None], len(y), 0) for a in (uw, uh, ud)]
        ref, bound = dr.spline_error_bound(y, *p)
        for fused in (True, False):
            assert np.all(np.abs(dr.spline_fp32(y, *p, fused)[0] - ref) <= bound), (name, fused)
        for defect in ("swap_d", "e_1.9"):
            r = float(np.max(np.abs(dr.spline_fp32(y, *p, defect=defect)[0] - ref) / bound))
            worst[defect] = min(worst.get(defect, np.inf), r)
            assert r > 1, (name, defect, r)
    print({k: f"{v:.0f}x the bound at least" for k, v in worst.items()})


def test_spline_fp32_emulation_meets_negative_discriminants():
    """dp_reference.spline_fp32 (spline_kernel's arithmetic in float32 on the host) finds fp32 discriminants below zero
    just under the knots of spline parameters with logits of std 3 -- where the unclamped kernel, like the fp32 graph,
    returns NaN -- and the clamped formula stays finite there and matches float64 away from such points."""
    import dp_reference as dr
    rng = np.random.default_rng(1)
    n = 300
    uw, uh, ud = (rng.normal(0, 3, (n, k)).astype(np.float32) for k in (10, 10, 9))
    _, _, ch = dr.spline_fp32(np.zeros(n, np.float32), uw, uh, ud)
    y = np.concatenate([(ch[:, k] - np.float32(d)).astype(np.float32) for k in range(1, 10)
                        for d in np.geomspace(1e-7, 1e-4, 20)])
    r = np.tile(np.arange(n), 9 * 20)
    out, disc, _ = dr.spline_fp32(y, uw[r], uh[r], ud[r])
    assert int((disc < 0).sum()) > 0
    assert np.isfinite(out).all() and (np.abs(out) <= 5).all()
    o32 = vo._rqs_inverse(torch.from_numpy(y).view(1, 1, -1), torch.from_numpy(uw[r]).view(1, 1, -1, 10),
                          torch.from_numpy(uh[r]).view(1, 1, -1, 10), torch.from_numpy(ud[r]).view(1, 1, -1, 9))
    assert bool(torch.isnan(o32).any())                 # the fp32 graph itself
    ref = dr.rqs_inverse(y.astype(np.float64), uw[r], uh[r], ud[r])
    assert float(np.median(np.abs(out - ref))) < 1e-5
    # forward / inverse round trip in float64
    x = rng.uniform(-5, 5, n)
    yy, _ = dr.rqs_forward(x, uw, uh, ud)
    assert float(np.abs(dr.rqs_inverse(yy, uw, uh, ud) - x).max()) < 1e-6


def _rqs_forward(x, uw, uh, ud, B=5.0):
    """transforms.rational_quadratic_spline(inverse=False), scalar restatement."""
    nb = len(uw)
    w = torch.softmax(uw, 0); w = 1e-3 + (1 - 1e-3 * nb) * w
    cw = F.pad(torch.cumsum(w, 0), (1, 0)); cw = 2 * B * cw - B; cw[0], cw[-1] = -B, B
    h = torch.softmax(uh, 0); h = 1e-3 + (1 - 1e-3 * nb) * h
    ch = F.pad(torch.cumsum(h, 0), (1, 0)); ch = 2 * B * ch - B; ch[0], ch[-1] = -B, B
    c = math.log(math.exp(1 - 1e-3) - 1)
    d = 1e-3 + F.softplus(torch.cat([torch.tensor([c]), ud, torch.tensor([c])]))
    k = int(torch.sum(x >= cw[:-1]).item()) - 1
    k = min(max(k, 0), nb - 1)
    W_, H_ = cw[k + 1] - cw[k], ch[k + 1] - ch[k]
    delta = H_ / W_
    th = (x - cw[k]) / W_
    num = H_ * (delta * th ** 2 + d[k] * th * (1 - th))
    den = delta + (d[k] + d[k + 1] - 2 * delta) * th * (1 - th)
    return ch[k] + num / den


def test_spline_inverse_inverts_forward():
    torch.manual_seed(3)
    for _ in range(50):
        uw, uh, ud = torch.randn(10) * 1.5, torch.randn(10) * 1.5, torch.randn(9)
        x = torch.rand(()) * 9.0 - 4.5
        y = _rqs_forward(x.double(), uw.double(), uh.double(), ud.double())
        xr = vo._rqs_inverse(y.view(1, 1, 1), uw.double().view(1, 1, 1, 10), uh.double().view(1, 1, 1, 10),
                             ud.double().view(1, 1, 1, 9))
        assert abs(float(xr) - float(x)) < 1e-6
    # identity outside the tails
    out = vo._rqs_inverse(torch.tensor([[[7.5]]]), torch.zeros(1, 1, 1, 10), torch.zeros(1, 1, 1, 10), torch.zeros(1, 1, 1, 9))
    assert float(out) == 7.5


def test_flow_flip_folding_identity(oracle_weights):
    """The CUDA path folds the channel flips of the coupling block into its weights (even number of
    flips).  Check the algebra on the oracle: flips + plain weights == no flips + permuted weights."""
    W = oracle_weights("medium")
    a = vo.arch_of(W)
    torch.manual_seed(5)
    z = torch.randn(1, a["inter"], 9)
    ref = vo.flow_reverse(W, z.clone(), a)
    half = a["inter"] // 2
    s = z.clone()
    for step in range(a["flow_n"]):
        f = a["flow_n"] - 1 - step
        p = f"flow.flows.{2 * f}."
        rev = step % 2 == 0
        Wl = dict(W)
        if rev:
            Wl[p + "pre.weight"] = W[p + "pre.weight"].flip(1)
            Wl[p + "post.weight"] = W[p + "post.weight"].flip(0)
            Wl[p + "post.bias"] = W[p + "post.bias"].flip(0)
        cond = s[:, half:] if rev else s[:, :half]
        h = vo._conv(Wl, p + "pre", cond)
        h = vo._wn(Wl, p + "enc.", h, a)
        m = vo._conv(Wl, p + "post", h)
        if rev:
            s = torch.cat([s[:, :half] - m, s[:, half:]], 1)
        else:
            s = torch.cat([s[:, :half], s[:, half:] - m], 1)
    assert torch.allclose(s, ref, atol=1e-5)


def test_polyphase_equals_conv_transpose():
    """The CUDA path runs ConvTranspose1d(k, stride u, pad (k-u)/2) as u phase convolutions."""
    torch.manual_seed(7)
    for (u, k) in ((8, 16), (4, 8), (2, 4)):
        cin, cout, T = 4, 3, 11
        x = torch.randn(1, cin, T); w = torch.randn(cin, cout, k); b = torch.randn(cout)
        ref = F.conv_transpose1d(x, w, b, stride=u, padding=(k - u) // 2)
        out = torch.zeros(1, cout, T * u)
        pad = (k - u) // 2
        for p in range(u):
            pp = p + pad
            for d in range(-k, k + 1):
                kk = d * u + pp
                if 0 <= kk < k:
                    for q in range(T):
                        i = q - d
                        if 0 <= i < T:
                            out[0, :, q * u + p] += w[:, :, kk].T @ x[0, :, i]
        out += b[None, :, None]
        assert torch.allclose(out, ref, atol=1e-5)


def test_synthetic_ids_layout():
    ids = vo.synthetic_ids(5, utt=0)
    assert len(ids) == 12 and ids[0] == 1 and ids[-1] == 2
    assert all(ids[2:-1:2] == 0) and all(ids[1:-1:2] >= 3)
    from sonata_b200 import workload
    assert np.array_equal(ids, workload.synthetic_ids(5, utt=0))
