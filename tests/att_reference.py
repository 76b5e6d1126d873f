"""float64 restatement of the text encoder's relative-position attention (VITS `MultiHeadAttention` with `window_size`,
oracle/vits_oracle.py `_mha`), written out band by band rather than through the oracle's rel_to_abs / abs_to_rel
reshapes, and the accuracy bound the CUDA attention is held to against it.

Layout as the engine keeps it: time-major [T][channels], heads side by side in the channel dimension."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# The tensor-core attention (two 3xTF32 grouped GEMMs around the softmax) is held to
#     max |att0 - ref| <= ATT_MULT * (max |att0_fp32 - ref|) + ATT_FLOOR * max |ref|
# per utterance, where att0_fp32 is the fp32 CUDA-core attention kernel on the same Q / K / V.  The floor is the
# precision of the split operands themselves: hi + lo carries 21-22 significant bits, so even T = 1 (P = 1, out = v +
# E_v) is 2^-22 |v| away from float64 (measured 5.9e-7 at |ref| = 2.7).  Measured on an H100 SXM (80 GB HBM3, 400 W
# power limit), medium voice, layer 0, max |err| per utterance, |ref| <= 2.7:
#     T          1        31-65           95-257          639-641         1279-1280
#     fp32     1.2e-7   4.1e-7-8.1e-7    5.8e-7-1.3e-6    2.7e-6-2.9e-6   5.0e-6-5.3e-6
#     wgmma    5.9e-7   1.8e-6-3.4e-6    2.9e-6-3.6e-6    3.6e-6-3.8e-6   3.9e-6-4.1e-6
# (the fp32 fallback at T = 1281: 5.5e-6).  The CPU emulation in test_oracle.py puts a P.V contraction with a single
# TF32 MMA (1.3e-3), two of the three split products (8.3e-4), or no chunk flush (2.6e-5) at T = 1280 above this
# bound (1.5e-5 there); the chunk-flushed 3xTF32 contraction emulates at 1.8e-6.
ATT_MULT = 2.0
ATT_FLOOR = 2e-6


def fp32_att_bound(T, scale):
    """Bound of the fp32 CUDA-core attention kernel itself (backends 0 / 2, and every job past 1280 ids), so that it is not
    only the tensor-core path's yardstick: (8 + T / 16) ulp of max |ref|.  Each output of that kernel sums its T
    products in four fp32 FMA chains of T / 4 keys; measured on the H100 above, its error grows as ~T / 35 ulp of max |ref|
    (0.8 ulp at T = 1, 3.7 at 63, 19 at 640, 35 at 1280, 37 at 1281), which leaves at least 1.9x margin at every length
    tested, while a wrong band index, a dropped term or a reduced-precision accumulation lands orders of magnitude above."""
    return (8 + T / 16) * 2.0 ** -24 * scale


def project_qkv(T, layer, ids):
    """fp64 x0 = emb[ids] * sqrt(H) and its q / k / v projections [T][H] each (voicegen.make_tensors tensors)."""
    emb = np.asarray(T["enc_p.emb.weight"], dtype=np.float64)
    H = emb.shape[1]
    x0 = emb[np.asarray(ids)] * np.sqrt(H)
    p = f"enc_p.encoder.attn_layers.{layer}."
    out = []
    for c in ("conv_q", "conv_k", "conv_v"):
        w = np.asarray(T[p + c + ".weight"], dtype=np.float64)[:, :, 0]
        out.append(x0 @ w.T + np.asarray(T[p + c + ".bias"], dtype=np.float64))
    return x0, out


def rel_embeddings(T, layer):
    p = f"enc_p.encoder.attn_layers.{layer}."
    return (np.asarray(T[p + "emb_rel_k"], dtype=np.float64)[0], np.asarray(T[p + "emb_rel_v"], dtype=np.float64)[0])


def _band(T, window):
    """(d, rows i, keys j = i + d - window) of the relative band, clipped to the utterance."""
    i = np.arange(T)
    for d in range(2 * window + 1):
        j = i + d - window
        ok = (j >= 0) & (j < T)
        yield d, i[ok], j[ok]


def attention_head(q, k, v, relk, relv):
    """One head: q, k, v [T][D], relk / relv [2w+1][D] -> (P [T][T], out [T][D]), in the dtype of q (float64 for the
    reference; float32 gives an fp32 yardstick).
    scores_ij = q_i.k_j / sqrt(D) + [|j-i| <= w] q_i.relk[j-i+w] / sqrt(D);  P = softmax over the T keys;
    out_i = sum_j P_ij v_j + sum_{|j-i| <= w} P_ij relv[j-i+w]."""
    dt = np.asarray(q).dtype
    q, k, v, relk, relv = (np.asarray(a, dtype=dt) for a in (q, k, v, relk, relv))
    Tn, D = q.shape
    window = (relk.shape[0] - 1) // 2
    qs = q / dt.type(np.sqrt(D))
    S = qs @ k.T
    L = qs @ relk.T
    for d, i, j in _band(Tn, window):
        S[i, j] += L[i, d]
    S = S - S.max(axis=1, keepdims=True)
    P = np.exp(S)
    P /= P.sum(axis=1, keepdims=True)
    out = P @ v
    for d, i, j in _band(Tn, window):
        out[i] += P[i, j, None] * relv[d]
    return P, out


def attention(q, k, v, relk, relv, heads):
    """All heads in float64: q, k, v [T][H] -> (list of P per head, out [T][H])."""
    q, k, v = (np.asarray(a, dtype=np.float64) for a in (q, k, v))
    D = q.shape[1] // heads
    Ps, outs = [], []
    for h in range(heads):
        s = slice(h * D, (h + 1) * D)
        P, o = attention_head(q[:, s], k[:, s], v[:, s], relk, relv)
        Ps.append(P)
        outs.append(o)
    return Ps, np.concatenate(outs, axis=1)


def simt_pv(x, w):
    """P.V in the order of the fp32 CUDA-core attention kernel (kernels_misc.cu attention_kernel): four fp32 FMA chains
    over the key groups j // 4 = part (mod 4), combined as (c0 + c1) + (c2 + c3)."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from emu_tc_accuracy import fp32_fma
    groups = (np.arange(x.shape[1]) // 4) % 4
    c = [fp32_fma(x[:, groups == part], w[groups == part]) for part in range(4)]
    return (c[0] + c[1]) + (c[2] + c[3])


def emulated_pv_errors(P, V, chunk=8):
    """max |P.V - (P.V)_fp64| of emulated contractions (tools/emu_tc_accuracy.py model): the fp32 CUDA-core kernel's
    order, and 3xTF32 on the tensor core flushed every `chunk` K-steps (conv_tf.cu: 2 K-blocks of 32 keys = 8 tf32
    K-steps) with the degradations the attention bound must catch."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from emu_tc_accuracy import emulate
    x, w = np.asarray(P, dtype=np.float32), np.asarray(V, dtype=np.float32)
    ref = x.astype(np.float64) @ w.astype(np.float64)
    err = lambda y: float(np.abs(y - ref).max())
    return {
        "fp32_simt": err(simt_pv(x, w)),
        "3xtf32": err(emulate(x, w, "tf32", "rz", chunk)),
        "1xtf32": err(emulate(x, w, "tf32", "rz", chunk, products=("hh",))),
        "2_products": err(emulate(x, w, "tf32", "rz", chunk, products=("hh", "lh"))),
        "no_flush": err(emulate(x, w, "tf32", "rz", 0)),
    }
