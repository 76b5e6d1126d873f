"""float64 restatement of the text encoder (oracle/vits_oracle.py `text_encoder`), written out stage by stage from the
`voicegen.make_tensors` tensors rather than through the oracle, the yardstick arithmetics the CUDA stages are measured
against, and the bounds they are held to.

Layout as the engine keeps it: time-major [rows][channels], one utterance, zero padding outside it.  Each stage takes its
input as the engine captured it (a debug job's `enc.*` captures) and returns its output in the engine's layout:
    enc.emb        emb[ids] * sqrt(H)
    enc.{l}.qkv    Q | K | V of layer l, 1x1 conv of the layer input (enc.emb, or enc.{l-1}.ln2)
    enc.{l}.att    relative-position attention of enc.{l}.qkv (tests/att_reference.py), heads side by side
    enc.{l}.o      conv_o(enc.{l}.att)
    enc.{l}.ln1    LN1(layer input + enc.{l}.o)
    enc.{l}.ffn1   relu(conv_1(enc.{l}.ln1)), k = 3, padding 1 / 1
    enc.{l}.ffn2   conv_2(enc.{l}.ffn1), k = 3
    enc.{l}.ln2    LN2(enc.{l}.ln1 + enc.{l}.ffn2); the last layer's is the engine's `x`
    stats          enc_p.proj(x): m_p | logs_p

Every stage evaluates through an `Arith`:
    "f64"  the reference (float64, on the GPU when one is present);
    "f32"  float32: each conv one sequential FMA chain per output in the kernels' (32-channel K-block, tap, channel) order,
           a two-pass float32 LayerNorm, and for the attention a float32 softmax with P.V in the fp32 CUDA-core kernel's
           order (att_reference.simt_pv).  The yardstick of backend 0 (and 2), of every LayerNorm and of the attention;
    "emu"  3xTF32 as conv_tf.cu computes it (tools/emu_tc_accuracy.emulate: operands split hi + lo, hi*hi, lo*hi, hi*lo
           per 8-channel K-step, the accumulator rounded toward zero, flushed into a float32 running sum every 2 K-blocks
           of 32 channels on 1x1 convs and every K-block x k taps on k = 3).  The yardstick of backend 1's contractions;
           LayerNorm and attention evaluate as in "f32".
Keyword mutations of an Arith model plausible kernel mistakes, for the CPU test that shows the bounds catch them.

Bounds (stage_check), each at least 2x above the worst value measured on an H100 SXM (80 GB HBM3, 700 W power limit) by
tests/test_encoder_gpu.py -s (medium / high / x_low voices; edge batches of 1 .. 1281 ids on backend 1, backend 1 with
the fp32 attention and backend 0; medium 32 x 256 and high 1 x 512 phonemes on backend 1):
    enc.emb      bit for bit with float32(emb) * float32(sqrt(H)).
    backend 1 contractions (qkv, o, ffn1 after the ReLU, ffn2, stats), per 128-row tile:
                 TF_MULT * max |emu - ref| + TF_FLOOR * max |ref|
    backend 0 contractions, per utterance: F32_MULT * max |f32 - ref| + F32_FLOOR * max |ref|
    LayerNorms, per utterance: LN_MULT * max |ln32 - ref| + LN_FLOOR * max |ref| (the floor covers rsqrtf)
    attention, per utterance: ATT_MULT * max |att32 - ref| + ATT_FLOOR * max |ref|, att32 the host float32 emulation
                 of the fp32 attention kernel.  At layer 0, where the fp32 kernel's own error on the same Q / K / V is
                 known, the GPU test asserts it lies within ATT_CAL of the emulation's, both ways.
Measured worst fractions of these bounds are quoted beside each constant."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import att_reference as ar  # noqa: E402
import dec_reference as dr  # noqa: E402

DEV = dr.DEV
TILE = 128
LN_EPS = 1e-5
KB = 32                 # channels of a K-block (conv_tf.cu and conv_simt.cu)
KSTEP = 8               # channels of one tf32 MMA K-step

# Measured on the H100 runs named in the module docstring; beside each constant the worst fraction of the bound seen on
# any tile or utterance of any stage, voice and configuration (medium and high share their encoder weights).
TF_MULT = 4.0           # qkv / o / ffn1 / ffn2 / stats on backend 1: at most 0.33 (x_low enc.l.qkv, T = 31)
TF_FLOOR = 2.0 ** -22
F32_MULT = 4.0          # the same on backend 0: at most 0.24 (the kernels' error is about the FMA chain's own)
F32_FLOOR = 2.0 ** -22
LN_MULT = 4.0           # both LayerNorms, every backend: at most 0.31
LN_FLOOR = 2.0 ** -22
ATT_MULT = 4.0          # fp32 attention kernel (backend 0, SB200_ATT_SIMT=1, T > 1280): at most 0.19; tensor-core
ATT_FLOOR = 2.0 ** -18  # attention: at most 0.41.  The floor is the tensor-core path's: its split operands leave up to
                        # 4.7e-6 at |ref| 2.3 at any T (att_reference.py), which 2^-22 (0.46 for the fp32 kernel at
                        # ATT_MULT 4) put at 1.7x the bound.  At T = 1280 this bound is ~1.5e-5, near an unflushed P.V's
                        # 2.6e-5 (att_reference.py): the flush there stays test_oracle.py's to show.
ATT_CAL = 4.0           # layer 0, fp32 kernel error / host float32 emulation error, either way: at most 2.02
# end to end (x and stats from the ids, no captures): E2E_MULT x the host chain's own error (f32 for backend 0, emu
# with the float32 attention for backend 1) + E2E_FLOOR x max |ref|: at most 0.34
E2E_MULT = 4.0
E2E_FLOOR = 2.0 ** -21


def arch(T):
    return dr.arch(T)


def _np(a):
    return dr._np(a)


# --------------------------------------------------------------------------- arithmetic
def round_to_bits(x32, bits):
    """tools/emu_tc_accuracy.round_to_bits on a torch float32 tensor."""
    u = x32.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    drop = 24 - bits
    u = u + ((1 << (drop - 1)) - 1) + ((u >> drop) & 1)
    u = ((u >> drop) << drop) & 0xFFFFFFFF
    u = torch.where(u >= 2 ** 31, u - 2 ** 32, u)
    return u.to(torch.int32).view(torch.float32)


def _to_f32_rz(x64):
    y = x64.float()
    over = y.double().abs() > x64.abs()
    return torch.where(over, torch.nextafter(y, torch.zeros_like(y)), y)


def emulate(x, w, chunk, products=("hh", "lh", "hl")):
    """tools/emu_tc_accuracy.emulate(x, w, "tf32", "rz", chunk, products) on torch float32 tensors x [M][K], w [K][N]
    (test_encoder_host.py checks the two agree bit for bit)."""
    xh = round_to_bits(x, 11)
    xl = round_to_bits(x - xh, 11)
    wh = round_to_bits(w, 11)
    wl = round_to_bits(w - wh, 11)
    parts = {"h": (xh.double(), wh.double()), "l": (xl.double(), wl.double())}
    pairs = [(parts[p[0]][0], parts[p[1]][1]) for p in products]
    M, K = x.shape
    total = torch.zeros(M, w.shape[1], dtype=torch.float32, device=x.device)
    acc = torch.zeros_like(total)
    steps = 0
    for k0 in range(0, K, KSTEP):
        for a, b in pairs:
            acc = _to_f32_rz(acc.double() + a[:, k0:k0 + KSTEP] @ b[k0:k0 + KSTEP])
        steps += 1
        if chunk and steps % chunk == 0:
            total = total + acc
            acc = torch.zeros_like(acc)
    return total + acc if chunk else acc


def fma_chain(x, w):
    """Sequential float32 FMA chain over K: x [M][K], w [K][N] (tools/emu_tc_accuracy.fp32_fma on torch tensors)."""
    x, w = x.double(), w.double()
    acc = torch.zeros(x.shape[0], w.shape[1], dtype=torch.float32, device=x.device)
    for k in range(x.shape[1]):
        acc = (acc.double() + x[:, k:k + 1] * w[k:k + 1]).float()
    return acc


def simt_pv(p, v):
    """att_reference.simt_pv on torch float32 tensors: four FMA chains over the key groups (j // 4) % 4, combined as
    (c0 + c1) + (c2 + c3)."""
    g = (torch.arange(p.shape[1], device=p.device) // 4) % 4
    c = [fma_chain(p[:, g == part], v[g == part]) for part in range(4)]
    return (c[0] + c[1]) + (c[2] + c[3])


class Arith:
    """Evaluation of the encoder's stages (module docstring).  Mutations:
        products=(..)       the emulated conv `conv` (or every conv) issues only these of hh / lh / hl per K-step
        no_flush=True       the emulated conv `conv` (or every conv) accumulates without the chunk flush
        conv=name           restricts products / no_flush to the conv whose weight prefix ends with `name`
        edge_rows=(a, b)    k = 3 convs read row a before the utterance and row b after it instead of zeros
        ffn_pad=(l, r)      k = 3 convs pad l rows before and r after (the graph: 1 / 1)
        ln_eps=e            LayerNorm epsilon e
        ln_var=kind         "unbiased" (divides by C - 1) or "onepass" (E[x^2] - mean^2 in the mode's precision)
        window=w            attention band of half-width w (the voice's window is 4)
        drop_relv_last=True the relative-value band term is left out of the last row
        zero_keys=True      keys [T, round_up(T, 32)) (zero Q.K score) stay inside the softmax sum
        rel_layer=l         attention takes layer l's relative embeddings
        swap_stats=True     the m and logs halves of stats trade places"""

    def __init__(self, mode, **mut):
        assert mode in ("f64", "f32", "emu")
        self.mode = mode
        self.dt = torch.float64 if mode == "f64" else torch.float32
        self.dev = DEV
        self.mut = mut

    def t(self, a, dt=None):
        dt = self.dt if dt is None else dt
        if torch.is_tensor(a):
            return a.to(self.dev, dt)
        return torch.from_numpy(np.ascontiguousarray(a)).to(self.dev, dt)

    # ---------------------------------------------------------------- convolution
    def conv(self, x, w, b, name, relu=False):
        """[rows][cin] -> [rows][cout]: (relu) b + conv(x, w [cout][cin][k]), padding (k - 1) / 2 each side."""
        x = self.t(x)
        w = np.asarray(w, dtype=np.float32)
        cout, cin, k = w.shape
        rows = x.shape[0]
        pl, pr = self.mut.get("ffn_pad", ((k - 1) // 2, k // 2)) if k > 1 else (0, 0)
        xp = torch.zeros(rows + pl + pr, cin, dtype=x.dtype, device=self.dev)
        xp[pl:pl + rows] = x
        edge = self.mut.get("edge_rows")
        if edge is not None and k > 1:
            xp[:pl] = self.t(edge[0])
            xp[pl + rows:] = self.t(edge[1])
        n_out = rows + pl + pr - (k - 1)
        taps = [xp[t:t + n_out] for t in range(k)]
        wt = torch.from_numpy(np.ascontiguousarray(w)).to(self.dev)            # float32 [cout][cin][k]
        if self.mode == "f64":
            y = sum(taps[t] @ wt[:, :, t].double().T for t in range(k)) + self.t(b)
        else:
            # K in the kernels' order: 32-channel K-block, then tap, then channel
            nkb = cin // KB
            xk = torch.stack([xi.float() for xi in taps], 1).reshape(n_out, k, nkb, KB).transpose(1, 2).reshape(n_out, -1)
            wk = wt.permute(2, 1, 0).reshape(k, nkb, KB, cout).transpose(0, 1).reshape(-1, cout)
            if self.mode == "f32":
                y = fma_chain(xk, wk)
            else:
                hit = self.mut.get("conv") is None or name.endswith(self.mut["conv"])
                chunk = 0 if hit and self.mut.get("no_flush") else (2 * KB // KSTEP if k == 1 else k * KB // KSTEP)
                prods = self.mut.get("products", ("hh", "lh", "hl")) if hit else ("hh", "lh", "hl")
                y = emulate(xk, wk, chunk, prods)
            y = y + self.t(b, torch.float32)
        return torch.relu(y) if relu else y

    # ---------------------------------------------------------------- LayerNorm
    def layer_norm(self, x, r, g, b):
        """LN over channels of x + r, eps 1e-5, biased variance, two-pass."""
        v = self.t(x) + self.t(r)
        C = v.shape[1]
        mean = v.sum(1, keepdim=True) / C
        kind = self.mut.get("ln_var")
        if kind == "onepass":
            var = (v * v).sum(1, keepdim=True) / C - mean * mean
        else:
            d = v - mean
            var = (d * d).sum(1, keepdim=True) / (C - 1 if kind == "unbiased" else C)
        eps = self.mut.get("ln_eps", LN_EPS)
        rstd = 1.0 / torch.sqrt(var + eps)
        return (v - mean) * rstd * self.t(g) + self.t(b)

    # ---------------------------------------------------------------- attention
    def attention(self, qkv, relk, relv, heads):
        """[T][3H] -> [T][H] (att_reference.attention in float64; its float32 softmax and simt_pv order otherwise)."""
        qkv = _np(qkv)
        T, H = qkv.shape[0], qkv.shape[1] // 3
        D = H // heads
        q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
        w = self.mut.get("window")
        if w is not None:
            c = (relk.shape[0] - 1) // 2
            relk, relv = relk[c - w:c + w + 1], relv[c - w:c + w + 1]
        if self.mut.get("zero_keys"):
            tz = (T + 31) // 32 * 32
            z = lambda a: np.concatenate([a, np.zeros((tz - T, a.shape[1]))])
            q, k, v = z(q), z(k), z(v)
        if self.mode == "f64":
            Ps, out = ar.attention(q, k, v, relk, relv, heads)
        else:
            Ps, outs = [], []
            rv = torch.from_numpy(np.asarray(relv, np.float32)).to(self.dev)
            for h in range(heads):
                s = slice(h * D, (h + 1) * D)
                P, _ = ar.attention_head(*(np.asarray(a, dtype=np.float32) for a in (q[:, s], k[:, s], v[:, s], relk,
                                                                                     relv)))
                Pt = torch.from_numpy(P).to(self.dev)
                o = simt_pv(Pt, torch.from_numpy(np.asarray(v[:, s], np.float32)).to(self.dev))
                n, win = P.shape[0], (relv.shape[0] - 1) // 2
                for d in range(2 * win + 1):                    # the band term, fma'd after the four key quarters
                    i = torch.arange(n, device=self.dev)
                    j = i + d - win
                    ok = (j >= 0) & (j < n)
                    o[ok] = (o[ok].double() + Pt[i[ok], j[ok], None].double() * rv[d].double()).float()
                Ps.append(P)
                outs.append(o.cpu().numpy())
            out = np.concatenate(outs, 1)
        out = np.array(out[:T], dtype=np.float64)
        if self.mut.get("drop_relv_last"):
            win = (relv.shape[0] - 1) // 2
            for h in range(heads):
                for d in range(2 * win + 1):
                    j = T - 1 + d - win
                    if 0 <= j < T:
                        out[T - 1, h * D:(h + 1) * D] -= Ps[h][T - 1, j] * np.asarray(relv[d], np.float64)
        return self.t(out)


# --------------------------------------------------------------------------- stages
def embed(T, ids, ar_):
    """emb[ids] * sqrt(H): float64 in "f64", else float32(emb) * float32(sqrt(H)) as the engine computes it."""
    emb = np.asarray(T["enc_p.emb.weight"])
    H = emb.shape[1]
    ids = np.asarray(ids, dtype=np.int64)
    if ar_.mode == "f64":
        return ar_.t(emb.astype(np.float64)[ids] * np.sqrt(H))
    return ar_.t(emb.astype(np.float32)[ids] * np.sqrt(np.float32(H)))


def _p(l):
    return f"enc_p.encoder.attn_layers.{l}.", f"enc_p.encoder.ffn_layers.{l}."


def qkv(T, l, x, ar_):
    p = _p(l)[0]
    w = np.concatenate([np.asarray(T[p + c + ".weight"]) for c in ("conv_q", "conv_k", "conv_v")])
    b = np.concatenate([np.asarray(T[p + c + ".bias"], np.float64) for c in ("conv_q", "conv_k", "conv_v")])
    return ar_.conv(x, w, b, p + "qkv")


def attention(T, l, qkv_, ar_):
    a = arch(T)
    relk, relv = ar.rel_embeddings(T, ar_.mut.get("rel_layer", l))
    return ar_.attention(qkv_, relk, relv, a["heads"])


def conv_o(T, l, x, ar_):
    p = _p(l)[0] + "conv_o"
    return ar_.conv(x, T[p + ".weight"], np.asarray(T[p + ".bias"], np.float64), p)


def ln(T, l, which, xr, ar_):
    p = f"enc_p.encoder.norm_layers_{which}.{l}"
    return ar_.layer_norm(xr[0], xr[1], np.asarray(T[p + ".gamma"], np.float64), np.asarray(T[p + ".beta"], np.float64))


def ffn(T, l, i, x, ar_):
    p = _p(l)[1] + f"conv_{i}"
    return ar_.conv(x, T[p + ".weight"], np.asarray(T[p + ".bias"], np.float64), p, relu=(i == 1))


def proj(T, x, ar_):
    y = ar_.conv(x, T["enc_p.proj.weight"], np.asarray(T["enc_p.proj.bias"], np.float64), "enc_p.proj")
    if ar_.mut.get("swap_stats"):
        I = y.shape[1] // 2
        y = torch.cat([y[:, I:], y[:, :I]], 1)
    return y


def stages(T):
    """[(output capture, input capture(s), kind, fn(x, arith))] of the chain ids -> enc.emb -> ... -> stats, in order.
    kind: "emb", "conv", "att" or "ln"; an "ln" stage's input is the pair (residual stream, branch output)."""
    a = arch(T)
    out, prev = [("enc.emb", "ids", "emb", lambda ids, ar_: embed(T, ids, ar_))], "enc.emb"
    for l in range(a["layers"]):
        p = f"enc.{l}."
        out += [
            (p + "qkv", prev, "conv", lambda x, ar_, l=l: qkv(T, l, x, ar_)),
            (p + "att", p + "qkv", "att", lambda x, ar_, l=l: attention(T, l, x, ar_)),
            (p + "o", p + "att", "conv", lambda x, ar_, l=l: conv_o(T, l, x, ar_)),
            (p + "ln1", (prev, p + "o"), "ln", lambda x, ar_, l=l: ln(T, l, 1, x, ar_)),
            (p + "ffn1", p + "ln1", "conv", lambda x, ar_, l=l: ffn(T, l, 1, x, ar_)),
            (p + "ffn2", p + "ffn1", "conv", lambda x, ar_, l=l: ffn(T, l, 2, x, ar_)),
            (p + "ln2", (p + "ln1", p + "ffn2"), "ln", lambda x, ar_, l=l: ln(T, l, 2, x, ar_)),
        ]
        prev = p + "ln2"
    out.append(("stats", prev, "conv", lambda x, ar_: proj(T, x, ar_)))
    return out


def inputs(src, caps):
    return tuple(caps[s] for s in src) if isinstance(src, tuple) else caps[src]


def run_chain(T, ids, ar_):
    """Every stage of one utterance from its ids, each from the previous stages' outputs in `ar_`'s arithmetic; "x" is
    the last layer's ln2."""
    res = {"ids": np.asarray(ids)}
    for name, src, _, fn in stages(T):
        res[name] = fn(inputs(src, res), ar_)
    res["x"] = res[f"enc.{arch(T)['layers'] - 1}.ln2"]
    return res


# --------------------------------------------------------------------------- bounds
def tile_max(a, tile=TILE):
    return dr.tile_max(a, tile)


def yardstick(kind, backend):
    """The Arith mode a stage's bound is built from: emu for backend-1 contractions, f32 for everything else."""
    return "emu" if kind == "conv" and backend == 1 else "f32"


def row_bounds(kind, ref, yard, backend):
    """The bound of every row of a stage: per 128-row tile for backend-1 contractions, per utterance otherwise."""
    ref, yard = _np(ref), _np(yard)
    n = ref.shape[0]
    if kind == "conv" and backend == 1:
        b = TF_MULT * tile_max(yard - ref) + TF_FLOOR * tile_max(ref)
        return np.repeat(b, TILE)[:n]
    mult, floor = {"conv": (F32_MULT, F32_FLOOR), "ln": (LN_MULT, LN_FLOOR), "att": (ATT_MULT, ATT_FLOOR)}[kind]
    return np.full(n, mult * float(np.abs(yard - ref).max()) + floor * float(np.abs(ref).max()))


def stage_check(kind, got, ref, yard, backend):
    """(max |got - ref|, max |yard - ref|, largest ratio of a row's error to its bound, that row)."""
    got, ref, yard = _np(got), _np(ref), _np(yard)
    err = np.abs(got - ref).reshape(ref.shape[0], -1).max(axis=1)
    r = err / row_bounds(kind, ref, yard, backend)
    k = int(np.argmax(r))
    return float(err.max()), float(np.abs(yard - ref).max()), float(r[k]), k


def e2e_check(got, ref, chain):
    got, ref, chain = _np(got), _np(ref), _np(chain)
    e, ec = float(np.abs(got - ref).max()), float(np.abs(chain - ref).max())
    return e, ec, e / (E2E_MULT * ec + E2E_FLOOR * float(np.abs(ref).max()))
