"""float64 restatement of the reverse residual-coupling flow and the HiFi-GAN decoder (oracle/vits_oracle.py
`flow_reverse` / `decoder`), written out stage by stage from the `voicegen.make_tensors` tensors rather than through the
oracle, a bf16x2 emulation of the same stages (the operand split conv_tc.cu computes, without its fp32 accumulation), and
the bounds the CUDA stages are held to.

Layout as the engine keeps it: time-major [rows][channels], one utterance, zero padding outside it.  Each stage takes its
input as the engine captured it and returns its output in the engine's channel order:
    flow.{f}   z after the coupling layer flow.flows.{2f} (f = flow_n - 1 first).  The engine folds the graph's Flip
               layers into the weights, so z keeps z_p's channel order: after an odd number of couplings the graph's z is
               the capture reversed along channels.  flow.0 is z.
    dec.pre    conv_pre(z) (+ dec.cond(g) on multi-speaker voices), frame rows
    dec.up{i}  ConvTranspose i of leaky_relu(previous stage), rows = frames x U (U = product of the rates so far)
    dec.mrf{i} the mean of the ResBlocks of stage i over dec.up{i}
    wav        tanh(conv_post(leaky_relu(dec.mrf{last}, 0.01)))

Every function evaluates its convolutions through an `Arith`: "f64" (the reference: float64, on the GPU when one is
present, as tools/conv_unit.conv_ref does), "f32" (float32, each conv one FMA chain per output as the fp32 CUDA-core
kernels accumulate: the fp32-class yardstick of backend 0 and the waveform) or "emu" (the bf16x2 emulation: every conv
operand after the leaky-ReLU prologue and every weight split into bf16 hi + lo, hi*hi + lo*hi + hi*lo summed in
float64).  Keyword mutations of an Arith model plausible kernel mistakes for
the CPU test that shows the bounds catch them."""
import numpy as np
import torch
import torch.nn.functional as F

DEV = torch.device("cuda" if torch.cuda.is_available() else "cpu")
TILE = 128              # rows of a conv_tc.cu tile at every row level
POST_BLOCK = 512        # rows a conv_post CTA stages
SLOPE = 0.1             # leaky-ReLU slope inside the decoder
POST_SLOPE = 0.01       # before conv_post (torch's default)

# Backend 1 (bf16x2 wgmma) stages are held, on every 128-row tile of the stage's row level, to
#     max |got - ref| <= mult * max |emu - ref| + TC_FLOOR * max |ref|
# (tc_bound), where ref is this module in float64 and emu the bf16x2 emulation, both from the kernel's own captured stage
# input, and mult is TC_MULT, or TC_MULT_RB1 on the ResBlock1 MRF stages.  The emulation has the kernel's split and none
# of its fp32 rounding; the floor covers that rounding (outputs, residual sums, the fp32 gate and MRF scale) on tiles where
# the split's own error is small.  A ResBlock1 stage chains 18 convs (two per dilation) with up to 256 x 11-term sums, and
# there the fp32 accumulation the emulation omits is of the split's own size: up to 3.1x the emulation's error.
# Measured on an H100 SXM (80 GB HBM3, 700 W power limit), medium / high / x_low / 4-speaker medium voices, frame counts
# {1, 2, 127, 128, 129, 255, 257, 700} in one batch, and medium 32 x 256 / high 16 x 512 phonemes, largest fraction of
# the bound on any tile (tests/test_flow_decoder_gpu.py -s prints the tables):
#     flow.{f}                      max |err| 1.6e-5 .. 2.9e-5   at most 0.34 of the bound: 2.9x margin
#     dec.pre, dec.up{i}            max |err| 1.5e-5 .. 4.4e-5   at most 0.44: 2.3x margin
#     dec.mrf{i}, ResBlock2         max |err| 5.6e-6 .. 1.1e-5   at most 0.33: 3.0x margin
#     dec.mrf{i}, ResBlock1         max |err| 1.1e-5 .. 3.8e-5   at most 0.77 at mult 4 (high dec.mrf0, full size),
#                                                                so mult 8 there: about 0.4, 2.5x margin
# Streaming decoder chunk passes, same H100, held to the same bounds (tests/test_chunk_decoder_gpu.py -s): the edge pass
# of each voice and backend (chunks of 1, 2, 127 .. 129, 180, 200 frames and whole latents of 290 .. 1030 frames) and
# 32 chunks of 51 frames on medium, largest fraction of the bound on any tile of any chunk:
#     dec.pre, dec.up{i}            max |err| 1.6e-5 .. 3.1e-5   at most 0.44
#     dec.mrf{i}, ResBlock2         max |err| 5.5e-6 .. 9.3e-6   at most 0.34
#     dec.mrf{i}, ResBlock1         max |err| 1.1e-5 .. 2.2e-5   at most 0.37 at mult 8
# tests/test_flow_decoder_host.py shows each emulated kernel mistake at least 3x above this bound.
TC_MULT = 4.0
TC_MULT_RB1 = 8.0
TC_FLOOR = 2.0 ** -20

# The waveform and every backend-0 (fp32 CUDA-core) stage are held, per utterance, to
#     max |got - ref| <= F32_MULT * max |f32 - ref| + F32_FLOOR * max |ref|
# (f32_bound), f32 being the same stage in float32 from the same captured input, each conv one sequential FMA chain per
# output (a blocked host GEMM accumulates more accurately than the CUDA-core kernels: conv_pre's 1344-term sums on
# backend 0 measured 7x the error of torch's fp32 CPU conv).
# Measured on the H100 above (same runs): max |err| 6.1e-7 .. 5.6e-6 on backend 0's stages and 4.9e-7 .. 1.0e-6 on the
# waveform, at most 0.31 of the bound: 3.2x margin.  Chunk passes (same runs as above): max |err| 5.4e-7 .. 4.7e-6 on
# backend 0's stages, at most 0.31, and 4.8e-7 .. 6.0e-7 on the waveform, at most 0.23.
F32_MULT = 4.0
F32_FLOOR = 2.0 ** -21


# --------------------------------------------------------------------------- architecture
def arch(T):
    a = [int(x) for x in np.asarray(T["hp.arch"])]
    keys = ["hidden", "inter", "filter", "heads", "layers", "kernel", "window", "n_vocab", "resblock", "up_init",
            "flow_n", "wn_layers", "flow_kernel", "dp_kernel", "dp_bins", "sample_rate"]
    d = dict(zip(keys, a))
    d["up_rates"] = [int(x) for x in np.asarray(T["hp.up_rates"])]
    d["up_kernels"] = [int(x) for x in np.asarray(T["hp.up_kernels"])]
    d["res_kernels"] = [int(x) for x in np.asarray(T["hp.res_kernels"])]
    d["res_dils"] = [[int(y) for y in r] for r in np.asarray(T["hp.res_dils"])]
    return d


def cond_vector(T, prefix, sid):
    """prefix.weight @ emb_g[sid] + prefix.bias in float64 (a speaker's conditioning), or None on single-speaker voices."""
    if "emb_g.weight" not in T:
        return None
    e = np.asarray(T["emb_g.weight"], dtype=np.float64)[int(sid or 0)]
    return np.asarray(T[prefix + ".weight"], dtype=np.float64)[:, :, 0] @ e + np.asarray(T[prefix + ".bias"], np.float64)


# --------------------------------------------------------------------------- arithmetic
def bf16_split(x32):
    """(hi, lo) of a float32 tensor as float64: hi = bf16_rn(x), lo = bf16_rn(x - hi) (x - hi is exact in fp32)."""
    hi = x32.to(torch.bfloat16).to(torch.float32)
    lo = (x32 - hi).to(torch.bfloat16)
    return hi.double(), lo.double()


def _shift(x, o):
    """Rows q of the result are x[q + o], zero outside x."""
    n = x.shape[0]
    y = torch.zeros_like(x)
    lo, hi = max(0, -o), min(n, n - o)
    if lo < hi:
        y[lo:hi] = x[lo + o:hi + o]
    return y


class Arith:
    """Evaluation of a stage's convolutions, on the GPU when one is present.  mode "f64", "f32" or "emu" (module
    docstring).  Mutations (emu, except post_edge which is f64):
        drop_hilo=name    the conv whose weight prefix is `name` skips its hi(x)*lo(w) products
        halo_hi=True      inputs on the halo rows of each 128-row output tile (rows another tile owns) lose their lo half
        up_shift=(i, p)   phase p of ConvTranspose i reads every tap one row later
        bias_rows=(g, b)  rows of 128-row granule g take bias b instead of the stage's bias (dec.pre)
        mrf_scale=s       the MRF mean uses s instead of 1/3
        pad_weight=w      x_low's widened coupling pre reads the first target channel with weight w into every hidden
                          channel (one column of the zero padding)
        post_edge=True    conv_post drops every tap that crosses a 512-row block edge"""

    def __init__(self, mode, **mut):
        assert mode in ("f64", "f32", "emu")
        self.mode = mode
        self.dt = torch.float32 if mode == "f32" else torch.float64
        self.dev = DEV
        self.mut = mut

    def t(self, a):
        if torch.is_tensor(a):
            return a.to(self.dev, self.dt)
        return torch.from_numpy(np.ascontiguousarray(a)).to(self.dev, self.dt)

    def _w(self, w):
        return torch.from_numpy(np.ascontiguousarray(np.asarray(w, dtype=np.float32))).to(self.dev)

    def _bias(self, b, rows, cout):
        if b is None:
            return torch.zeros(cout, dtype=self.dt, device=self.dev)
        b = self.t(b)
        g = self.mut.get("bias_rows")
        if g is not None:
            b = b.expand(rows, cout).clone()
            b[g[0] * TILE:(g[0] + 1) * TILE] = self.t(g[1])
        return b

    def act(self, x, slope):
        """The leaky-ReLU prologue in the mode's precision: float32 x * slope in the emulation, as the kernel does."""
        if slope == 1.0:
            return x
        if self.mode == "emu":
            x32 = x.float()
            return torch.where(x32 > 0, x32, x32 * slope).double()
        return torch.where(x > 0, x, x * slope)

    def conv(self, x, w, b, dil=1, slope=1.0, name="", pad=None):
        """[rows][cin] -> [rows][cout]: b + conv(leaky_relu(x, slope), w [cout][cin][k], dilation dil), zero padding
        dil (k - 1) / 2 (or `pad`) rows each side."""
        x = self.t(x)
        k = np.asarray(w).shape[2]
        pad = dil * (k - 1) // 2 if pad is None else pad
        rows, cout = x.shape[0], np.asarray(w).shape[0]
        bias = self._bias(b, rows, cout)
        xin = self.act(x, slope)
        if self.mode == "f64":
            return F.conv1d(xin.T[None], self._w(w).double(), None, dilation=dil, padding=pad)[0].T + bias
        offs = [t * dil - pad for t in range(k)]
        if self.mode == "f32":
            return self._chain(xin, w, offs) + bias
        return self._taps(xin.float(), w, offs, name) + bias

    def _chain(self, x32, w, offs, shift=0):
        """fp32 emulation of sum_t x[q + offs[t]] . w[:, :, t]^T as one FMA chain per output over (tap, channel), the
        order and rounding class of the fp32 CUDA-core kernels (a blocked host GEMM accumulates more accurately)."""
        w = self._w(w)
        y = torch.zeros(x32.shape[0], w.shape[0], dtype=torch.float32, device=self.dev)
        for t, o in enumerate(offs):
            xs = _shift(x32, o + shift).double()
            wt = w[:, :, t].double()
            for c in range(xs.shape[1]):
                y = (y.double() + xs[:, c:c + 1] * wt[:, c][None]).float()
        return y

    def _taps(self, x32, w, offs, name, shift=0):
        """bf16x2 emulation of sum_t x[q + offs[t] + shift] . w[:, :, t]^T (rows outside x read zero)."""
        xh, xl = bf16_split(x32)
        wh, wl = bf16_split(self._w(w))
        drop = self.mut.get("drop_hilo") == name
        halo = self.mut.get("halo_hi", False)
        q = torch.arange(x32.shape[0], device=self.dev)
        y = torch.zeros(x32.shape[0], wh.shape[0], dtype=torch.float64, device=self.dev)
        for t, o in enumerate(offs):
            o = o + shift
            sh, sl = _shift(xh, o), _shift(xl, o)
            if halo:
                sl = sl * (((q + o) // TILE) == (q // TILE))[:, None]
            Wh, Wl = wh[:, :, t].T, wl[:, :, t].T
            y += sh @ Wh + sl @ Wh
            if not drop:
                y += sh @ Wl
        return y

    def conv_transpose(self, x, w, b, u, i):
        """ConvTranspose1d i of leaky_relu(x, 0.1): w [cin][cout][k], stride u, padding (k - u) / 2 -> [rows * u][cout].
        The emulation runs it as u polyphase convs (output row q u + p reads input rows q - d for every d with
        0 <= d u + p + pad < k, kernel index d u + p + pad), as the engine's weight images lay it out."""
        x = self.t(x)
        w = np.asarray(w)
        k = w.shape[2]
        pad = (k - u) // 2
        xin = self.act(x, SLOPE)
        if self.mode == "f64":
            y = F.conv_transpose1d(xin.T[None], self._w(w).double(), None, stride=u, padding=pad)[0].T
            return y + self.t(b)
        rows, cout = x.shape[0], w.shape[1]
        y = torch.zeros(rows, u, cout, dtype=self.dt, device=self.dev)
        for p in range(u):
            ds = [d for d in range(-k, k + 1) if 0 <= d * u + p + pad < k]
            wp = np.stack([w[:, :, d * u + p + pad].T for d in ds], axis=2)        # [cout][cin][taps]
            shift = 1 if self.mut.get("up_shift") == (i, p) else 0
            if self.mode == "f32":
                y[:, p] = self._chain(xin, wp, [-d for d in ds], shift)
            else:
                y[:, p] = self._taps(xin.float(), wp, [-d for d in ds], f"dec.ups.{i}", shift)
        return y.reshape(rows * u, cout) + self.t(b)

    def post(self, x, w):
        """tanh(conv_post(leaky_relu(x, 0.01))), k = 7, padding 3, no bias."""
        x = self.t(x)
        xin = torch.where(x > 0, x, x * POST_SLOPE)
        wt = self._w(w).to(self.dt)
        if self.mode == "f32":
            return torch.tanh(self._chain(xin, w, list(range(-3, 4))))
        if not self.mut.get("post_edge"):
            return torch.tanh(F.conv1d(xin.T[None], wt, None, padding=3)[0].T)
        q = torch.arange(x.shape[0], device=self.dev)
        y = torch.zeros(x.shape[0], 1, dtype=self.dt, device=self.dev)
        for t in range(7):
            o = t - 3
            keep = (((q + o) // POST_BLOCK) == (q // POST_BLOCK))[:, None]
            y += (_shift(xin, o) * keep) @ wt[:, :, t].T
        return torch.tanh(y)


# --------------------------------------------------------------------------- stages
def coupling(T, s, z, ar, sid=None):
    """Coupling step s (graph layer flow.flows.{2f}, f = flow_n - 1 - s) on the engine's z [rows][inter]."""
    a = arch(T)
    I, H, n = a["inter"], a["hidden"], a["wn_layers"]
    half = I // 2
    f = a["flow_n"] - 1 - s
    p = f"flow.flows.{2 * f}."
    z = ar.t(z)
    zg = z if s % 2 == 0 else z.flip(1)         # the graph's z before the layer's Flip
    zf = zg.flip(1)
    x0, x1 = zf[:, :half], zf[:, half:]
    pw = ar.mut.get("pad_weight")
    if pw is not None:
        w = np.zeros((H, I, 1), np.float32)
        w[:, :half] = T[p + "pre.weight"]
        w[:, half, 0] = pw
        h = ar.conv(zf, w, T[p + "pre.bias"], name=p + "pre")
    else:
        h = ar.conv(x0, T[p + "pre.weight"], T[p + "pre.bias"], name=p + "pre")
    gc = cond_vector(T, p + "enc.cond_layer", sid)
    out = None
    for l in range(n):
        b = np.asarray(T[p + f"enc.in_layers.{l}.bias"], np.float64)
        if gc is not None:
            b = b + gc[2 * H * l:2 * H * (l + 1)]
        xi = ar.conv(h, T[p + f"enc.in_layers.{l}.weight"], ar.t(torch.from_numpy(b)), name=p + f"enc.in_layers.{l}")
        acts = torch.tanh(xi[:, :H]) * torch.sigmoid(xi[:, H:])
        rs = ar.conv(acts, T[p + f"enc.res_skip_layers.{l}.weight"], T[p + f"enc.res_skip_layers.{l}.bias"],
                     name=p + f"enc.res_skip_layers.{l}")
        if l < n - 1:
            h = h + rs[:, :H]
            out = rs[:, H:] if out is None else out + rs[:, H:]
        else:
            out = rs if out is None else out + rs
    m = ar.conv(out, T[p + "post.weight"], T[p + "post.bias"], name=p + "post")
    zg = torch.cat([x0, x1 - m], 1)
    return zg.flip(1) if s % 2 == 0 else zg


def dec_pre(T, z, ar, sid=None):
    b = np.asarray(T["dec.conv_pre.bias"], np.float64)
    c = cond_vector(T, "dec.cond", sid)
    if c is not None:
        b = b + c
    return ar.conv(z, T["dec.conv_pre.weight"], ar.t(torch.from_numpy(b)), name="dec.conv_pre")


def dec_up(T, i, x, ar):
    a = arch(T)
    return ar.conv_transpose(x, T[f"dec.ups.{i}.weight"], T[f"dec.ups.{i}.bias"], a["up_rates"][i], i)


def dec_mrf(T, i, x, ar):
    """Mean of stage i's ResBlocks (ResBlock2: x += conv_m(lrelu x); ResBlock1: x += conv2_m(lrelu conv1_m(lrelu x)))."""
    a = arch(T)
    x = ar.t(x)
    nk = len(a["res_kernels"])
    xs = None
    for j, (rk, rd) in enumerate(zip(a["res_kernels"], a["res_dils"])):
        p = f"dec.resblocks.{i * nk + j}."
        xb = x
        for m, d in enumerate(rd):
            if a["resblock"] == 2:
                n = p + f"convs.{m}"
                xt = ar.conv(xb, T[n + ".weight"], T[n + ".bias"], dil=d, slope=SLOPE, name=n)
            else:
                n1, n2 = p + f"convs1.{m}", p + f"convs2.{m}"
                xt = ar.conv(xb, T[n1 + ".weight"], T[n1 + ".bias"], dil=d, slope=SLOPE, name=n1)
                xt = ar.conv(xt, T[n2 + ".weight"], T[n2 + ".bias"], dil=1, slope=SLOPE, name=n2)
            xb = xt + xb
        xs = xb if xs is None else xs + xb
    return xs * ar.mut.get("mrf_scale", 1.0 / nk)


def dec_post(T, x, ar):
    return ar.post(x, T["dec.conv_post.weight"])


def stages(T, sid=None):
    """[(output capture, input capture, fn(x, arith))] of the chain z_p -> flow.{f} ... -> z -> dec.pre -> dec.up{i} ->
    dec.mrf{i} -> wav, in order."""
    a = arch(T)
    out, prev = [], "z_p"
    for s in range(a["flow_n"]):
        name = f"flow.{a['flow_n'] - 1 - s}"
        out.append((name, prev, lambda x, ar, s=s: coupling(T, s, x, ar, sid)))
        prev = name
    out.append(("dec.pre", "z", lambda x, ar: dec_pre(T, x, ar, sid)))
    prev = "dec.pre"
    for i in range(len(a["up_rates"])):
        out.append((f"dec.up{i}", prev, lambda x, ar, i=i: dec_up(T, i, x, ar)))
        out.append((f"dec.mrf{i}", f"dec.up{i}", lambda x, ar, i=i: dec_mrf(T, i, x, ar)))
        prev = f"dec.mrf{i}"
    out.append(("wav", prev, lambda x, ar: dec_post(T, x, ar)))
    return out


def chunk_halo(T):
    """{stage: (left, right)} for z and the decoder stages: how many rows at each edge of a chunk (a slice of a latent
    decoded alone, every conv zero-padded at the slice's edges) may differ from the same rows of the whole latent
    decoded at once, in the stage's own rows (frames x U).  The rows between them read only rows of the slice, at every
    stage before them.  A centred conv of kernel k and dilation d adds d (k - 1) / 2 rows each side; a ConvTranspose of
    stride u, kernel k and padding p = (k - u) / 2 turns h rows into h u + k - p - u on the left (output row o reads
    input rows ceil((o + p - k + 1) / u) .. floor((o + p) / u)) and h u + p on the right; a stage's ResBlocks run side
    by side, so the MRF adds the largest of their chains."""
    a = arch(T)
    out = {"z": (0, 0)}
    h = (3, 3)                                           # conv_pre, k = 7
    out["dec.pre"] = h
    for i, (u, k) in enumerate(zip(a["up_rates"], a["up_kernels"])):
        p = (k - u) // 2
        h = (max(0, h[0] * u + k - p - u), h[1] * u + p)
        out[f"dec.up{i}"] = h
        grow = 0
        for rk, rd in zip(a["res_kernels"], a["res_dils"]):
            per = [d * (rk - 1) // 2 + ((rk - 1) // 2 if a["resblock"] == 1 else 0) for d in rd]
            grow = max(grow, sum(per))
        h = (h[0] + grow, h[1] + grow)
        out[f"dec.mrf{i}"] = h
    out["wav"] = (h[0] + 3, h[1] + 3)                    # conv_post, k = 7
    return out


def run_chain(T, z_p, ar, sid=None):
    """Every stage of one utterance from z_p, each from the previous stage's output in `ar`'s arithmetic."""
    res, cur = {"z_p": ar.t(z_p)}, None
    for name, src, fn in stages(T, sid):
        x = res["z"] if src == "z" else res[src]
        res[name] = fn(x, ar)
        if name == "flow.0":
            res["z"] = res[name]
    return res


# --------------------------------------------------------------------------- bounds
def _np(a):
    return a.detach().to("cpu", torch.float64).numpy() if torch.is_tensor(a) else np.asarray(a, dtype=np.float64)


def tile_max(a, tile=TILE):
    """Max |a| over each `tile` rows (all columns)."""
    a = np.abs(_np(a)).reshape(a.shape[0], -1).max(axis=1)
    n = (len(a) + tile - 1) // tile
    return np.pad(a, (0, n * tile - len(a))).reshape(n, tile).max(axis=1)


def tc_mult(T, stage):
    """The emulation-error multiplier of a stage's bound: TC_MULT_RB1 on ResBlock1 MRF stages, else TC_MULT."""
    return TC_MULT_RB1 if stage.startswith("dec.mrf") and arch(T)["resblock"] == 1 else TC_MULT


def tc_bound(ref, emu, mult=TC_MULT):
    """Per 128-row tile: mult * max |emu - ref| + TC_FLOOR * max |ref|."""
    ref, emu = _np(ref), _np(emu)
    return mult * tile_max(emu - ref) + TC_FLOOR * tile_max(ref)


def f32_bound(ref, f32):
    ref, f32 = _np(ref), _np(f32)
    return F32_MULT * float(np.abs(f32 - ref).max()) + F32_FLOOR * float(np.abs(ref).max())


def tc_check(got, ref, emu, mult=TC_MULT):
    """(max |got - ref|, max |emu - ref|, largest ratio of a tile's error to its bound, that tile)."""
    got, ref, emu = _np(got), _np(ref), _np(emu)
    err = tile_max(got - ref)
    r = err / tc_bound(ref, emu, mult)
    k = int(np.argmax(r))
    return float(err.max()), float(np.abs(emu - ref).max()), float(r[k]), k


def f32_check(got, ref, f32):
    got, ref = _np(got), _np(ref)
    e = float(np.abs(got - ref).max())
    return e, float(np.abs(_np(f32) - ref).max()), e / f32_bound(ref, f32)
