"""float64 restatement of the stochastic duration predictor (VITS `StochasticDurationPredictor`, reverse; oracle/vits_oracle.py
`sdp_reverse`), written out piece by piece from the `voicegen.make_tensors` tensors rather than through the oracle, a
float32 host emulation of the CUDA spline in the kernel's operation order, and the bounds the CUDA stages are held to.

Layout as the engine keeps it: time-major [T][channels], one utterance (zero padding outside it).  The two-channel z
keeps the columns of the graph's eps_w; the flips between the flows only alternate which column conditions (ccol) and
which is transformed (tcol): flow s = 0, 1, 2 is the graph's dp.flows.{7, 5, 3}, ccol = 1, 0, 1."""
import math

import numpy as np
import torch

FLOWS = (7, 5, 3)
NB = 10                 # spline bins
TAIL = 5.0              # spline tail bound: identity outside [-5, 5]
MIN_W = MIN_H = MIN_D = 1e-3

# dp.g and each flow's DDSConv output h are held, per utterance, to
#     max |got - ref| <= DP_MULT * max |fp32 - ref| + DP_FLOOR
# where fp32 is the oracle run in float32 (PyTorch on the host) on the kernel's own captured inputs and ref is this module
# in float64 (DP_FLOOR absolute: the residual stream reaches |h| = 70 at noise_w = 4, but a relative floor there would
# hide an LN eps of 1e-6).  Measured on an H100 SXM (80 GB HBM3, 400 W power limit), medium / high / 4-speaker medium
# voices, T in {1 .. 513}, noise_w in {0, 0.8, 4}, max |got - ref| per utterance:
#     dp.g   2.1e-6 .. 3.9e-6   (fp32 oracle 5.7e-7 .. 3.2e-6)   at most 0.52 of the bound: 1.9x margin
#     h      1.1e-6 .. 1.3e-5   (fp32 oracle 7.1e-7 .. 9.7e-6)   at most 0.36 of the bound: 2.8x margin
# The CPU test in test_oracle.py puts a tanh GELU (1.7e-3), LN eps 1e-6 (4.2e-5) and a 1x1 on one TF32 product (2.2e-3)
# above this bound (1.4e-5 there); a single-pass variance is indistinguishable from the two-pass one at this predictor's
# LN inputs (|channel mean| <= 0.6 std), so that test shows it above the bound on the same rows shifted by a common
# offset, which LayerNorm removes exactly.
DP_MULT = 4.0
DP_FLOOR = 2e-6

# The spline inverse is held, element by element, to
#     |got - ref| <= SPLINE_MULT * |spline_fp32 - ref| + SPLINE_K * 2^-24 * TAIL * (1 + 1 / F'(ref))
# (spline_error_bound).  The published root 2c / (-b - sqrt(b^2 - 4ac)) cancels in fp32 where a flat bin meets a steep
# derivative, and sqrt turns the disc's rounding into its square root at a bin's top, so the fp32 formula's own error
# there is not a function of the problem's conditioning alone; the first term is that error, taken from the kernel's
# arithmetic emulated on the host (the largest of the FMA-contracted and the uncontracted evaluation at y and +-2 ulp).
# The second term is a few ulp of the knot positions and of the input, over the forward slope F' at the float64 output.
# The CPU test in test_oracle.py puts a spline with d_k and d_{k+1} swapped (>= 1275x) and one with 1.9 delta for
# 2 delta in e (>= 47x) above this bound on the edge test's parameter sets.  Measured on the H100 above: at most 0.37 of
# the bound in the stage test (max |err| 2.0e-4), 2.7x margin; at most 0.32 on the edge sets (sigma 3; max |err| 6.4e-2
# at sigma 10, inside cancellation the host emulation shares), 3.1x margin.
SPLINE_MULT = 4.0
SPLINE_K = 16.0
# logw = (z0 - m0) * exp(-logs0): a subtraction, expf and a product; measured <= 2.5 ulp
LOGW_ULP = 6


# --------------------------------------------------------------------------- tensors
def _w(T, name):
    return np.asarray(T[name], dtype=np.float64)


def arch(T):
    H = np.asarray(T["dp.pre.weight"]).shape[0]
    k = np.asarray(T["dp.convs.convs_sep.0.weight"]).shape[2]
    return H, k


def ea_params(T):
    """(m0, logs0) of the ElementwiseAffine's first channel, as float32 values (what the engine keeps)."""
    return (float(np.float32(np.asarray(T["dp.flows.0.m"]).reshape(-1)[0])),
            float(np.float32(np.asarray(T["dp.flows.0.logs"]).reshape(-1)[0])))


# --------------------------------------------------------------------------- bands
def tf32(x):
    """Round-to-nearest-even to TF32 (10 explicit mantissa bits), for the degraded single-product variant."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0xFFF + ((b >> 13) & 1)) & ~np.uint64(0x1FFF)
    return b.astype(np.uint32).view(np.float32)


def conv1x1(x, w, b, dt=np.float64, one_tf32=False):
    """x [T][cin] . w[cout][cin][1]^T + b."""
    w2 = np.asarray(w, dtype=np.float64)[:, :, 0].T
    if one_tf32:
        return (tf32(x).astype(np.float64) @ tf32(w2).astype(np.float64) + np.asarray(b, dtype=np.float64)).astype(dt)
    return (np.asarray(x, dtype=dt) @ w2.astype(dt) + np.asarray(b, dtype=dt)).astype(dt)


def layer_norm(x, gamma, beta, dt=np.float64, eps=1e-5, one_pass=False):
    """modules.LayerNorm over the channels of [T][C]: biased variance, eps 1e-5; `one_pass` computes E[x^2] - E[x]^2."""
    x = np.asarray(x, dtype=dt)
    mean = x.mean(axis=1, keepdims=True, dtype=dt)
    if one_pass:
        var = (x * x).mean(axis=1, keepdims=True, dtype=dt) - mean * mean
    else:
        d = x - mean
        var = (d * d).mean(axis=1, keepdims=True, dtype=dt)
    return ((x - mean) / np.sqrt(var + dt(eps)) * np.asarray(gamma, dtype=dt) + np.asarray(beta, dtype=dt)).astype(dt)


def gelu(x, dt=np.float64, tanh=False):
    """Exact erf GELU (torch's default); `tanh` is the approximation."""
    x = np.asarray(x, dtype=dt)
    if tanh:
        return (dt(0.5) * x * (dt(1) + np.tanh(dt(math.sqrt(2 / math.pi)) * (x + dt(0.044715) * x ** 3)))).astype(dt)
    return (dt(0.5) * x * (dt(1) + torch.special.erf(torch.from_numpy(x * dt(1 / math.sqrt(2)))).numpy())).astype(dt)


def depthwise(x, w, b, dil, dt=np.float64):
    """Depthwise k-tap conv, dilation dil, zero padding outside the utterance: w [C][1][k]."""
    x = np.asarray(x, dtype=dt)
    w = np.asarray(w, dtype=dt)[:, 0, :]
    k = w.shape[1]
    Tn = x.shape[0]
    y = np.broadcast_to(np.asarray(b, dtype=dt), x.shape).copy()
    for t in range(k):
        o = (t - (k - 1) // 2) * dil
        lo, hi = max(0, -o), min(Tn, Tn - o)
        if lo < hi:
            y[lo:hi] += w[:, t] * x[lo + o:hi + o]
    return y


def ddsconv(T, p, x, dt=np.float64, **variant):
    """DDSConv (3 layers, dilation k^i): x += gelu(LN(1x1(gelu(LN(dw(x)))))).  variant: tanh=, one_pass=, eps=,
    one_tf32= (degradations for the bound test)."""
    _, k = arch(T)
    ln = dict(dt=dt, eps=variant.get("eps", 1e-5), one_pass=variant.get("one_pass", False))
    act = dict(dt=dt, tanh=variant.get("tanh", False))
    x = np.asarray(x, dtype=dt).copy()
    for i in range(3):
        y = depthwise(x, T[f"{p}convs_sep.{i}.weight"], T[f"{p}convs_sep.{i}.bias"], k ** i, dt)
        y = gelu(layer_norm(y, T[f"{p}norms_1.{i}.gamma"], T[f"{p}norms_1.{i}.beta"], **ln), **act)
        y = conv1x1(y, T[f"{p}convs_1x1.{i}.weight"], T[f"{p}convs_1x1.{i}.bias"], dt, variant.get("one_tf32", False))
        y = gelu(layer_norm(y, T[f"{p}norms_2.{i}.gamma"], T[f"{p}norms_2.{i}.beta"], **ln), **act)
        x = x + y
    return x


def dp_cond(T, x, sid=None, dt=np.float64, **variant):
    """g = proj(DDSConv(pre(x) + cond(emb_g[sid]))): the conditioning every flow adds ([T][H])."""
    h = conv1x1(x, T["dp.pre.weight"], T["dp.pre.bias"], dt)
    if "emb_g.weight" in T:
        e = _w(T, "emb_g.weight")[int(sid or 0)]
        h = h + (_w(T, "dp.cond.weight")[:, :, 0] @ e + _w(T, "dp.cond.bias")).astype(dt)
    h = ddsconv(T, "dp.convs.", h, dt, **variant)
    return conv1x1(h, T["dp.proj.weight"], T["dp.proj.bias"], dt)


def flow_cols(s):
    """(ccol, tcol) of flow s in the engine's unflipped z."""
    return (1, 0) if s % 2 == 0 else (0, 1)


def flow_pre(T, s, z, g, dt=np.float64):
    """h = pre(z[:, ccol]) + g: the flow's DDSConv input."""
    p = f"dp.flows.{FLOWS[s]}."
    zc = np.asarray(z, dtype=dt)[:, flow_cols(s)[0]]
    return zc[:, None] * _w(T, p + "pre.weight")[:, 0, 0].astype(dt) + _w(T, p + "pre.bias").astype(dt) + np.asarray(g, dtype=dt)


def flow_h(T, s, z, g, dt=np.float64, **variant):
    return ddsconv(T, f"dp.flows.{FLOWS[s]}.convs.", flow_pre(T, s, z, g, dt), dt, **variant)


def flow_h29(T, s, h, dt=np.float64):
    p = f"dp.flows.{FLOWS[s]}."
    return conv1x1(h, T[p + "proj.weight"], T[p + "proj.bias"], dt)


def spline_logits(h29, H):
    """(uw, uh, ud) of the spline from proj's output: the engine divides the width / height logits by sqrt(H) in fp32, so
    the float64 reference starts from those fp32 products (one rounding, also the fp32 graph's)."""
    h = np.asarray(h29, dtype=np.float32)
    inv = np.float32(1.0) / np.sqrt(np.float32(H))
    return ((h[:, :NB] * inv).astype(np.float64), (h[:, NB:2 * NB] * inv).astype(np.float64),
            h[:, 2 * NB:3 * NB - 1].astype(np.float64))


# --------------------------------------------------------------------------- rational-quadratic spline (float64)
def _knots(uw, uh, ud):
    """cumwidths, cumheights [n][NB+1] and derivatives [n][NB+1] of transforms.unconstrained_rational_quadratic_spline."""
    uw, uh, ud = (np.atleast_2d(np.asarray(a, dtype=np.float64)) for a in (uw, uh, ud))

    def cum(u):
        e = np.exp(u - u.max(axis=1, keepdims=True))
        w = MIN_W + (1 - MIN_W * NB) * e / e.sum(axis=1, keepdims=True)
        c = np.concatenate([np.zeros((u.shape[0], 1)), np.cumsum(w, axis=1)], axis=1)
        c = 2 * TAIL * c - TAIL
        c[:, 0], c[:, -1] = -TAIL, TAIL
        return c
    const = math.log(math.expm1(1 - MIN_D))
    udp = np.concatenate([np.full((ud.shape[0], 1), const), ud, np.full((ud.shape[0], 1), const)], axis=1)
    d = MIN_D + np.logaddexp(0.0, udp)
    return cum(uw), cum(uh), d


def _bin(loc, x):
    bl = loc.copy()
    bl[:, -1] += 1e-6
    return np.clip((x[:, None] >= bl).sum(axis=1) - 1, 0, NB - 1)


def rqs_inverse(y, uw, uh, ud):
    """Inverse spline per row (linear tails: identity outside [-5, 5]).  y [n]; logits [n][NB], [n][NB], [n][NB-1]."""
    y = np.asarray(y, dtype=np.float64)
    out = y.copy()
    inside = (y >= -TAIL) & (y <= TAIL)
    if not inside.any():
        return out
    cw, ch, d = _knots(np.atleast_2d(uw)[inside], np.atleast_2d(uh)[inside], np.atleast_2d(ud)[inside])
    x = y[inside]
    k = _bin(ch, x)
    r = np.arange(len(x))
    w, h = cw[r, k + 1] - cw[r, k], ch[r, k + 1] - ch[r, k]
    delta = h / w
    t = x - ch[r, k]
    d0 = d[r, k]
    e = d0 + d[r, k + 1] - 2 * delta
    a = t * e + h * (delta - d0)
    b = h * d0 - t * e
    c = -delta * t
    disc = np.maximum(b * b - 4 * a * c, 0.0)
    out[inside] = (2 * c) / (-b - np.sqrt(disc)) * w + cw[r, k]
    return out


def rqs_forward(x, uw, uh, ud):
    """Forward spline and its slope per row: (y, dy/dx) (identity, slope 1, outside [-5, 5])."""
    x = np.asarray(x, dtype=np.float64)
    y, slope = x.copy(), np.ones_like(x)
    inside = (x >= -TAIL) & (x <= TAIL)
    if not inside.any():
        return y, slope
    cw, ch, d = _knots(np.atleast_2d(uw)[inside], np.atleast_2d(uh)[inside], np.atleast_2d(ud)[inside])
    xi = x[inside]
    k = np.clip((xi[:, None] >= cw[:, :-1]).sum(axis=1) - 1, 0, NB - 1)
    r = np.arange(len(xi))
    w, h = cw[r, k + 1] - cw[r, k], ch[r, k + 1] - ch[r, k]
    delta = h / w
    th = (xi - cw[r, k]) / w
    d0, d1 = d[r, k], d[r, k + 1]
    den = delta + (d0 + d1 - 2 * delta) * th * (1 - th)
    y[inside] = ch[r, k] + h * (delta * th ** 2 + d0 * th * (1 - th)) / den
    slope[inside] = delta ** 2 * (d1 * th ** 2 + 2 * delta * th * (1 - th) + d0 * (1 - th) ** 2) / den ** 2
    return y, slope


def ea_inverse(z0, m0, logs0):
    """ElementwiseAffine^-1 of the first channel: logw = (z0 - m0) exp(-logs0)."""
    return (np.asarray(z0, dtype=np.float64) - m0) * math.exp(-logs0)


# --------------------------------------------------------------------------- fp32 emulation of spline_kernel
def _fma(a, b, c):
    """fp32 fused multiply-add (the exact product fits a double; one rounding of the sum, then to fp32)."""
    f = lambda v: np.asarray(v, dtype=np.float64)
    return (f(a) * f(b) + f(c)).astype(np.float32)


def spline_fp32(y, uw, uh, ud, fused=True, defect=None):
    """spline_kernel (kernels_misc.cu) one scalar operation at a time in float32, for rows of logits already scaled.
    fused: contract a*b + c into an FMA where nvcc may (the knot affine maps, a, b, disc = b*b - 4ac with b^2 fused, the
    output affine map).  defect: None, or a deliberately wrong kernel for the bound test: "swap_d" (d_k and d_{k+1}
    exchanged), "e_1.9" (1.9 delta for 2 delta in e).  Returns (out, disc, fp32 cumheights [n][NB+1]), disc before the
    clamp at 0 (NaN outside [-5, 5]); out is clamped to [-5, 5] like the kernel's."""
    f = np.float32
    y = np.asarray(y, dtype=f)
    n = len(y)
    uw, uh, ud = (np.atleast_2d(np.asarray(a, dtype=f)) for a in (uw, uh, ud))
    mad = (lambda a, b, c: _fma(a, b, c)) if fused else (lambda a, b, c: (a * b + c).astype(f))

    def cum(u):
        m = u.max(axis=1, keepdims=True)
        e = np.exp(u - m).astype(f)
        s = np.zeros(n, dtype=f)
        for k in range(NB):
            s = (s + e[:, k]).astype(f)
        c = np.zeros(n, dtype=f)
        out = np.empty((n, NB + 1), dtype=f)
        out[:, 0] = -TAIL
        scale = f(1.0) - f(1e-3) * f(NB)
        for k in range(NB):
            wk = mad(scale, (e[:, k] / s).astype(f), f(1e-3))
            c = (c + wk).astype(f)
            out[:, k + 1] = mad(f(2 * TAIL), c, f(-TAIL))
        out[:, NB] = TAIL
        return out

    def softplus(x):
        x = np.asarray(x, dtype=f)
        return np.where(x > f(20), x, np.log1p(np.exp(x).astype(f)).astype(f)).astype(f)
    cw, ch = cum(uw), cum(uh)
    cst = np.log((np.exp(f(1) - f(1e-3)).astype(f) - f(1)).astype(f)).astype(f)
    dv = np.empty((n, NB + 1), dtype=f)
    dv[:, 0] = dv[:, NB] = f(1e-3) + softplus(cst)
    dv[:, 1:NB] = (f(1e-3) + softplus(ud)).astype(f)
    loc = ch.copy()
    loc[:, NB] = (loc[:, NB] + f(1e-6)).astype(f)
    k = np.clip((y[:, None] >= loc).sum(axis=1) - 1, 0, NB - 1)
    r = np.arange(n)
    in_cw, in_ch = cw[r, k], ch[r, k]
    in_w, in_h = (cw[r, k + 1] - in_cw).astype(f), (ch[r, k + 1] - in_ch).astype(f)
    d0, d1 = dv[r, k], dv[r, k + 1]
    if defect == "swap_d":
        d0, d1 = d1, d0
    with np.errstate(all="ignore"):
        delta = (in_h / in_w).astype(f)
        t = (y - in_ch).astype(f)
        e = mad(f(-1.9 if defect == "e_1.9" else -2), delta, (d0 + d1).astype(f))
        a = mad(t, e, (in_h * (delta - d0).astype(f)).astype(f))
        b = mad(-t, e, (in_h * d0).astype(f))
        c = (-delta * t).astype(f)
        disc = mad(b, b, (-(f(4) * a).astype(f) * c).astype(f))
        root = ((f(2) * c).astype(f) / (-b - np.sqrt(np.maximum(disc, f(0))).astype(f)).astype(f)).astype(f)
        out = np.clip(mad(root, in_w, in_cw), f(-TAIL), f(TAIL))
    inside = (y >= -TAIL) & (y <= TAIL)
    return np.where(inside, out, y), np.where(inside, disc, np.nan), ch


def spline_error_bound(y, uw, uh, ud):
    """(float64 inverse of y, per-element bound of the fp32 spline): SPLINE_MULT x the error of the kernel's arithmetic
    emulated on the host + SPLINE_K ulp of TAIL over the forward slope at the float64 output.  Where the root formula
    cancels, which inputs its fp32 error hits depends on the last bits of every intermediate (the contracted and the
    uncontracted evaluation hit different ones), so the emulated error is the largest over both evaluations at y and at
    y +- 1, 2 ulp, each against its own float64 inverse: the size of the formula's error around y, not the luck of one
    evaluation.  y [n] fp32; uw / uh [n][NB] and ud [n][NB-1]: the fp32 logits the kernel uses (width / height logits
    already divided by sqrt(hidden))."""
    y = np.asarray(y, dtype=np.float32)
    uw, uh, ud = (np.asarray(a, dtype=np.float32) for a in (uw, uh, ud))
    ref = rqs_inverse(y.astype(np.float64), uw, uh, ud)
    max_abs = np.zeros_like(ref)
    for step in (-2, -1, 0, 1, 2):
        yo = y.copy()
        for _ in range(abs(step)):
            yo = np.nextafter(yo, np.float32(np.sign(step) * 10))
        ro = rqs_inverse(yo.astype(np.float64), uw, uh, ud)
        for fused in (True, False):
            e = np.abs(spline_fp32(yo, uw, uh, ud, fused)[0].astype(np.float64) - ro)
            max_abs = np.maximum(max_abs, np.where(np.isfinite(e), e, 0.0))
    _, slope = rqs_forward(ref, uw, uh, ud)
    return ref, SPLINE_MULT * max_abs + SPLINE_K * 2.0 ** -24 * TAIL * (1 + 1 / slope)


# --------------------------------------------------------------------------- spline edge cases
def edge_params(rng):
    """(name, uw, uh, ud) of the spline edge parameter sets: all-zero logits, sigma 1 / 3 / 10, saturated bins (logits
    +-50: width / height 0.01), derivative logits >= 20 (softplus's linear branch), <= -30 (d = 1e-3), and a narrow tall
    bin next to d = 1e-3."""
    sets = [("zero", np.zeros(10), np.zeros(10), np.zeros(9))]
    for sg in (1, 3, 10):
        for _ in range(6):
            sets.append((f"sigma{sg}", rng.normal(0, sg, 10), rng.normal(0, sg, 10), rng.normal(0, sg, 9)))
    sat = np.where(np.arange(10) % 3 == 0, 50.0, -50.0)
    sets.append(("saturated", sat, -sat, rng.normal(0, 1, 9)))
    sets.append(("softplus_linear", rng.normal(0, 2, 10), rng.normal(0, 2, 10), 20 + rng.uniform(0, 10, 9)))
    sets.append(("min_derivative", rng.normal(0, 2, 10), rng.normal(0, 2, 10), np.full(9, -30.0)))
    uh = np.full(10, -50.0); uh[4] = 50.0
    uw = np.full(10, 50.0); uw[4] = -50.0
    ud = np.zeros(9); ud[3] = ud[4] = -30.0
    sets.append(("narrow_tall_bin", uw, uh, ud))
    return [(n, *(np.asarray(a, dtype=np.float32) for a in (w, h, d))) for n, w, h, d in sets]


def edge_inputs(ch):
    """Inputs for one parameter set with fp32 knots ch: a dense sweep of [-5, 5], every knot and +-1..4 ulp around it,
    knot - 1e-7 .. 1e-4, and +-5, +-5 +- 1 ulp, +-6, +-inf, NaN."""
    f = np.float32
    xs = [np.linspace(-5, 5, 2001, dtype=f)]
    for k in ch:
        k = f(k)
        up, dn = k, k
        for _ in range(4):
            up, dn = np.nextafter(up, f(10)), np.nextafter(dn, f(-10))
            xs.append(np.array([up, dn], dtype=f))
        xs.append(np.array([k], dtype=f))
        xs.append((k - np.geomspace(1e-7, 1e-4, 16)).astype(f))
    five = f(5)
    xs.append(np.array([five, -five, np.nextafter(five, f(10)), np.nextafter(five, f(0)), np.nextafter(-five, f(-10)),
                        np.nextafter(-five, f(0)), 6, -6, np.inf, -np.inf, np.nan], dtype=f))
    return np.concatenate(xs)
