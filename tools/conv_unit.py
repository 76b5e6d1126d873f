"""Kernel unit check: one convolution through a backend vs torch conv1d (fp64).
Usage: python tools/conv_unit.py <backend> [quick | i,j,...]

Backends: 0 = conv_simt.cu (fp32 CUDA cores), 1 = conv_tc.cu (wgmma bf16x2), 2 = conv_tf.cu (wgmma 3xTF32, chunk-flushed).
On the wgmma kernels a CTA computes 128-row tiles of NT columns.  NT is the width of the voice's weight image, or a
32-column multiple part of it when the launch is small: the planners narrow the tile while m-tiles x (cout / NT) <= SMs
(`narrow_edge`).  The hook pads a launch to a multiple of 256 rows, like the engine's segment tables."""
import ctypes as C
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sonata_b200 import _native as N  # noqa: E402


def _sms():
    if torch.cuda.is_available():
        return torch.cuda.get_device_properties(0).multi_processor_count
    return 132                          # H100 SXM, what the planners assume without a device


SMS = _sms()


def narrow_edge(cout, nt):
    """Largest launch (rows, a multiple of the hook's 256-row padding) whose m-tiles x (cout / nt) column tiles still fit
    one per SM: up to it the planners may take nt-column tiles, one row more and they may not."""
    return SMS // (cout // nt) // 2 * 256


def valid_rows_mask(rows, seg_end, gran, seg_mul):
    q = np.arange(rows)
    return q < np.asarray(seg_end, dtype=np.int64)[q // gran] * seg_mul


def segment_table(lens, gran, seg_mul=1, gap=8):
    """Engine-style layout of segments of `lens` (granule-level rows, i.e. frames when seg_mul > 1): each starts on a
    granule, at least `gap` zero rows apart.  Returns (rows, seg_end per granule) at the launch's row level."""
    g = gran // seg_mul                 # granule in segment-table units
    ends, cur = [], 0
    for n in lens:
        span = (n + gap + g - 1) // g * g
        ends += [cur + n] * (span // g)
        cur += span
    return cur * seg_mul, ends


def conv_ref(x, w, b, dil, slope=1.0, act=0, res=None, scale=1.0):
    """fp64 reference of the epilogue before masking / accumulation: scale * (act(bias + conv(lrelu(x))) + res)."""
    k = w.shape[2]
    xin = torch.where(x > 0, x, x * slope).double()
    dev = "cuda" if torch.cuda.is_available() else "cpu"     # the fp64 reference of the big cases takes minutes on host cores
    ref = F.conv1d(xin.T[None].to(dev), w.double().to(dev), b.double().to(dev), dilation=dil, padding=dil * (k - 1) // 2)[0].T.cpu()
    if act == 1:
        ref = torch.relu(ref)
    if act == 2:
        ref = torch.tanh(ref[:, 0::2]) * torch.sigmoid(ref[:, 1::2])
    if res is not None:
        ref = ref + res.double()
    return ref * scale


def run_conv(backend, x, w, b, dil, slope=1.0, act=0, res=None, scale=1.0, seg_end=None, gran=None, seg_mul=1,
             y0=None, acc0=False, split=None, y1=None, acc1=False):
    """One launch through sb200_debug_conv_ex; y0 / y1 are updated in place (numpy fp32).  Returns "" or the error."""
    rows, cin = x.shape
    cout, _, k = w.shape
    if seg_end is None:
        seg_end, gran = [rows], (rows + 255) // 256 * 256
    fp = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_float))
    ends = np.ascontiguousarray(seg_end, dtype=np.int32)
    xn, wn, bn = (np.ascontiguousarray(t.numpy(), dtype=np.float32) for t in (x, w, b))
    rn = None if res is None else np.ascontiguousarray(res.numpy(), dtype=np.float32)
    err = N.sb200_error()
    rc = N.lib().sb200_debug_conv_ex(0, backend, fp(xn), rows, cin, fp(wn), fp(bn), cout, k, dil, slope, act, fp(rn), scale,
                                     ends.ctypes.data_as(C.POINTER(C.c_int32)), gran, seg_mul, fp(y0), int(acc0),
                                     cout if split is None else split, fp(y1), int(acc1), C.byref(err))
    if rc != 0:
        return C.string_at(err.message).decode() if err.message else f"error {rc}"
    return ""


def _inputs(rows, cin, cout, k, use_res, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, cin, generator=g)
    w = torch.randn(cout, cin, k, generator=g) / (cin * k) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    res = torch.randn(rows, cout, generator=g) if use_res else None
    return g, x, w, b, res


def run_case(backend, rows, cin, cout, k, dil, slope=1.0, act=0, use_res=False, scale=1.0, acc=False, valid=None, seed=0):
    """One segment [0, valid): max |err| of the valid rows against fp64, or (None, message).  Masked rows must come out
    exactly 0 (or keep what they held, under accumulate)."""
    g, x, w, b, res = _inputs(rows, cin, cout, k, use_res, seed)
    valid = rows if valid is None else valid
    x[valid:] = 0
    ycols = cout // 2 if act == 2 else cout
    y0 = torch.randn(rows, ycols, generator=g)
    ref = conv_ref(x, w, b, dil, slope, act, res, scale)
    if acc:
        ref = ref + y0.double()
    y = y0.numpy().copy()
    msg = run_conv(backend, x, w, b, dil, slope, act, res, scale, seg_end=[valid], gran=(rows + 255) // 256 * 256,
                   y0=y, acc0=acc)
    if msg:
        return None, msg
    gap = (y0.numpy()[valid:] if acc else np.zeros_like(y[valid:]))
    if not np.array_equal(y[valid:], gap):
        return float("inf"), ""
    return float(np.abs(y[:valid] - ref.numpy()[:valid]).max()) if valid else 0.0, ""


def run_segments(backend, lens, gran, seg_mul, cin, cout, k, dil, slope=1.0, act=0, use_res=False, scale=1.0, acc=False,
                 seed=0):
    """Several segments with gap rows in one launch (engine row map).  Gap rows of the input are zero, as the engine keeps
    them; the output buffer is seeded non-zero everywhere.  Returns (max |err| over valid rows, gap rows as required)."""
    rows, ends = segment_table(lens, gran, seg_mul)
    valid = torch.from_numpy(valid_rows_mask(rows, ends, gran, seg_mul))
    g, x, w, b, res = _inputs(rows, cin, cout, k, use_res, seed)
    x[~valid] = 0
    ycols = cout // 2 if act == 2 else cout
    y0 = torch.randn(rows, ycols, generator=g)
    ref = conv_ref(x, w, b, dil, slope, act, res, scale)
    if acc:
        ref = ref + y0.double()
    y = y0.numpy().copy()
    msg = run_conv(backend, x, w, b, dil, slope, act, res, scale, seg_end=ends, gran=gran, seg_mul=seg_mul, y0=y, acc0=acc)
    assert not msg, msg
    v = valid.numpy()
    gap_ok = np.array_equal(y[~v], y0.numpy()[~v] if acc else np.zeros_like(y[~v]))
    return float(np.abs(y[v] - ref.numpy()[v]).max()), gap_ok


def run_split(backend, lens, H, k, acc1, seed=0):
    """WaveNet res/skip layer (engine flow layers): columns [0, H) accumulate into y0 (the residual stream), [H, 2H) go to
    y1 (the skip sum, accumulated from the second layer on).  Returns ((err0, gaps0 ok), (err1, gaps1 ok))."""
    gran = 128
    rows, ends = segment_table(lens, gran)
    valid = torch.from_numpy(valid_rows_mask(rows, ends, gran, 1))
    g, x, w, b, _ = _inputs(rows, H, 2 * H, k, False, seed)
    x[~valid] = 0
    y0 = torch.randn(rows, H, generator=g)
    y1 = torch.randn(rows, H, generator=g)
    ref = conv_ref(x, w, b, 1)
    a, c = y0.numpy().copy(), y1.numpy().copy()
    msg = run_conv(backend, x, w, b, 1, seg_end=ends, gran=gran, y0=a, acc0=True, split=H, y1=c, acc1=acc1)
    assert not msg, msg
    v = valid.numpy()
    out = []
    for got, seed_buf, r, acc in ((a, y0, ref[:, :H], True), (c, y1, ref[:, H:], acc1)):
        r = r + seed_buf.double() if acc else r
        gap = seed_buf.numpy()[~v] if acc else np.zeros_like(got[~v])
        out.append((float(np.abs(got[v] - r.numpy()[v]).max()), np.array_equal(got[~v], gap)))
    return out


def tile_width_launches(backend, cin, cout, k, dil, act=0, res=0, acc=0, max_rows=40_000):
    """{tile width: smallest launch (rows) the planner gives that width}, queried in this process (SM count of the device)."""
    widths = {}
    for rows in range(256, max_rows + 1, 256):
        o = (C.c_int32 * 16)()
        if N.lib().sb200_debug_plan(backend, rows, cin, cout, k, dil, act, res, acc, o) != 0:
            break
        widths.setdefault(o[0], rows)
    return widths


# rows, cin, cout, k, dil, slope, act, res, scale, acc, valid
E64, E128, E128W, E256, EG, EG64 = (narrow_edge(64, 32), narrow_edge(128, 32), narrow_edge(128, 64), narrow_edge(256, 32),
                                     narrow_edge(384, 32), narrow_edge(384, 64))
CASES = [
    # one or two m-tiles: the narrowest column tiles; every flow / decoder layer shape, masked tails, accumulate,
    # residual, leaky-ReLU prologue, gate, negative scale
    (256, 32, 32, 1, 1, 1.0, 0, False, 1.0, False, None),
    (256, 32, 32, 3, 1, 0.1, 0, True, 1.0, False, 200),
    (512, 32, 32, 7, 12, 0.1, 0, True, 1 / 3, True, 450),
    (384, 64, 64, 5, 6, 0.1, 0, True, 1.0, False, 300),
    (256, 128, 128, 3, 2, 0.1, 0, True, 1.0, False, None),
    (256, 192, 384, 5, 1, 1.0, 2, False, 1.0, False, 250),
    (256, 192, 384, 1, 1, 1.0, 0, False, 1.0, True, None),
    (256, 192, 96, 1, 1, 1.0, 0, False, -1.0, True, None),
    (384, 256, 256, 11, 5, 0.1, 0, True, 1.0, False, 380),
    (256, 192, 576, 1, 1, 1.0, 0, False, 1.0, False, None),
    (256, 768, 192, 3, 1, 1.0, 0, False, 1.0, False, None),
    (256, 192, 768, 3, 1, 1.0, 1, False, 1.0, False, None),
    # both sides of each narrowing edge: the last launch that still takes narrow tiles (32 / 64 columns of a 64-, 128- or
    # 384-column image, 32 of the k11 layer's 64-column parts) and one 256-row block more, ragged valid rows
    (E64, 64, 64, 7, 12, 0.1, 0, True, 1 / 3, True, E64 - 19),
    (E64 + 45, 64, 64, 7, 12, 0.1, 0, True, 1 / 3, True, E64 + 17),
    (E128, 128, 128, 3, 2, 0.1, 0, True, 1.0, False, None),
    (E128 + 100, 128, 128, 7, 3, 0.1, 1, True, 1.0, False, E128 + 3),
    (E128W, 128, 128, 3, 2, 0.1, 0, True, 1.0, False, E128W - 1),
    (E128W + 1, 128, 128, 3, 2, 0.1, 0, True, 1.0, True, None),
    (EG, 192, 384, 5, 1, 1.0, 2, False, 1.0, False, EG - 80),
    (EG + 1, 192, 384, 5, 1, 1.0, 2, False, 1.0, False, None),
    (EG64 + 128, 192, 384, 1, 1, 1.0, 0, False, 1.0, True, None),
    (E256, 256, 256, 11, 5, 0.1, 0, True, 1.0, False, E256 - 50),
    (E256 + 77, 256, 256, 11, 5, 0.1, 0, True, 1.0, False, None),
    (333, 192, 96, 1, 1, 1.0, 0, True, -1.0, True, 301),
    # many more tiles than SMs (several tiles per CTA): the 32- and 64-channel ResBlock layers of the last
    # decoder stages, every (k, dilation) of ResBlock2 / ResBlock1, ragged tails inside a warp's 32 rows, accumulate /
    # residual / scale, ReLU, no residual
    (SMS * 128 * 3 + 384, 32, 32, 3, 2, 0.1, 0, True, 1.0, False, SMS * 128 * 3 + 300),
    (SMS * 128 * 5, 64, 64, 7, 12, 0.1, 0, True, 1 / 3, True, None),
    (20480, 192, 384, 5, 1, 1.0, 2, False, 1.0, False, 20000),
    (20480 + 128, 192, 384, 1, 1, 1.0, 0, False, 1.0, True, None),
    (300, 32, 32, 3, 2, 0.1, 0, True, 1.0, False, 290),
    (1000, 32, 32, 5, 2, 0.1, 0, True, 1.0, False, 777),
    (1000, 32, 32, 5, 6, 0.1, 0, True, 1 / 3, True, 999),
    (1000, 32, 32, 7, 3, 0.1, 0, True, 1.0, False, None),
    (SMS * 56 * 5 + 17, 32, 32, 7, 12, 0.1, 0, True, 1 / 3, True, SMS * 56 * 5),
    (SMS * 126 * 4 + 100, 32, 32, 3, 1, 0.1, 0, True, 1.0, False, None),
    (SMS * 110 * 3 + 5, 32, 32, 7, 5, 0.1, 1, False, 1.0, False, None),
    (40000, 32, 32, 11, 1, 0.1, 0, True, 1.0, False, None),
    (SMS * 128 * 6 + 77, 32, 32, 3, 1, 0.1, 0, False, 1.0, False, None),
    (SMS * 128 * 4, 32, 32, 11, 5, 0.1, 0, False, 1.0, True, SMS * 128 * 4 - 1000),
    (1000, 64, 64, 11, 5, 0.1, 0, True, 1 / 3, True, 901),
    (SMS * 128 * 7 + 19, 64, 64, 3, 1, 0.1, 0, False, 1.0, False, None),
    # an odd number of 128-row tiles whose last one is nearly empty, the window halo reaching past the array end
    (128 * 301 - 50, 64, 64, 11, 1, 0.1, 0, True, 1 / 3, True, 128 * 301 - 90),
    (128 * 299, 128, 128, 7, 1, 0.1, 0, True, 1.0, False, None),
]

# backend 2 = conv_tf.cu (wgmma 3xTF32 with chunk-flushed accumulation; the text-encoder / duration-predictor
# layers): fp32-class accuracy is the point, so these cases are held to TF_TOL against the fp64 reference (the fp32
# FMA chain of backend 0 measures 2e-6 .. 1e-5 on the same cases).  Shapes: every (cin, cout, k) of the encoder and
# the duration predictor, all three column tiles (96 / 64 / 32), ragged row counts, residual / scale / accumulate /
# masked rows, a leaky-ReLU prologue, both sides of the 192 -> 192 k3 layer's narrowing edge, many-tile launches, and the
# single-utterance shapes (a handful of tiles with a long K loop).
TF_TOL = 1.5e-5
ETF = narrow_edge(192, 32)
TF_CASES = [
    (256, 192, 576, 1, 1, 1.0, 0, False, 1.0, False, None),
    (256, 192, 192, 1, 1, 1.0, 0, False, 1.0, False, None),
    (256, 192, 768, 3, 1, 1.0, 1, False, 1.0, False, None),
    (256, 768, 192, 3, 1, 1.0, 0, False, 1.0, False, None),
    (256, 192, 384, 1, 1, 1.0, 0, False, 1.0, False, None),
    (256, 192, 32, 1, 1, 1.0, 0, False, 1.0, False, None),
    (300, 192, 192, 1, 1, 1.0, 0, True, 0.5, True, 290),
    (640, 64, 64, 3, 1, 1.0, 0, True, 1.0, False, 600),
    (384, 96, 128, 5, 2, 0.1, 0, False, 1.0, False, 380),
    (128, 32, 32, 1, 1, 1.0, 0, False, 1.0, False, 100),
    (256, 416, 64, 3, 1, 1.0, 0, True, 1.0, False, 250),       # odd K-block count, two tiles
    (512, 768, 192, 3, 1, 1.0, 1, False, 1.0, False, 258),      # the single-utterance ffn2 shape (72 stages on 4 CTAs)
    (ETF, 192, 192, 3, 1, 1.0, 0, False, 1.0, False, ETF - 17),
    (ETF + 300, 192, 192, 3, 1, 1.0, 0, False, 1.0, False, ETF + 17),
    (18432, 192, 576, 1, 1, 1.0, 0, False, 1.0, False, 18000),
    (18432, 768, 192, 3, 1, 1.0, 0, True, 1.0, False, None),
    (18432 + 128, 192, 768, 3, 1, 1.0, 1, False, 1.0, False, None),
    # x_low (96 hidden channels): qkv, conv_o, ffn1, ffn2 and proj of the encoder, the duration predictor's 96 -> 96 and
    # 96 -> 32 1x1 layers, the single-utterance ffn2 shape and a many-tile ffn2 with a residual
    (256, 96, 288, 1, 1, 1.0, 0, False, 1.0, False, None),
    (256, 96, 96, 1, 1, 1.0, 0, False, 1.0, False, 201),
    (256, 96, 384, 3, 1, 1.0, 1, False, 1.0, False, None),
    (256, 384, 96, 3, 1, 1.0, 0, False, 1.0, False, 255),
    (256, 96, 192, 1, 1, 1.0, 0, False, 1.0, False, None),
    (300, 96, 96, 1, 1, 1.0, 0, True, 0.5, True, 290),
    (256, 96, 32, 1, 1, 1.0, 0, False, 1.0, False, None),
    (512, 384, 96, 3, 1, 1.0, 0, False, 1.0, False, 258),
    (18432, 384, 96, 3, 1, 1.0, 0, True, 1.0, False, 18000),
]

# Several segments in one launch (the engine's packed batches).  (lens, gran, seg_mul, cin, cout, k, dil, slope, act, res,
# scale, acc): X-level granules of 64 ids with segment ends ragged inside a 128-row tile and a 2-row segment shorter than
# the conv's halo (also at x_low's 96 / 384 channels); Y-level granules of 128 frames; a decoder level at U = 4 / 8 rows per frame (gran = 128 U, seg_mul = U).
SEG_CASES = [
    ((50, 2, 100, 77, 3), 64, 1, 192, 192, 3, 1, 1.0, 0, False, 1.0, False),
    ((50, 2, 100, 77, 3), 64, 1, 192, 576, 1, 1, 1.0, 0, False, 1.0, True),
    ((50, 2, 100, 77, 3), 64, 1, 192, 768, 3, 1, 1.0, 1, True, 0.5, True),
    ((50, 2, 100, 77, 3, 48), 64, 1, 96, 384, 3, 1, 1.0, 1, False, 1.0, False),
    ((50, 2, 100, 77, 3, 48), 64, 1, 384, 96, 3, 1, 1.0, 0, True, 1.0, False),
    ((130, 2, 5, 300), 128, 1, 192, 384, 5, 1, 1.0, 2, False, 1.0, False),
    ((130, 2, 5, 300), 128, 1, 128, 128, 11, 5, 0.1, 0, True, 1 / 3, True),
    ((3, 20, 7, 1), 512, 4, 64, 64, 7, 12, 0.1, 0, True, 1 / 3, True),
    ((3, 20, 7, 1), 1024, 8, 32, 32, 11, 5, 0.1, 0, True, 1.0, False),
]
SPLIT_CASES = [((130, 2, 5, 300), 192, 1), ((77, 640), 192, 1)]      # (lens, H, k): flow res/skip 1x1 layers

# Tile-width invariance: (backend, cin, cout, k, dil, act, res, acc) -- flow / decoder shapes on backend 1, encoder shapes
# on backend 2.
WIDTH_CASES = [
    (1, 192, 384, 5, 1, 2, 0, 0),
    (1, 192, 384, 1, 1, 0, 0, 1),
    (1, 128, 128, 3, 1, 0, 1, 0),
    (1, 256, 256, 11, 1, 0, 0, 0),
    (2, 192, 576, 1, 1, 0, 0, 0),
    (2, 192, 768, 3, 1, 1, 0, 0),
    (2, 768, 192, 3, 1, 0, 0, 0),
]


def width_invariance(backend, cin, cout, k, dil, act, res, acc, seed=3):
    """The same leading rows through one launch per tile width the planner can choose: returns ({width: rows}, list of
    (width, rows compared, bitwise equal)) for every output row whose receptive field lies inside both inputs."""
    launches = tile_width_launches(backend, cin, cout, k, dil, act, res, acc)
    big = max(launches.values())
    g, x, w, b, r = _inputs(big, cin, cout, k, bool(res), seed)
    ycols = cout // 2 if act == 2 else cout
    y0 = torch.randn(big, ycols, generator=g).numpy()
    outs = {}
    for nt, rows in launches.items():
        y = y0[:rows].copy()
        msg = run_conv(backend, x[:rows].contiguous(), w, b, dil, 1.0, act, None if r is None else r[:rows].contiguous(),
                       1.0, y0=y, acc0=bool(acc))
        assert not msg, msg
        outs[nt] = y
    small = min(launches.values())
    keep = small - dil * (k - 1) // 2           # rows below this see only rows of the smaller input
    first = outs[min(outs)]
    return launches, [(nt, keep, bool(np.array_equal(y[:keep], first[:keep]))) for nt, y in outs.items()]


if __name__ == "__main__":
    backend = int(sys.argv[1]) if len(sys.argv) > 1 else 1
    cases = TF_CASES if backend == 2 else CASES
    if len(sys.argv) > 2:      # "quick" = first three cases, or a comma-separated list of case indices
        cases = cases[:3] if sys.argv[2] == "quick" else [cases[int(i)] for i in sys.argv[2].split(",")]
    worst = 0.0
    for c in cases:
        e, msg = run_case(backend, *c)
        print(f"backend {backend} case {c}: " + (f"max|err| {e:.3e}" if e is not None else f"ERROR {msg}"), flush=True)
        if e is None:
            sys.exit(2)
        worst = max(worst, e)
    print("worst", worst)
    sys.exit(0 if worst < (TF_TOL if backend == 2 else 1e-4) else 1)
