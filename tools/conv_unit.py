"""Kernel unit check: one convolution through a backend vs torch conv1d (fp64 on CPU).
Usage: python tools/conv_unit.py <backend> [quick]"""
import ctypes as C
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sonata_b200 import _native as N  # noqa: E402


def run_case(backend, rows, cin, cout, k, dil, slope=1.0, act=0, use_res=False, scale=1.0, acc=False, valid=None, seed=0):
    lib = N.lib()
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, cin, generator=g)
    w = torch.randn(cout, cin, k, generator=g) / (cin * k) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    res = torch.randn(rows, cout, generator=g) if use_res else None
    valid = rows if valid is None else valid
    x[valid:] = 0
    ycols = cout // 2 if act == 2 else cout
    y0 = torch.randn(rows, ycols, generator=g) if acc else torch.zeros(rows, ycols)
    y0[valid:] = 0
    xin = torch.where(x > 0, x, x * slope).double()
    dev = "cuda" if torch.cuda.is_available() else "cpu"     # the fp64 reference of the big cases takes minutes on host cores
    ref = F.conv1d(xin.T[None].to(dev), w.double().to(dev), b.double().to(dev), dilation=dil, padding=dil * (k - 1) // 2)[0].T.cpu()
    if act == 1:
        ref = torch.relu(ref)
    if act == 2:
        ref = torch.tanh(ref[:, 0::2]) * torch.sigmoid(ref[:, 1::2])
    if res is not None:
        ref = ref + res.double()
    ref = ref * scale
    if acc:
        ref = ref + y0.double()
    ref[valid:] = 0
    y = y0.clone().contiguous().numpy()
    xn, wn, bn = x.contiguous().numpy(), w.contiguous().numpy(), b.contiguous().numpy()
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    rn = None if res is None else res.contiguous().numpy()
    err = N.sb200_error()
    rc = lib.sb200_debug_conv(0, backend, fp(xn), rows, cin, fp(wn), fp(bn), cout, k, dil, slope, act,
                              None if rn is None else fp(rn), scale, 1 if acc else 0, fp(y), valid, C.byref(err))
    if rc != 0:
        msg = C.string_at(err.message).decode() if err.message else ""
        return None, msg
    e = float(np.abs(y - ref.numpy()).max())
    return e, ""


CASES = [
    # rows, cin, cout, k, dil, slope, act, res, scale, acc, valid
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
    # persistent multi-tile paths: several tiles per CTA on both half-pipelines (resident and ring weights)
    (148 * 128 * 3 + 384, 32, 32, 3, 2, 0.1, 0, True, 1.0, False, 148 * 128 * 3 + 300),
    (148 * 128 * 5, 64, 64, 7, 12, 0.1, 0, True, 1 / 3, True, None),
    (20480, 192, 384, 5, 1, 1.0, 2, False, 1.0, False, 20000),
    (20480 + 128, 192, 384, 1, 1, 1.0, 0, False, 1.0, True, None),
    (9 * 148 * 128 // 4, 128, 128, 3, 2, 0.1, 0, True, 1.0, False, None),
    # 32-channel layers (TMA-staged epilogue, cat mode): every (k, dilation) of ResBlock2 / ResBlock1, ragged tails,
    # accumulate / residual / scale, many tiles per CTA on both accumulator stages
    (300, 32, 32, 3, 2, 0.1, 0, True, 1.0, False, 290),
    (1000, 32, 32, 5, 2, 0.1, 0, True, 1.0, False, 777),
    (1000, 32, 32, 5, 6, 0.1, 0, True, 1 / 3, True, 999),
    (1000, 32, 32, 7, 3, 0.1, 0, True, 1.0, False, None),
    (148 * 56 * 5 + 17, 32, 32, 7, 12, 0.1, 0, True, 1 / 3, True, 148 * 56 * 5),
    (148 * 126 * 4 + 100, 32, 32, 3, 1, 0.1, 0, True, 1.0, False, None),
    (148 * 110 * 3 + 5, 32, 32, 7, 5, 0.1, 1, False, 1.0, False, None),
    (40000, 32, 32, 11, 1, 0.1, 0, True, 1.0, False, None),
    # TMA-staged epilogue (conv_tc MODE 2) with nothing to fetch: the staging tile is rewritten every tile, so the
    # agent's "store has been read out" signal is the only thing that orders it (regression: WAR race)
    (148 * 128 * 6 + 77, 32, 32, 3, 1, 0.1, 0, False, 1.0, False, None),
    (148 * 128 * 4, 32, 32, 11, 5, 0.1, 0, False, 1.0, True, 148 * 128 * 4 - 1000),
    # coalesced epilogue (conv_tc MODE 1: 64- / 96- / 128-channel outputs turned through shared memory): ragged row
    # counts inside a warp's 32 rows, gap rows under accumulate, ReLU, negative scale, 3 column chunks
    (1000, 64, 64, 11, 5, 0.1, 0, True, 1 / 3, True, 901),
    (148 * 128 * 2 + 45, 128, 128, 7, 3, 0.1, 1, True, 1.0, False, 148 * 128 * 2),
    (333, 192, 96, 1, 1, 1.0, 0, True, -1.0, True, 301),
    (148 * 128 * 7 + 19, 64, 64, 3, 1, 0.1, 0, False, 1.0, False, None),
    # streamed weights + TMA-staged epilogue + tile pairs with an ODD number of m-tiles: the last pair's second member lies
    # wholly past the end of the array (loads zero-filled, its stores clipped by the tensor map)
    (128 * 301 - 50, 64, 64, 11, 1, 0.1, 0, True, 1 / 3, True, 128 * 301 - 90),
    (128 * 299, 128, 128, 7, 1, 0.1, 0, True, 1.0, False, None),
]

# backend 2 = conv_tf.cu (wgmma 3xTF32 with chunk-flushed accumulation; the text-encoder / duration-predictor
# layers): fp32-class accuracy is the point, so these cases are held to TF_TOL against the fp64 reference (the fp32
# FMA chain of backend 0 measures 2e-6 .. 1e-5 on the same cases).  Shapes: every (cin, cout, k) of the encoder and
# the duration predictor, all three column tiles (96 / 64 / 32), ragged row counts (odd number of 128-row tiles in
# the last pair), residual / scale / accumulate / masked rows, a leaky-ReLU prologue, multi-tile persistent runs, and the
# single-utterance shapes (a handful of tiles with a long K loop).
TF_TOL = 1.5e-5
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
    (148 * 256 * 2 + 300, 192, 192, 3, 1, 1.0, 0, False, 1.0, False, 148 * 256 * 2 + 17),
    (18432, 192, 576, 1, 1, 1.0, 0, False, 1.0, False, 18000),
    (18432, 768, 192, 3, 1, 1.0, 0, True, 1.0, False, None),
    (18432 + 128, 192, 768, 3, 1, 1.0, 1, False, 1.0, False, None),
]

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
