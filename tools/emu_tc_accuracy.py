"""CPU emulation of tensor-core accumulation error, to decide whether the text encoder / duration predictor can leave
the fp32 CUDA cores (round-2 planning; see DESIGN.md §4: `ceil(exp(logw))` is a cliff).

Model (to be checked against a run of tools/conv_unit.py on the target GPU):
  * operands are rounded to the MMA's input format (bf16: 8 significant bits, tf32: 11) and split v = hi + lo;
  * one MMA adds an EXACT partial sum of its K-step (16 products for bf16, 8 for tf32) to the fp32 accumulator and the
    accumulator is rounded TOWARD ZERO (`--acc rn` switches to round-to-nearest for comparison);
  * products accumulate in the order hi*hi, lo*hi, hi*lo per K-step, like conv_tc.cu issues them;
  * `chunk` > 0: the accumulator is flushed every `chunk` K-steps into an fp32 round-to-nearest sum (what an
    `mma.sync` kernel with register accumulators could do for free).

Usage:  python tools/emu_tc_accuracy.py            (prints a table; pure numpy, ~1 minute)
The attention's P.V contraction is emulated by tests/att_reference.py (emulated_pv_errors) on the synthetic voice.
"""
import argparse

import numpy as np


def round_to_bits(x: np.ndarray, bits: int) -> np.ndarray:
    """Round-to-nearest-even of fp32 values to `bits` significant bits (bf16: 8, tf32: 11), result in fp32."""
    x = np.asarray(x, dtype=np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    drop = 24 - bits
    half = (1 << (drop - 1)) - 1
    u = u + half + ((u >> drop) & 1)
    u = (u >> drop) << drop
    return (u & 0xFFFFFFFF).astype(np.uint32).view(np.float32)


def to_f32(x64: np.ndarray, mode: str) -> np.ndarray:
    y = x64.astype(np.float32)
    if mode == "rn":
        return y
    over = np.abs(y.astype(np.float64)) > np.abs(x64)          # RN went away from zero: step back
    return np.where(over, np.nextafter(y, np.float32(0)), y).astype(np.float32)


def emulate(x, w, fmt, acc_mode, chunk, products=("hh", "lh", "hl")):
    """x [M,K], w [K,N] fp32 -> emulated tensor-core result [M,N] fp32.  `products`: which of the split products
    (x part, w part) each K-step issues, in order; ("hh",) is a single unsplit MMA."""
    bits, kstep = (8, 16) if fmt == "bf16" else (11, 8)
    xh = round_to_bits(x, bits); xl = round_to_bits(x - xh, bits)
    wh = round_to_bits(w, bits); wl = round_to_bits(w - wh, bits)
    parts = {"h": (xh, wh), "l": (xl, wl)}
    pairs = [(parts[p[0]][0], parts[p[1]][1]) for p in products]
    M, K = x.shape
    N = w.shape[1]
    total = np.zeros((M, N), dtype=np.float32)
    acc = np.zeros((M, N), dtype=np.float32)
    steps = 0
    for k0 in range(0, K, kstep):
        sl = slice(k0, k0 + kstep)
        for a, b in pairs:
            part = a[:, sl].astype(np.float64) @ b[sl].astype(np.float64)      # exact enough: 16 products in fp64
            acc = to_f32(acc.astype(np.float64) + part, acc_mode)
        steps += 1
        if chunk and steps % chunk == 0:
            total = (total + acc).astype(np.float32)                           # fp32 RN add in registers
            acc = np.zeros_like(acc)
    return (total + acc).astype(np.float32) if chunk else acc


def fp32_fma(x, w):
    acc = np.zeros((x.shape[0], w.shape[1]), dtype=np.float32)
    for k in range(x.shape[1]):                                                # sequential fp32 FMA chain
        acc = (acc.astype(np.float64) + x[:, k:k + 1].astype(np.float64) * w[k:k + 1].astype(np.float64)).astype(np.float32)
    return acc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=192)
    ap.add_argument("--n", type=int, default=48)
    ap.add_argument("--acc", default="rz", choices=["rz", "rn"])
    args = ap.parse_args()
    rng = np.random.default_rng(7)
    print(f"accumulator rounding model: {args.acc};  errors are max |y - y_fp64| with |y| ~ 1")
    print(f"{'K':>6s} {'fp32 FMA':>10s} {'bf16x2':>10s} {'bf16x2 c4':>10s} {'3xTF32':>10s} {'3xTF32 c8':>10s} {'3xTF32 c4':>10s}")
    for K in (192, 576, 768, 2304, 2816):
        x = rng.standard_normal((args.m, K)).astype(np.float32)
        w = (rng.standard_normal((K, args.n)) / np.sqrt(K)).astype(np.float32)
        ref = x.astype(np.float64) @ w.astype(np.float64)
        row = [np.abs(fp32_fma(x, w) - ref).max(),
               np.abs(emulate(x, w, "bf16", args.acc, 0) - ref).max(),
               np.abs(emulate(x, w, "bf16", args.acc, 4) - ref).max(),
               np.abs(emulate(x, w, "tf32", args.acc, 0) - ref).max(),
               np.abs(emulate(x, w, "tf32", args.acc, 8) - ref).max(),
               np.abs(emulate(x, w, "tf32", args.acc, 4) - ref).max()]
        print(f"{K:6d} " + " ".join(f"{e:10.2e}" for e in row), flush=True)


if __name__ == "__main__":
    main()
