"""The fused 64-channel ResBlock2 stage kernel (`resblock_tc.cu`) against the same stage built from six layer-wise
bf16x2 conv launches (`sb200_debug_conv_ex`, backend 1), bit for bit: per branch b, x1 = x + conv1(lrelu(x)) and
ys (+)= (x1 + conv2(lrelu(x1))) / 3.  Outputs are compared by a SHA-256 digest of every 128-row tile, so a mismatch names
the tiles that differ.  Cases: segment edges inside the halo of a tile edge at the stage's real row map (granule
128 x 64 rows, seg_mul 64, as the medium voice's second upsampling level) and at arbitrary rows, a launch shorter than
one halo, a nearly empty last tile, and the row counts of one 128-phoneme utterance and of a 32-utterance batch, each at
grid caps 1, 5 and 0.  The host tests check the kernel's plan (shared memory, registers, window rows) through
`sb200_debug_resblock2_plan`."""
import ctypes as C
import hashlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from sonata_b200 import _native as N  # noqa: E402

# the medium voice's ResBlock2 branches: kernel sizes and the dilations of their two convs
KS = (3, 5, 7)
DILS = ((1, 2), (2, 6), (3, 12))
U = 64                                   # rows per frame at the 64-channel stage (upsampling 8 x 8)

# (name, segment lens in frames (seg_mul = U) or rows (seg_mul = 1) or a total row count, gran, seg_mul, grid caps)
CASES = [
    ("edges_in_tile_halos", (37, 2, 36, 90), 128 * U, U, (1, 5, 0)),
    ("edges_at_any_row", (300, 7, 1000, 45, 555), 128, 1, (1, 5, 0)),
    ("shorter_than_one_halo", 30, None, 1, (1, 5, 0)),
    ("nearly_empty_last_tile", 128 * 45 + 3, None, 1, (1, 5, 0)),
    ("one_utterance_rows", (870,), 128 * U, U, (1, 5, 0)),
    ("batch_of_32_rows", (1785,) * 32, 128 * U, U, (1, 5, 0)),
]


def i32(v):
    return (C.c_int32 * len(v))(*v)


def stage_desc():
    return i32(KS), i32([d for pair in DILS for d in pair])


def plan(rows, ks=KS, dils=DILS):
    o = (C.c_int32 * 8)()
    rc = N.lib().sb200_debug_resblock2_plan(rows, len(ks), i32(ks), i32([d for p in dils for d in p]), o)
    return None if rc else list(o)


def test_plan_fits_one_cta_per_sm():
    """Tile of 128 rows; the x window of the new x1 rows: from h2 - h1 = 1 row past the tile's start (k = 3) to
    h2 + h1 = 36 + 9 rows past its end (k = 7); x1 with conv2's 36 halo rows on each side; the saved halos 2 (2 + 12 + 36)
    rows; an 8-slot ring of 8 KB weight images: within the 227 KB of shared memory and the SM's 64 K registers."""
    m, win, x1rows, ring, smem, grid, threads, regs = plan(57344)
    assert (m, win, x1rows, ring) == (128, 128 + 45 - 1, 128 + 2 * 36, 8)
    assert smem == 1024 + ring * 8192 + (win + x1rows + 2 * (2 + 12 + 36)) * 256 + 8 * (2 * ring + 2)
    assert smem <= 227 * 1024
    assert threads == 384 and regs <= 65536
    assert grid == min(plan(57344)[5], (57344 + 127) // 128)
    assert plan(30)[5] == 1 and plan(128 * 45 + 3)[5] == 46


def test_plan_rejects_what_the_kernel_does_not_take():
    """The next tile's 2 h2 halo rows of x1 must be among the tile's 128 new rows: a conv2 halo above 64 rows is not
    taken."""
    assert plan(4096, ks=(7,), dils=((1, 22),)) is None
    assert plan(4096, ks=(7,), dils=((1, 21),)) is not None


def layout(case):
    name, lens, gran, seg_mul, _ = case
    import conv_unit as cu
    if gran is None:
        return lens, [lens], (lens + 255) // 256 * 256
    rows, ends = cu.segment_table(lens, gran, seg_mul)
    return rows, ends, gran


def inputs(case):
    name, _, _, seg_mul, _ = case
    import conv_unit as cu
    rows, ends, gran = layout(case)
    rng = np.random.default_rng(sum(map(ord, name)))
    x = rng.standard_normal((rows, 64), dtype=np.float32)
    x[~cu.valid_rows_mask(rows, ends, gran, seg_mul)] = 0          # gap rows of the input are zero, as the engine keeps them
    ws = [(rng.standard_normal((64, 64, k), dtype=np.float32) / np.float32((64 * k) ** 0.5)) for k in KS for _ in range(2)]
    bs = [rng.standard_normal(64, dtype=np.float32) * np.float32(0.1) for _ in range(2 * len(KS))]
    return x, ws, bs, ends, gran


def layer_wise(case):
    """The stage as run_decoder's layer-wise loop runs it: six conv_tc launches."""
    import conv_unit as cu
    import torch
    x, ws, bs, ends, gran = inputs(case)
    seg_mul = case[3]
    ys = np.zeros_like(x)
    xt = torch.from_numpy(x)
    for b, (k, (d1, d2)) in enumerate(zip(KS, DILS)):
        x1 = np.zeros_like(x)
        msg = cu.run_conv(1, xt, torch.from_numpy(ws[2 * b]), torch.from_numpy(bs[2 * b]), d1, 0.1, 0, xt, 1.0,
                          seg_end=ends, gran=gran, seg_mul=seg_mul, y0=x1)
        assert not msg, msg
        x1t = torch.from_numpy(x1)
        msg = cu.run_conv(1, x1t, torch.from_numpy(ws[2 * b + 1]), torch.from_numpy(bs[2 * b + 1]), d2, 0.1, 0, x1t,
                          1.0 / len(KS), seg_end=ends, gran=gran, seg_mul=seg_mul, y0=ys, acc0=b > 0)
        assert not msg, msg
    return ys


def fused(case):
    x, ws, bs, ends, gran = inputs(case)
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    w = np.ascontiguousarray(np.concatenate([a.ravel() for a in ws]))
    b = np.ascontiguousarray(np.concatenate(bs))
    y = np.full_like(x, np.nan)
    ks, dils = stage_desc()
    err = N.sb200_error()
    rc = N.lib().sb200_debug_resblock2_stage(0, fp(x), x.shape[0], len(KS), ks, dils, fp(w), fp(b),
                                             i32(np.asarray(ends, dtype=np.int32).tolist()), gran, case[3], fp(y),
                                             C.byref(err))
    assert rc == 0, C.string_at(err.message).decode() if err.message else rc
    return y


def digests(a, rows=128):
    """SHA-256 of every `rows`-row block of `a`, as "<block>:<hex>" strings."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    return np.array([f"{t // rows}:{hashlib.sha256(a[t:t + rows].tobytes()).hexdigest()}" for t in range(0, len(a), rows)])


@pytest.fixture
def grid_cap(lib_built):
    lib = N.lib()
    prev = lib.sb200_debug_conv_grid_cap(0)
    yield lambda cap: lib.sb200_debug_conv_grid_cap(cap)
    lib.sb200_debug_conv_grid_cap(prev)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fused_stage_keeps_the_bits_of_six_convs(case, grid_cap):
    grid_cap(0)
    want = digests(layer_wise(case))
    for cap in case[4]:
        grid_cap(cap)
        got = digests(fused(case))
        bad = [t.split(":")[0] for t, u in zip(got, want) if t != u]
        assert not bad, (case[0], cap, "tiles", bad[:20], len(bad))
