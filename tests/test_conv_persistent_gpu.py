"""The persistent bf16x2 conv kernel (`conv_tc.cu`): each CTA walks a static list of tiles, so the bits of every output
must not depend on how many CTAs share the work.  Each shape runs with one CTA per column tile walking every m-tile,
with a few CTAs whose count does not divide the m-tiles, and with the planner's full grid (`sb200_debug_conv_grid_cap`),
and the three results must be equal bit for bit.  The host test checks the plan's grid / residency / occupancy slots."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from sonata_b200 import _native as N  # noqa: E402

SMS = 132                       # the planner assumes an H100 SXM where no device is visible
SMEM_PER_SM = 228 * 1024
ACT_NONE, ACT_GATE = 0, 2


def plan(rows, cin, cout, k, dil, act=ACT_NONE, res=0, acc=0):
    o = (C.c_int32 * 16)()
    assert N.lib().sb200_debug_plan(1, rows, cin, cout, k, dil, act, res, acc, o) == 0
    return list(o)


def test_plan_grid_residency_and_occupancy_slots():
    shapes = [(32, 32, 7, 12, ACT_NONE, 1, 0), (32, 32, 3, 1, ACT_NONE, 1, 1), (64, 64, 7, 6, ACT_NONE, 1, 0),
              (128, 128, 7, 3, ACT_NONE, 1, 1), (256, 256, 11, 5, ACT_NONE, 1, 0), (192, 384, 5, 1, ACT_GATE, 0, 0),
              (192, 384, 1, 1, ACT_NONE, 0, 1), (96, 192, 1, 1, ACT_NONE, 0, 0)]
    for lay in shapes:
        cin = lay[0]
        for rows in (100, 900, 20_000, 460_000, 14_700_000):
            p = plan(rows, *lay)
            nt, wnt, mt, ntn, stages, smem, win, grid, resident, per_sm = p[:10]
            assert p[10:] == [0] * 6, (lay, rows, p)
            assert resident == int(cin // 32 <= stages), (lay, rows, p)
            assert per_sm >= 1 and per_sm * (smem + 1024) <= SMEM_PER_SM, (lay, rows, p)
            assert grid % ntn == 0 and ntn <= grid <= mt * ntn, (lay, rows, p)
            if mt * ntn <= SMS * per_sm:
                assert grid == mt * ntn, (lay, rows, p)        # one tile per CTA
            else:
                assert SMS * per_sm - ntn < grid <= SMS * per_sm, (lay, rows, p)
    # the hot ResBlock layers: the 32- and 64-channel ones keep their weights resident, the 128-channel one streams them
    assert plan(14_700_000, 32, 32, 7, 12, ACT_NONE, 1, 0)[8] == 1
    assert plan(3_700_000, 64, 64, 7, 6, ACT_NONE, 1, 0)[8] == 1
    assert plan(460_000, 128, 128, 7, 3, ACT_NONE, 1, 0)[8] == 0


@pytest.fixture
def grid_cap(lib_built):
    lib = N.lib()
    prev = lib.sb200_debug_conv_grid_cap(0)
    yield lambda cap: lib.sb200_debug_conv_grid_cap(cap)
    lib.sb200_debug_conv_grid_cap(prev)


def _inputs(rows, cin, cout, k, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, cin, generator=g)
    w = torch.randn(cout, cin, k, generator=g) / (cin * k) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    res = torch.randn(rows, cout, generator=g)
    return x, w, b, res, torch.randn(rows, cout, generator=g).numpy()


# (name, lens or rows, gran, seg_mul, cin, cout, k, dil, slope, act, use_res, scale, acc)
CASES = [
    ("resident_k7_res_acc_gaps", (700, 3, 1500, 260), 128, 1, 32, 32, 7, 12, 0.1, ACT_NONE, True, 1 / 3, True),
    ("resident_64_res_gaps", (130, 2, 900, 77), 512, 4, 64, 64, 5, 6, 0.1, ACT_NONE, True, 1.0, False),
    ("streamed_128_res", (1000, 5, 2200), 128, 1, 128, 128, 7, 3, 0.1, ACT_NONE, True, 1.0, False),
    ("streamed_gate", (800, 2300), 128, 1, 192, 384, 5, 1, 1.0, ACT_GATE, False, 1.0, False),
    ("nearly_empty_last_tile", 128 * 45 + 3, None, 1, 32, 32, 3, 1, 0.1, ACT_NONE, True, 1.0, True),
    ("nearly_empty_last_tile_streamed", 128 * 29 + 1, None, 1, 128, 128, 3, 2, 0.1, ACT_NONE, False, 1.0, True),
]


def _run(case, cap):
    import conv_unit as cu
    import torch
    name, lens, gran, seg_mul, cin, cout, k, dil, slope, act, use_res, scale, acc = case
    if gran is None:
        rows, ends, gran = lens, [lens], (lens + 255) // 256 * 256
    else:
        rows, ends = cu.segment_table(lens, gran, seg_mul)
    valid = cu.valid_rows_mask(rows, ends, gran, seg_mul)
    x, w, b, res, y0 = _inputs(rows, cin, cout, k, seed=len(name))
    x[torch.from_numpy(~valid)] = 0
    y = np.ascontiguousarray(y0[:, : (cout // 2 if act == ACT_GATE else cout)])
    msg = cu.run_conv(1, x, w, b, dil, slope, act, res if use_res else None, scale, seg_end=ends, gran=gran,
                      seg_mul=seg_mul, y0=y, acc0=acc)
    assert not msg, msg
    return y, valid


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_bits_do_not_depend_on_the_grid(case, grid_cap):
    cin, cout, k = case[4], case[5], case[6]
    out = {}
    for cap in (1, 5, 0):       # one CTA per column tile; 5 CTAs (or one per column tile, if more); the full grid
        grid_cap(cap)
        out[cap], valid = _run(case, cap)
    grid_cap(0)
    for cap in (1, 5):
        assert np.array_equal(out[cap], out[0]), (case[0], cap)
    # gap rows: exact zeros, or the accumulated buffer's prior contents
    y0 = _inputs(len(valid), cin, cout, k, seed=len(case[0]))[4][:, : out[0].shape[1]]
    gap = y0[~valid] if case[12] else np.zeros_like(out[0][~valid])
    assert np.array_equal(out[0][~valid], gap), case[0]


@pytest.mark.gpu
def test_split_outputs_do_not_depend_on_the_grid(grid_cap):
    """The flow's res/skip layer: columns [0, H) accumulate into y0, [H, 2H) into y1."""
    import conv_unit as cu
    import torch
    outs = []
    for cap in (1, 3, 0):
        grid_cap(cap)
        rows, ends = cu.segment_table((130, 2, 5, 900), 128)
        valid = cu.valid_rows_mask(rows, ends, 128, 1)
        x, w, b, _, y1 = _inputs(rows, 192, 384, 1, seed=7)
        x[torch.from_numpy(~valid)] = 0
        a = np.ascontiguousarray(y1[:, :192])
        c = np.ascontiguousarray(y1[:, 192:])
        assert not cu.run_conv(1, x, w, b, 1, seg_end=ends, gran=128, y0=a, acc0=True, split=192, y1=c, acc1=True)
        outs.append((a, c))
    grid_cap(0)
    for a, c in outs[:2]:
        assert np.array_equal(a, outs[2][0]) and np.array_equal(c, outs[2][1])


@pytest.mark.gpu
def test_synthesis_does_not_depend_on_the_grid(voice_paths, grid_cap):
    """A whole utterance batch: every conv_tc launch of the flow, conv_pre, the phase-fused ConvTranspose layers and the
    ResBlocks, run on 1 CTA per column tile, 7 CTAs and the full grid."""
    import sonata_b200
    from sonata_b200 import PiperSynthesisConfig, workload
    m = sonata_b200.from_config_path(voice_paths["medium"], device=0)
    try:
        m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.0, 1.0, 0.0))
        batches = [workload.synthetic_ids(n, utt=90 + i) for i, n in enumerate((40, 9))]
        wavs = {}
        for cap in (0, 7, 1):
            grid_cap(cap)
            wavs[cap] = [a.samples.as_slice().copy() for a in m.infer_batch_with_values(batches)]
        grid_cap(0)
    finally:
        m.close()
    for cap in (7, 1):
        for got, ref in zip(wavs[cap], wavs[0]):
            assert np.array_equal(np.asarray(got), np.asarray(ref)), cap
