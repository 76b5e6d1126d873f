"""Staged epilogue operands of the bf16x2 conv kernel (`conv_tc.cu`) on the shapes `test_conv_ws_gpu.py` lacks: the
64-channel k = 7, dilation 12 ResBlock conv with residual, accumulation and gap rows at seg_mul 4 (the one whose staging
fills the 227 KB opt-in limit), and the same with a nearly empty last tile, each at grid caps 1, 5 and 0.  Every output
must keep the bits of the kernel before staging.  Fixture: `tests/golden/conv_tc/conv_tc_staged_outputs.npz`
(generator alongside), per-tile SHA-256 digests written by that kernel's build; inputs come from each case's seed."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_conv_ws_gpu as W  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "conv_tc", "conv_tc_staged_outputs.npz")
ACT_NONE = 0

# (name, segment lens (or total rows), gran, seg_mul, cin, cout, k, dil, slope, act, use_res, scale, acc, split)
CASES = [
    ("nt64_k7_dil12_res_acc_gaps", (1300, 2, 1900, 77), 512, 4, 64, 64, 7, 12, 0.1, ACT_NONE, True, 1 / 3, True, None),
    ("nt64_k7_dil12_res_acc_nearly_empty_last_tile", 128 * 70 + 1, None, 1, 64, 64, 7, 12, 0.1, ACT_NONE, True, 1 / 3,
     True, None),
]


def test_cases_are_staged_at_64_columns():
    import conv_unit as cu
    import ctypes as C
    from sonata_b200 import _native as N
    for name, lens, gran, seg_mul, cin, cout, k, dil, slope, act, use_res, scale, acc, split in CASES:
        rows = lens if gran is None else cu.segment_table(lens, gran, seg_mul)[0]
        b = C.c_int32(0)
        assert N.lib().sb200_debug_plan_staging(rows, cin, cout, k, dil, act, int(use_res), int(acc), C.byref(b)) == 0
        assert W.plan(rows, cin, cout, k, dil, act, int(use_res), int(acc))[0] == 64 and b.value == 2 * 128 * 64 * 4, name


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_staged_conv_keeps_the_bits_of_the_previous_kernel(case, grid_cap):
    want = np.load(GOLDEN)["conv_" + case[0]]
    for cap in (1, 5, 0):
        grid_cap(cap)
        got = W.digests(W.run_case(case))
        assert np.array_equal(got, want), (case[0], cap, "output:tile", W.mismatches(got, want))


grid_cap = W.grid_cap
