"""Writes conv_tc_staged_outputs.npz, the fixture of tests/test_conv_staged_gpu.py: for each seeded case there (one
launch of the bf16x2 conv kernel), a SHA-256 digest of every 128-row tile of every output.  The inputs are not stored:
each case regenerates them from its seed with numpy's PCG64 generator.  `source` records which build wrote the digests.

The committed fixture was written by the build of commit 7281c9b, the kernel before staged epilogue operands, on an
H100:

    SB200_LIB=/path/to/that/libsonata_b200.so \\
        python tests/golden/conv_tc/make_conv_tc_staged_golden.py "commit 7281c9b" [out.npz]
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_conv_staged_gpu as T  # noqa: E402
import test_conv_ws_gpu as W  # noqa: E402
from sonata_b200 import _native as N  # noqa: E402


def main():
    if len(sys.argv) < 2:
        raise SystemExit("usage: make_conv_tc_staged_golden.py SOURCE-DESCRIPTION [out.npz]")
    out = sys.argv[2] if len(sys.argv) > 2 else os.path.join(HERE, "conv_tc_staged_outputs.npz")
    N.lib().sb200_debug_conv_grid_cap(0)
    d = {"source": np.array(sys.argv[1] + " (" + N.LIB_PATH.rsplit("/", 1)[-1] + ")")}
    for c in T.CASES:
        d["conv_" + c[0]] = W.digests(W.run_case(c))
    np.savez_compressed(out, **d)
    for k, v in d.items():
        print(k, v.size)


if __name__ == "__main__":
    main()
