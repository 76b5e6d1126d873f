"""The warp-specialized bf16x2 conv kernel (`conv_tc.cu`) against outputs stored from the build before it: a producer
warpgroup loads and converts the windows while two MMA warpgroups run the MMAs and the epilogue, and every output must
keep its bits.  The shapes cover every tile width (32, 64, 96, 128 columns), resident and streamed weights, residual,
accumulation, split outputs, the gate, a single CTA walking every tile (the ring wraps many times) and nearly empty last
tiles, each at grid caps 1, 5 and 0.  Whole medium and high syntheses cover the phase-fused ConvTranspose layers at
grid caps 0, 7 and 1.  Fixtures: `tests/golden/conv_tc/` (generator alongside): the inputs are regenerated from each
case's seed, and the fixture holds a SHA-256 digest of every 128-row tile of every output (every utterance of a
synthesis), written by the build of the kernel before warp specialization, so a mismatch names the tiles that differ."""
import ctypes as C
import hashlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from sonata_b200 import _native as N  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "conv_tc", "conv_tc_outputs.npz")
ACT_NONE, ACT_GATE = 0, 2

# (name, segment lens (or total rows), gran, seg_mul, cin, cout, k, dil, slope, act, use_res, scale, acc, split)
CASES = [
    ("nt32_resident_res_acc_wraps", (7000, 3, 9000, 260), 128, 1, 32, 32, 7, 12, 0.1, ACT_NONE, True, 1 / 3, True, None),
    ("nt64_resident_res_gaps", (1300, 2, 1900, 77), 512, 4, 64, 64, 5, 6, 0.1, ACT_NONE, True, 1.0, False, None),
    ("nt96_streamed_acc", (5000, 2, 1800), 128, 1, 192, 96, 1, 1, 1.0, ACT_NONE, False, 1.0, True, None),
    ("nt64_streamed_res", (6000, 5, 3200), 128, 1, 128, 128, 7, 3, 0.1, ACT_NONE, True, 1.0, False, None),
    ("nt128_resident_res", (5000, 4100), 128, 1, 64, 128, 3, 1, 0.1, ACT_NONE, True, 0.5, False, None),
    ("nt128_gate", (4000, 2300), 128, 1, 192, 384, 5, 1, 1.0, ACT_GATE, False, 1.0, False, None),
    ("nt128_split_acc", (5200, 2, 1900), 128, 1, 192, 384, 1, 1, 1.0, ACT_NONE, False, 1.0, True, 192),
    ("nearly_empty_last_tile", 128 * 45 + 3, None, 1, 32, 32, 3, 1, 0.1, ACT_NONE, True, 1.0, True, None),
    ("nearly_empty_last_tile_nt128", 128 * 70 + 1, None, 1, 128, 128, 3, 2, 0.1, ACT_NONE, False, 1.0, True, None),
]
SYNTH = [("medium", (40, 9)), ("high", (30, 7))]


def plan(rows, cin, cout, k, dil, act=ACT_NONE, res=0, acc=0):
    o = (C.c_int32 * 16)()
    assert N.lib().sb200_debug_plan(1, rows, cin, cout, k, dil, act, res, acc, o) == 0
    return list(o)


def run_case(case):
    """One launch of `case` on seeded inputs (gap rows of the input zero, as the engine keeps them); returns the outputs
    (y0, and y1 when the case splits)."""
    import conv_unit as cu
    import torch
    name, lens, gran, seg_mul, cin, cout, k, dil, slope, act, use_res, scale, acc, split = case
    if gran is None:
        rows, ends, gran = lens, [lens], (lens + 255) // 256 * 256
    else:
        rows, ends = cu.segment_table(lens, gran, seg_mul)
    valid = cu.valid_rows_mask(rows, ends, gran, seg_mul)
    rng = np.random.default_rng(sum(map(ord, name)))
    x = rng.standard_normal((rows, cin)).astype(np.float32)
    x[~valid] = 0
    w = (rng.standard_normal((cout, cin, k)) / (cin * k) ** 0.5).astype(np.float32)
    b = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    res = torch.from_numpy(rng.standard_normal((rows, cout)).astype(np.float32)) if use_res else None
    ycols = cout // 2 if act == ACT_GATE else cout
    yinit = rng.standard_normal((rows, ycols)).astype(np.float32)
    if split is None:
        y0, y1 = np.ascontiguousarray(yinit), None
    else:
        y0, y1 = np.ascontiguousarray(yinit[:, :split]), np.ascontiguousarray(yinit[:, split:])
    msg = cu.run_conv(1, torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b), dil, slope, act, res, scale,
                      seg_end=ends, gran=gran, seg_mul=seg_mul, y0=y0, acc0=acc, split=split, y1=y1, acc1=acc)
    assert not msg, (name, msg)
    return [y0] if y1 is None else [y0, y1]


def synthesize(voice_path, lens):
    """Waveforms of one deterministic batch (zero noise scales), one per utterance."""
    import sonata_b200
    from sonata_b200 import PiperSynthesisConfig, workload
    m = sonata_b200.from_config_path(voice_path, device=0)
    try:
        m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.0, 1.0, 0.0))
        batches = [workload.synthetic_ids(n, utt=90 + i) for i, n in enumerate(lens)]
        return [np.asarray(a.samples.as_slice()).copy() for a in m.infer_batch_with_values(batches)]
    finally:
        m.close()


def digests(arrays, rows=128):
    """SHA-256 of every `rows`-row block of each array, as "<array>:<block>:<hex>" strings."""
    out = []
    for i, a in enumerate(arrays):
        a = np.ascontiguousarray(a, dtype=np.float32)
        for t in range(0, max(len(a), 1), rows):
            out.append(f"{i}:{t // rows}:{hashlib.sha256(a[t:t + rows].tobytes()).hexdigest()}")
    return np.array(out)


def mismatches(got, want):
    """Blocks whose digest differs (or that one side lacks), for the assertion message."""
    g, w = set(got.tolist()), set(want.tolist())
    return sorted({":".join(d.split(":")[:2]) for d in g ^ w})[:20]


def test_cases_reach_every_tile_width_and_weight_mode():
    """The cases launch at the widths and weight modes they are named for."""
    import conv_unit as cu
    seen = set()
    for name, lens, gran, seg_mul, cin, cout, k, dil, slope, act, use_res, scale, acc, split in CASES:
        rows = lens if gran is None else cu.segment_table(lens, gran, seg_mul)[0]
        p = plan(rows, cin, cout, k, dil, act, int(use_res), int(acc))
        nt, resident = p[0], p[8]
        assert f"nt{nt}" in name or name == "nearly_empty_last_tile", (name, p)
        assert ("resident" in name) <= bool(resident) and ("streamed" in name) <= (not resident), (name, p)
        seen.add((nt, resident))
    assert {nt for nt, _ in seen} == {32, 64, 96, 128} and {r for _, r in seen} == {0, 1}


@pytest.fixture
def grid_cap(lib_built):
    lib = N.lib()
    prev = lib.sb200_debug_conv_grid_cap(0)
    yield lambda cap: lib.sb200_debug_conv_grid_cap(cap)
    lib.sb200_debug_conv_grid_cap(prev)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_keeps_the_bits_of_the_previous_kernel(case, grid_cap):
    want = np.load(GOLDEN)["conv_" + case[0]]
    for cap in (1, 5, 0):
        grid_cap(cap)
        got = digests(run_case(case))
        assert np.array_equal(got, want), (case[0], cap, "output:tile", mismatches(got, want))


@pytest.mark.gpu
@pytest.mark.parametrize("q,lens", SYNTH, ids=[s[0] for s in SYNTH])
def test_synthesis_keeps_the_bits_of_the_previous_kernel(q, lens, voice_paths, grid_cap):
    """Every conv_tc launch of a synthesis, including the phase-fused ConvTranspose layers (u = 8 / 8 / 4 on medium,
    8 / 8 / 2 / 2 on high), launched as ordinary convs over their row-major u*cout-column output."""
    want = np.load(GOLDEN)["synth_" + q]
    for cap in (0, 7, 1):
        grid_cap(cap)
        got = digests(synthesize(voice_paths[q], lens), rows=128 * 256)
        assert np.array_equal(got, want), (q, cap, "utterance:block", mismatches(got, want))
