"""Host logic of the wgmma launch planners (`conv_tc.cu` / `conv_tf.cu` plan()), through `sb200_debug_plan`: planning
only, nothing is launched, so this runs without a GPU.

The property that matters most: the reference's `speak_batch` is a loop of B=1 runs, and this implementation promises
the same bits for an utterance whether it is synthesised alone or inside a batch (`test_batched_equals_sequential`,
`test_frontends_on_the_device` check it on the device, with exact equality).  The planners pick tile widths from the
launch SIZE -- which changes no summation order: a wgmma gives an output element the same bits at every N, which
`test_conv_results_do_not_depend_on_tile_width` checks on the device for each width -- but the choice that DOES change
arithmetic (the chunk length of the flushed accumulation) must depend on the layer's shape alone."""
import ctypes as C

import pytest

from sonata_b200 import _native as N
from sonata_b200 import voicegen

ROWS = (100, 128, 700, 3000, 20_000, 300_000, 4_000_000)
SMEM_MAX = 227 * 1024
BUDGET = 227 * 1024 - 1024                           # two ring stages, after the 1024-byte alignment slack
SMS = 132                                            # the planners assume an H100 SXM when no device is visible
ACT_NONE, ACT_RELU, ACT_GATE = 0, 1, 2


def plan(backend, rows, cin, cout, k, dil, act=ACT_NONE, res=0, acc=0):
    o = (C.c_int32 * 16)()
    rc = N.lib().sb200_debug_plan(backend, rows, cin, cout, k, dil, act, res, acc, o)
    return None if rc else list(o)


def phase_fused_layers(q):
    """(cin, cout, k, dil, act, res, acc) of each ConvTranspose1d run as one conv of u*cout columns.  Its taps are the
    union of the phases' taps, derived as voice.cu does: output q*u + p reads input q + off through kernel index
    p + pad - off*u.  On every shipped voice that union is {-1, 0, 1}, a centred k = 3 conv."""
    a = voicegen.ARCH[q]
    L, ch = [], a["up_init"]
    for u, k in zip(a["up_rates"], a["up_kernels"]):
        pad = (k - u) // 2
        taps = {off for p in range(u) for off in range(-k, k + 1) if 0 <= p + pad - off * u < k}
        assert taps == {-1, 0, 1}, (q, u, k, taps)
        L.append((ch, u * (ch // 2), 3, 1, ACT_NONE, 0, 0))
        ch //= 2
    return L


def decoder_and_flow_layers(q):
    """(cin, cout, k, dil, act, res, acc) of every conv_tc layer of a voice."""
    a = voicegen.ARCH[q]
    H, half = a["hidden"], a["inter"] // 2
    L = {(half, H, 1, 1, ACT_NONE, 0, 0), (H, 2 * H, a["flow_kernel"], 1, ACT_GATE, 0, 0), (H, 2 * H, 1, 1, ACT_NONE, 0, 1),
         (H, H, 1, 1, ACT_NONE, 0, 1), (H, half, 1, 1, ACT_NONE, 0, 0), (a["inter"], a["up_init"], 7, 1, ACT_NONE, 0, 0)}
    L |= set(phase_fused_layers(q))
    ch = a["up_init"]
    for _ in a["up_rates"]:
        ch //= 2
        for k, dils in zip(a["res_kernels"], a["res_dils"]):
            for d in dils:
                if a["resblock"] == 2:
                    L |= {(ch, ch, k, d, ACT_NONE, 1, acc) for acc in (0, 1)}
                else:
                    L |= {(ch, ch, k, d, ACT_NONE, 0, 0)} | {(ch, ch, k, 1, ACT_NONE, 1, acc) for acc in (0, 1)}
    return sorted(L)


def encoder_layers(q):
    a = voicegen.ARCH[q]
    H, F, k = a["hidden"], a["filter"], a["kernel"]
    return [(H, 3 * H, 1, 1, ACT_NONE, 0, 0), (H, H, 1, 1, ACT_NONE, 0, 0), (H, F, k, 1, ACT_RELU, 0, 0), (F, H, k, 1, ACT_NONE, 0, 0),
            (H, 2 * a["inter"], 1, 1, ACT_NONE, 0, 0)]


def two_stages_fit(win, k, cols, images):
    """Two ring stages of a window (`images` images of win x 128 B) and k taps of `images` weight images of cols rows."""
    return 2 * (images * win * 128 + k * images * cols * 128) <= BUDGET


@pytest.mark.parametrize("q", ["medium", "high"])
def test_arithmetic_class_does_not_depend_on_launch_size(q):
    for lay in decoder_and_flow_layers(q):
        for rows in ROWS:
            p = plan(1, rows, *lay)
            assert p is not None, (lay, rows)
            nt, wnt, mt, ntn, stages, smem, win = p[:7]
            assert smem <= SMEM_MAX and stages >= 2 and wnt % nt == 0 and nt % 32 == 0, (lay, rows, p)
            if nt < wnt:                       # narrow tiles: only while no SM would get a second tile, or when two stages
                assert mt * ntn <= SMS or not two_stages_fit(win, lay[2], wnt, 1), (lay, rows, p)   # of the full width
                                                                                                   # do not fit
    for lay in encoder_layers(q):
        chunks = set()
        for rows in ROWS:
            p = plan(2, rows, *lay)
            assert p is not None, (lay, rows)
            nth, wnth, mt, ntn, stages, chunk_kb, smem, win = p[:8]
            chunks.add(chunk_kb)
            assert smem <= SMEM_MAX and stages >= 2 and wnth % nth == 0 and nth in (32, 64, 96), (lay, rows, p)
            if nth < wnth:
                assert mt * (lay[1] // 32) <= SMS or not two_stages_fit(win, lay[2], wnth, 2), (lay, rows, p)
        assert len(chunks) == 1, (lay, chunks)


@pytest.mark.parametrize("q", ["medium", "high", "x_low", "low"])
def test_phase_fused_transposed_convs_plan_at_every_size(q):
    """The phase-fused ConvTranspose carries bf16 images only (its phases keep fp32 ones for backend 0), so on the
    tensor-core backends conv_tc must take it at every launch size."""
    for lay in phase_fused_layers(q):
        for rows in ROWS:
            p = plan(1, rows, *lay)
            assert p is not None and p[5] <= SMEM_MAX, (q, lay, rows, p)


def test_tile_width_cases_reach_several_widths():
    """The device-side bit-identity check (tools/conv_unit.py WIDTH_CASES) launches each shape once per tile width the
    planner picks over launch sizes: every shape must reach at least two widths, the narrowest being 32 columns, and
    the narrowing edges the kernel cases straddle must be where the planner switches."""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import conv_unit as cu
    for case in cu.WIDTH_CASES:
        w = cu.tile_width_launches(*case)
        assert len(w) >= 2 and min(w) == 32, (case, w)
    for cout, nt, lay in ((64, 32, (64, 64, 7, 12, ACT_NONE, 1, 1)), (384, 32, (192, 384, 5, 1, ACT_GATE, 0, 0)),
                          (256, 32, (256, 256, 11, 5, ACT_NONE, 1, 0))):
        e = cu.narrow_edge(cout, nt)
        assert plan(1, e, *lay)[0] == nt and plan(1, e + 1, *lay)[0] > nt, (cout, e)


def test_hot_layers_get_the_configurations_design_md_describes():
    # 32-channel ResBlock conv (dec.mrf2 at C2 size): one 32-column tile, two stages
    p = plan(1, 14_700_000, 32, 32, 3, 1, ACT_NONE, 1, 0)
    assert p[:2] == [32, 32] and p[4] == 2
    # 256-channel k11 / dilation 5 ResBlock conv: two stages of the 128-column images do not fit, 64-column parts do
    p = plan(1, 460_000, 256, 256, 11, 5, ACT_NONE, 1, 0)
    assert (p[0], p[1]) == (64, 128) and p[5] <= SMEM_MAX
    # flow in_layer on a big launch: full 128-column tiles
    p = plan(1, 57_600, 192, 384, 5, 1, ACT_GATE, 0, 0)
    assert (p[0], p[1]) == (128, 128)
    # the same layer for one utterance: 32-column parts of the 128-row images, no more tiles than SMs
    p = plan(1, 900, 192, 384, 5, 1, ACT_GATE, 0, 0)
    assert (p[0], p[1]) == (32, 128) and p[2] * p[3] <= SMS
    # encoder: 1x1 layers flush every two K-blocks, k-tap layers every K-block
    assert plan(2, 100_000, 192, 576, 1, 1)[5] == 2 and plan(2, 100_000, 192, 768, 3, 1, ACT_RELU)[5] == 1
    # unsupported shapes are refused, not mis-planned
    assert plan(1, 1000, 48, 64, 3, 1) is None and plan(2, 1000, 192, 100, 1, 1) is None
