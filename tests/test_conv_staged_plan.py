"""Host logic of the staged epilogue operands of the bf16x2 conv kernel (`conv_tc.cu`): the producers stage each tile's
residual and accumulated output in shared memory while the MMAs run, on tiles wider than 32 columns where that fits
beside the ring at the tile width and CTAs per SM the kernel is planned with otherwise.  Planning only
(`sb200_debug_plan_staging`, `sb200_debug_plan`), so this runs without a GPU."""
import ctypes as C

from sonata_b200 import _native as N
from sonata_b200 import voicegen

SMEM_MAX = 227 * 1024
ACT_NONE, ACT_GATE = 0, 2

# (cin, cout, k, dil, act, res, acc) -> (tile width, CTAs per SM) at 100, 900, 20 000, 460 000 and 14 700 000 rows, as
# planned before staging existed (the shapes of test_conv_persistent_gpu.py's plan test)
UNSTAGED_PLANS = {
    (32, 32, 7, 12, ACT_NONE, 1, 0): [(32, 2)] * 5,
    (32, 32, 3, 1, ACT_NONE, 1, 1): [(32, 2)] * 5,
    (64, 64, 7, 6, ACT_NONE, 1, 0): [(32, 2), (32, 2), (64, 1), (64, 1), (64, 1)],
    (128, 128, 7, 3, ACT_NONE, 1, 1): [(32, 2), (32, 2), (64, 1), (64, 1), (64, 1)],
    (256, 256, 11, 5, ACT_NONE, 1, 0): [(32, 1), (32, 1), (64, 1), (64, 1), (64, 1)],
    (192, 384, 5, 1, ACT_GATE, 0, 0): [(32, 2), (32, 2), (128, 1), (128, 1), (128, 1)],
    (192, 384, 1, 1, ACT_NONE, 0, 1): [(32, 2), (32, 2), (128, 1), (128, 1), (128, 1)],
    (96, 192, 1, 1, ACT_NONE, 0, 0): [(32, 2), (32, 2), (96, 1), (96, 1), (96, 1)],
}
# ResBlock rows of the medium voice: C1 (one utterance, ~1 660 frames) and C2 (32 of them), x64 / x256 upsampled
MEDIUM_ROWS = {64: (1_660 * 64, 52_600 * 64), 32: (1_660 * 256, 52_600 * 256)}


def plan(rows, cin, cout, k, dil, act=ACT_NONE, res=0, acc=0):
    o = (C.c_int32 * 16)()
    assert N.lib().sb200_debug_plan(1, rows, cin, cout, k, dil, act, res, acc, o) == 0
    return list(o)


def staging(rows, cin, cout, k, dil, act=ACT_NONE, res=0, acc=0):
    b = C.c_int32(-1)
    assert N.lib().sb200_debug_plan_staging(rows, cin, cout, k, dil, act, res, acc, C.byref(b)) == 0
    return b.value


def medium_resblock_layers():
    a = voicegen.ARCH["medium"]
    assert a["resblock"] == 2
    ch, out = a["up_init"], []
    for _ in a["up_rates"]:
        ch //= 2
        for k, dils in zip(a["res_kernels"], a["res_dils"]):
            out += [(ch, ch, k, d, ACT_NONE, 1, acc) for d in dils for acc in (0, 1)]
    return out


def test_medium_mrf1_convs_are_staged_and_mrf2_convs_are_not():
    """Every 64-channel ResBlock conv is staged; the 32-channel ones (two 32-column CTAs per SM) are not."""
    layers = [lay for lay in medium_resblock_layers() if lay[0] in MEDIUM_ROWS]
    assert {lay[0] for lay in layers} == {32, 64}
    for lay in layers:
        for rows in MEDIUM_ROWS[lay[0]]:
            p = plan(rows, *lay)
            want = (int(lay[5]) + int(lay[6])) * 128 * p[0] * 4 if p[0] > 32 else 0   # residual (+ accumulated output)
            assert staging(rows, *lay) == want, (lay, rows)
            assert p[0] == lay[1] and p[5] <= SMEM_MAX, (lay, rows)


def test_staging_keeps_tile_width_and_ctas_per_sm():
    for lay, want in UNSTAGED_PLANS.items():
        for rows, (nt, per_sm) in zip((100, 900, 20_000, 460_000, 14_700_000), want):
            p = plan(rows, *lay)
            assert (p[0], p[9]) == (nt, per_sm), (lay, rows, p)
            assert p[10:] == [0] * 6, (lay, rows, p)


def test_only_launches_that_read_are_staged():
    assert staging(460_000, 192, 384, 5, 1, ACT_GATE, 0, 0) == 0           # gate: per-element epilogue
    assert staging(460_000, 96, 192, 1, 1, ACT_NONE, 0, 0) == 0            # reads nothing
    assert staging(460_000, 192, 384, 1, 1, ACT_NONE, 0, 1) > 0            # the flow's accumulated res/skip layer
    # 64-channel k7 dil 12 with residual and accumulation: exactly the 227 KB opt-in limit
    assert plan(3_366_400, 64, 64, 7, 12, ACT_NONE, 1, 1)[5] == SMEM_MAX
    # where staging would not fit beside the ring, the launch is planned as before
    assert staging(460_000, 256, 256, 11, 5, ACT_NONE, 1, 0) == 0
