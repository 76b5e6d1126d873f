// A whole HiFi-GAN ResBlock2 stage of 64 channels as one wgmma kernel (bf16x2, sm_90a):
//   ys = (1/nbr) sum_b [ x1_b + conv2_b(lrelu(x1_b)) ],   x1_b = x + conv1_b(lrelu(x)),
// where the layer-wise formulation (engine.cu run_decoder) runs six conv_tc launches that each read and write a full fp32
// activation.  Here the stage input is read once per tile (with its halo) and the mean is written once.
//
// Bits.  Every conv keeps the arithmetic of the conv_tc launch it replaces: the accumulator starts at zero, the MMA issue
// order per accumulator is (K-block, tap, K step, hi*hi, lo*hi, hi*lo) on the same pre-split, pre-swizzled weight images
// (ConvW::wtc), the A operand is split(lrelu(v)) with the same splitter, and the epilogues are conv_tc's store_group:
//   conv1:           x1 = fmaf(acc + bias, 1, x * 1)
//   conv2, branch 0: ys = fmaf(acc + bias, s, x1 * s)            s = 1 / nbr
//   conv2, later:    ys = fmaf(acc + bias, s, x1 * s + ys)
// x1 is 0 at invalid rows (gap rows and rows outside the array), which is what the layer-wise conv2 reads from its
// buffer; ys is 0 at invalid rows.  A wgmma row depends on its own A row alone, so a tile may place rows anywhere in
// its 64-row blocks.
//
// Tiles.  A persistent CTA per SM walks a contiguous run of 128-row output tiles [t0, t0 + 128), in order, so that no
// row of x1 is computed twice: per branch (h1, h2: the halos of its conv1 and conv2), conv1 computes only the tile's 128
// new x1 rows [t0 + h2, t0 + 128 + h2), one 64-row block per MMA warpgroup, and the 2 h2 rows before them are the ones
// the previous tile computed, saved in shared memory.  conv2 then runs over the tile (one block per warpgroup) and folds
// into the mean, held in registers by the thread that owns the same outputs in every branch.  Before its first tile a
// CTA runs the conv1s alone over the tile before it, which seeds those halos.  Per tile the fp32 x window
// [t0 + min(h2 - h1), t0 + 128 + max(h2 + h1)) is loaded once (rows outside the array zero-filled).  So the kernel runs
// exactly the MMAs of the six layer-wise launches, plus one conv1 tile per CTA.
//
// Shared memory: the weight ring, the x window, x1 [t0 - h2, t0 + 128 + h2) of the current branch, and each branch's
// saved halo rows, all fp32 rows of 256 bytes with 16-byte chunk j at j ^ 2 (row & 7), so a warp's fragment and epilogue
// accesses (8 consecutive rows x 32 bytes) hit every bank exactly twice.  The A fragments are split from the fp32 rows
// as they are loaded (split images would not fit beside them), so the residuals stay exact.
//
// Roles: two MMA warpgroups (fragments, wgmma, epilogues), and one producer warpgroup whose first thread streams the
// weight images (one 8 KB cp.async.bulk per (conv, K-block, tap) through an 8-slot ring, full / empty mbarriers), and
// whose other three warps load the next tile's x window once the last conv1 of the tile has read it (cp.async, completion
// on an mbarrier).  Every mbarrier wait carries conv_tc's trap watchdog.
#include "engine.h"
#include "tc_common.cuh"
#include <algorithm>
#include <climits>

namespace sb200 {

namespace {

using namespace tcx;

constexpr int RB_M = 128;                     // output rows per tile
constexpr int RB_C = 64;                      // channels
constexpr int RB_ROW = RB_C * 4;              // bytes of one fp32 row
constexpr int RB_IMG = RB_C * 128;            // one weight image: 64 output columns x [hi | lo] of a 32-channel K-block
constexpr int RB_RING = 8;                    // weight ring slots
constexpr int RB_MAX_BR = 4;                  // branches of a stage
constexpr int RB_CONSUMERS = 256;             // two MMA warpgroups
constexpr int RB_LOADERS = 96;                // producer warps 1-3: the x window
constexpr int RB_THREADS = RB_CONSUMERS + 128;
constexpr int RB_PRODUCER_REGS = 40, RB_CONSUMER_REGS = 232;   // setmaxnreg: 128 * 40 + 256 * 232 <= 65536
constexpr int RB_BAR_BYTES = 8 * (2 * RB_RING + 2);

struct Rb2Conv {
    const uint8_t* wtc;          // [K-block][tap] images (ConvW::wtc of a 64-column layer: one n-tile)
    const float* bias;
    int ntaps, h;                // h: the halo, -min_off = max_off
    int off[SB_MAX_TAPS];
};
struct Rb2Args {
    const float* x; float* y;    // [map.rows][64]
    RowMap map;
    float scale;                 // 1 / nbr
    int nbr;
    Rb2Conv c[RB_MAX_BR][2];
    int lo, win;                 // x window: rows [t0 + lo, t0 + lo + win)
    int x1rows, hrows;           // x1 rows (128 + 2 max h2); saved halo rows (sum of 2 h2)
    int hoff[RB_MAX_BR];         // first saved halo row of each branch
    int ntiles;
};

// fp32 row `row` of a buffer, channel `ch` (even: an 8-byte pair)
__device__ __forceinline__ uint32_t rb_addr(uint32_t buf, int row, int ch) {
    return buf + (uint32_t)row * RB_ROW + ((uint32_t)((ch >> 2) ^ ((row & 7) << 1)) << 4) + 4u * (uint32_t)(ch & 3);
}
__device__ __forceinline__ float lrelu(float v) { return fmaxf(v, v * 0.1f); }

// A fragments of K-block kb for rows R0 and R0 + 8 (the m16n8k16 layout per warp, as conv_tc's load_frag), split from
// the fp32 rows through the leaky-ReLU prologue
__device__ __forceinline__ void load_frag(uint32_t buf, int R0, int kb, int c, uint32_t (&ah)[2][4], uint32_t (&al)[2][4]) {
#pragma unroll
    for (int ks = 0; ks < 2; ks++) {
        const int ch = kb * 32 + 16 * ks + 2 * c;
        const float2 v0 = lds64(rb_addr(buf, R0, ch)), v1 = lds64(rb_addr(buf, R0 + 8, ch));
        const float2 v2 = lds64(rb_addr(buf, R0, ch + 8)), v3 = lds64(rb_addr(buf, R0 + 8, ch + 8));
        ah[ks][0] = split2(lrelu(v0.x), lrelu(v0.y), al[ks][0]);
        ah[ks][1] = split2(lrelu(v1.x), lrelu(v1.y), al[ks][1]);
        ah[ks][2] = split2(lrelu(v2.x), lrelu(v2.y), al[ks][2]);
        ah[ks][3] = split2(lrelu(v3.x), lrelu(v3.y), al[ks][3]);
    }
}
__device__ __forceinline__ void mma_tap(float* acc, const uint32_t (&ah)[2][4], const uint32_t (&al)[2][4], uint32_t wimg) {
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 2; ks++) {
        const uint64_t dwh = sw128_desc(wimg + 32u * ks);
        const uint64_t dwl = sw128_desc(wimg + 64u + 32u * ks);
        wgmma_rs<WG_BF16, 64>(acc, ah[ks], dwh);
        wgmma_rs<WG_BF16, 64>(acc, al[ks], dwh);
        wgmma_rs<WG_BF16, 64>(acc, ah[ks], dwl);
    }
    wg_commit();
}

// One conv over this warpgroup's 64-row block: acc = sum over (K-block, tap), row r reading buffer row base + r + off[tap].
// The weight images are ring slots wseq, wseq + 1, ...  Fragments are double-buffered across the (K-block, tap) steps,
// taken in pairs: the group before retired (wait_group 1) before its set is reloaded.
__device__ __forceinline__ void conv_block(float (&acc)[32], const Rb2Conv& cw, uint32_t buf, int base, int rw, int c,
                                           uint32_t W0, uint32_t FULL, uint32_t EMPTY, uint32_t wseq) {
#pragma unroll
    for (int i = 0; i < 32; i++) acc[i] = 0.f;
    acc_fence<32>(acc);
    uint32_t ah[2][2][4], al[2][2][4];
    const int nkt = 2 * cw.ntaps;                       // (K-block, tap) steps, K-block major; even
    for (int kt = 0; kt < nkt; kt += 2) {
#pragma unroll
        for (int n = 0; n < 2; n++) {
            const int k2 = kt + n;
            const uint32_t seq = wseq + (uint32_t)k2, s = seq % RB_RING;
            mbar_wait<false>(FULL + 8u * s, (seq / RB_RING) & 1u);
            const int kb = k2 / cw.ntaps, t = k2 - kb * cw.ntaps;
            load_frag(buf, base + rw + cw.off[t], kb, c, ah[n], al[n]);
            mma_tap(acc, ah[n], al[n], W0 + s * RB_IMG);
            wg_wait1();
            // every group but the newest has retired: the previous step's slot is free
            if (k2 > 0) mbar_arrive(EMPTY + 8u * ((seq - 1) % RB_RING));
        }
    }
    wg_wait0();
    mbar_arrive(EMPTY + 8u * ((wseq + nkt - 1) % RB_RING));
    acc_fence<32>(acc);
}

__global__ void __launch_bounds__(RB_THREADS, 1) resblock2_tc_kernel(const __grid_constant__ Rb2Args a) {
    pdl_trigger();
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw), W0 = (raw + 1023u) & ~1023u;
    const uint32_t X = W0 + RB_RING * RB_IMG, X1 = X + (uint32_t)a.win * RB_ROW;
    const uint32_t H = X1 + (uint32_t)a.x1rows * RB_ROW;        // saved halo rows of every branch
    const uint32_t FULL = H + (uint32_t)a.hrows * RB_ROW;       // full[s]: slot s's image landed
    const uint32_t EMPTY = FULL + 8u * RB_RING;                  // empty[s]: both MMA warpgroups done reading slot s
    const uint32_t XFULL = EMPTY + 8u * RB_RING;                 // the tile's x window landed
    const uint32_t XEMPTY = XFULL + 8u;                          // the tile's last conv1 has read it
    const int tid = threadIdx.x;
    if (tid == 0) {
        for (int s = 0; s < RB_RING; s++) {
            mbar_init(FULL + 8u * s, 1);
            mbar_init(EMPTY + 8u * s, RB_CONSUMERS);
        }
        mbar_init(XFULL, RB_LOADERS);                            // one cp.async arrival per loader thread
        mbar_init(XEMPTY, RB_CONSUMERS);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // this CTA's tiles [first, last), after the conv1-only pass over tile first - 1
    const int first = (int)((long long)blockIdx.x * a.ntiles / gridDim.x);
    const int last = (int)((long long)(blockIdx.x + 1) * a.ntiles / gridDim.x);

    if (tid >= RB_CONSUMERS) {
        // ================================== producer warpgroup: weights and x windows ==================================
        setmaxnreg_dec<RB_PRODUCER_REGS>();
        const int ptid = tid - RB_CONSUMERS;
        if (ptid < 32) {
            // weights are constants: streamed without waiting for the predecessor
            if (ptid != 0) return;
            uint32_t seq = 0;
            for (int tile = first - 1; tile < last; tile++)
                for (int b = 0; b < a.nbr; b++)
                    for (int cv = 0; cv < (tile < first ? 1 : 2); cv++) {
                        const Rb2Conv& cw = a.c[b][cv];
                        for (int i = 0; i < 2 * cw.ntaps; i++, seq++) {
                            const uint32_t s = seq % RB_RING;
                            if (seq >= RB_RING) mbar_wait<false>(EMPTY + 8u * s, (seq / RB_RING - 1) & 1u);
                            mbar_expect_tx(FULL + 8u * s, RB_IMG);
                            bulk_g2s(W0 + s * RB_IMG, cw.wtc + (size_t)i * RB_IMG, RB_IMG, FULL + 8u * s);
                        }
                    }
            return;
        }
        pdl_wait();
        const int lt = ptid - 32;
        int it = 0;
        for (int tile = first - 1; tile < last; tile++, it++) {
            if (it > 0) mbar_wait<false>(XEMPTY, (uint32_t)(it - 1) & 1u);
            const int r0 = tile * RB_M + a.lo;
            for (int idx = lt; idx < a.win * 16; idx += RB_LOADERS) {
                const int row = idx >> 4, ch = idx & 15, gr = r0 + row;
                const bool ok = gr >= 0 && gr < a.map.rows;
                cp_async16(X + (uint32_t)row * RB_ROW + ((uint32_t)(ch ^ ((row & 7) << 1)) << 4),
                           ok ? a.x + (size_t)gr * RB_C + ch * 4 : a.x, ok ? 16u : 0u);
            }
            cp_async_commit();
            cp_async_mbar_arrive(XFULL);
        }
        cp_async_wait<0>();
        return;
    }

    // ================================= two MMA warpgroups: fragments, wgmma, epilogues =================================
    setmaxnreg_inc<RB_CONSUMER_REGS>();
    pdl_wait();
    const int warp = tid >> 5, lane = tid & 31;
    const int wg = warp >> 2, g = lane >> 2, c = lane & 3;
    const int rw = (warp & 3) * 16 + g;                  // rows rw and rw + 8 of each 64-row block
    float acc[32], ys[32];
    uint32_t wseq = 0;
    int it = 0;
    for (int tile = first - 1; tile < last; tile++, it++) {
        const int t0 = tile * RB_M;
        const bool seed = tile < first;                  // conv1s only: the halos of tile `first`
        mbar_wait<false>(XFULL, (uint32_t)it & 1u);
        for (int b = 0; b < a.nbr; b++) {
            const Rb2Conv& c1 = a.c[b][0];
            const Rb2Conv& c2 = a.c[b][1];
            const int h2 = c2.h, nh = 2 * h2;
            // ---- conv1 over the new x1 rows [t0 + h2, t0 + 128 + h2): new row i reads x window row i + xs + off, and
            // is x1 row nh + i (x1 row j: row t0 - h2 + j) ----
            const int xs = h2 - a.lo;
            conv_block(acc, c1, X, wg * 64 + xs, rw, c, W0, FULL, EMPTY, wseq);
            wseq += 2 * c1.ntaps;
            named_bar_sync(1, RB_CONSUMERS);            // the previous conv2 has read x1
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int i = wg * 64 + rw + 8 * h;
                const bool valid = row_valid(a.map, t0 + h2 + i);
#pragma unroll
                for (int p = 0; p < 8; p++) {
                    const int n = 8 * p + 2 * c;
                    float2 v = make_float2(0.f, 0.f);
                    if (valid) {
                        const float2 bias = *reinterpret_cast<const float2*>(c1.bias + n);
                        const float2 r = lds64(rb_addr(X, i + xs, n));
                        const float o0 = acc[4 * p + 2 * h] + bias.x, o1 = acc[4 * p + 2 * h + 1] + bias.y;
                        v = make_float2(fmaf(o0, 1.f, r.x * 1.f), fmaf(o1, 1.f, r.y * 1.f));
                    }
                    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(rb_addr(X1, nh + i, n)), "f"(v.x), "f"(v.y) : "memory");
                }
            }
            // x1 rows [0, nh): the previous tile's, saved (on the seed pass they are never read)
            for (int k = tid; k < nh * 16; k += RB_CONSUMERS) {
                const int j = k >> 4, ch = 4 * (k & 15);
                const float4 v = lds128(rb_addr(H, a.hoff[b] + j, ch));
                sts128u(rb_addr(X1, j, ch), make_uint4(__float_as_uint(v.x), __float_as_uint(v.y), __float_as_uint(v.z),
                                                        __float_as_uint(v.w)));
            }
            if (b == a.nbr - 1) mbar_arrive(XEMPTY);     // the loaders may fetch the next tile's window
            named_bar_sync(1, RB_CONSUMERS);            // x1 complete
            // the next tile's x1 rows [0, nh) are this tile's [128, 128 + nh)
            for (int k = tid; k < nh * 16; k += RB_CONSUMERS) {
                const int j = k >> 4, ch = 4 * (k & 15);
                const float4 v = lds128(rb_addr(X1, RB_M + j, ch));
                sts128u(rb_addr(H, a.hoff[b] + j, ch), make_uint4(__float_as_uint(v.x), __float_as_uint(v.y),
                                                                   __float_as_uint(v.z), __float_as_uint(v.w)));
            }
            if (seed) continue;
            // ---- conv2 over the tile: block wg; tile row r reads x1 row r + off + h2 ----
            conv_block(acc, c2, X1, wg * 64 + h2, rw, c, W0, FULL, EMPTY, wseq);
            wseq += 2 * c2.ntaps;
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int r = wg * 64 + rw + 8 * h;
                const bool valid = row_valid(a.map, t0 + r);
#pragma unroll
                for (int p = 0; p < 8; p++) {
                    const int n = 8 * p + 2 * c;
                    float2 v = make_float2(0.f, 0.f);
                    if (valid) {
                        const float2 bias = *reinterpret_cast<const float2*>(c2.bias + n);
                        const float2 x1 = lds64(rb_addr(X1, r + h2, n));
                        const float o0 = acc[4 * p + 2 * h] + bias.x, o1 = acc[4 * p + 2 * h + 1] + bias.y;
                        float m0 = x1.x * a.scale, m1 = x1.y * a.scale;
                        if (b > 0) { m0 += ys[4 * p + 2 * h]; m1 += ys[4 * p + 2 * h + 1]; }
                        v = make_float2(fmaf(o0, a.scale, m0), fmaf(o1, a.scale, m1));
                    }
                    ys[4 * p + 2 * h] = v.x;
                    ys[4 * p + 2 * h + 1] = v.y;
                }
            }
        }
        if (seed) continue;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int q = t0 + wg * 64 + rw + 8 * h;
            if (q >= a.map.rows) continue;
#pragma unroll
            for (int p = 0; p < 8; p++)
                *reinterpret_cast<float2*>(a.y + (size_t)q * RB_C + 8 * p + 2 * c) =
                    make_float2(ys[4 * p + 2 * h], ys[4 * p + 2 * h + 1]);
        }
    }
}

size_t rb_smem(const Rb2Args& a) {
    return 1024 + (size_t)RB_RING * RB_IMG + (size_t)(a.win + a.x1rows + a.hrows) * RB_ROW + RB_BAR_BYTES;
}

// The stage's launch arguments, or false when a conv is not a centred 64-channel layer with a bf16x2 image of one
// 64-column tile, or a halo does not fit the tile and shared memory
bool rb_args(const std::vector<ResBW>& res, const float* x, float* y, const RowMap& map, Rb2Args& a) {
    if (res.empty() || res.size() > RB_MAX_BR) return false;
    a = Rb2Args{};
    a.x = x; a.y = y; a.map = map;
    a.nbr = (int)res.size();
    a.scale = 1.0f / (float)res.size();
    int h2max = 0, hi = INT_MIN;
    a.lo = INT_MAX;
    for (int b = 0; b < a.nbr; b++) {
        if (res[b].c1.size() != 2) return false;
        for (int cv = 0; cv < 2; cv++) {
            const ConvW& w = res[b].c1[cv];
            if (!w.wtc || w.tc_nt != RB_C || w.cin != RB_C || w.cout != RB_C || w.cond_off >= 0) return false;
            if (w.span != -2 * w.min_off) return false;
            Rb2Conv& cw = a.c[b][cv];
            cw.wtc = reinterpret_cast<const uint8_t*>(w.wtc); cw.bias = w.bias;
            cw.ntaps = w.ntaps; cw.h = -w.min_off;
            std::copy(w.tap_off, w.tap_off + SB_MAX_TAPS, cw.off);
        }
        const int h1 = a.c[b][0].h, h2 = a.c[b][1].h;
        h2max = std::max(h2max, h2);
        a.lo = std::min(a.lo, h2 - h1);
        hi = std::max(hi, h2 + h1);
        a.hoff[b] = a.hrows;
        a.hrows += 2 * h2;
    }
    if (2 * h2max > RB_M) return false;               // the next tile's halo rows are among this tile's new rows
    a.win = RB_M + hi - a.lo;
    a.x1rows = RB_M + 2 * h2max;
    a.ntiles = (map.rows + RB_M - 1) / RB_M;
    return rb_smem(a) <= 227 * 1024;
}

int rb_grid(const Rb2Args& a) {
    int grid = wg_num_sms();
    if (g_conv_tc_grid_cap > 0) grid = std::min(grid, g_conv_tc_grid_cap);
    return std::max(1, std::min(grid, a.ntiles));
}

}  // namespace

bool resblock2_tc_plan(const std::vector<ResBW>& res, int rows, int* out8) {
    Rb2Args a;
    if (!rb_args(res, nullptr, nullptr, RowMap{nullptr, 1, 1, rows}, a)) return false;
    if (out8) {
        const int v[8] = {RB_M, a.win, a.x1rows, RB_RING, (int)rb_smem(a), rb_grid(a), RB_THREADS,
                          RB_PRODUCER_REGS * 128 + RB_CONSUMER_REGS * RB_CONSUMERS};
        std::copy(v, v + 8, out8);
    }
    return true;
}

void launch_resblock2_tc(const std::vector<ResBW>& res, const float* x, float* y, const RowMap& map, cudaStream_t st) {
    Rb2Args a;
    if (!rb_args(res, x, y, map, a)) throw_launch_error("resblock2_tc: stage shape not supported");
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 7))
        throw_launch_error("resblock2_tc: misaligned activations");
    static PerDeviceOnce once;
    once.run([] { cudaFuncSetAttribute(resblock2_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024); });
    launch_pdl(resblock2_tc_kernel, dim3(rb_grid(a)), dim3(RB_THREADS), rb_smem(a), st, a);
    g_launch_count++;
    check_launch("resblock2_tc");
}

}  // namespace sb200
