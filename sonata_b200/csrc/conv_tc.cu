// wgmma implicit-GEMM Conv1d with a 2-term BF16 split ("bf16x2", fp32 accumulate in registers), sm_90a.
//
// Same contract as conv_simt.cu (ConvArgs): out[q][n] = epi(bias[n] + sum_t sum_c f(x[q+off_t][c]) w[t][c][n]).
// GEMM view per tile: D[128 rows x NT cols] += A_t[128 x 32] . W_t[32 x NT] over (32-channel K-block, tap).
//
// Precision.  A single reduced-precision MMA misses the 1e-3 waveform tolerance (TF32: 1.9e-3 / 3.6e-3 on
// the medium / high voice).  Every operand is therefore split  v = hi + lo,  hi = bf16_rn(v),
// lo = bf16_rn(v - hi)  (16 mantissa bits together) and three MMAs accumulate  hi*hi + lo*hi + hi*lo.
// End-to-end waveform error 2e-5 / 3.5e-5 (oracle emulation) -- the same as a 3xTF32 split at half the MMAs
// (K = 16 per bf16 MMA against 8 per tf32 MMA).
//
// Persistent CTAs: the grid is as many CTAs as can be resident at once, and each walks a static list of 128-row x
// NT-column tiles.  A CTA keeps one n-tile (blockIdx % ntiles_n) and takes the m-tiles blockIdx / ntiles_n + i * (grid /
// ntiles_n): the CTAs of one m-tile run side by side, so the re-reads of its window come from L2.
//
// Warp-specialized: producer warps load and convert (one warpgroup on 32-column tiles, two on wider ones, which run one
// CTA per SM), two MMA warpgroups (tile rows 0-63 / 64-127) run the MMAs and the epilogue.  They hand off through a two-stage ring over the CTA's flat sequence of (tile, K-block) steps; each
// stage has a full and an empty mbarrier.  While the MMA warpgroups work on one step, the producer loads and converts the
// next (a deeper ring, where shared memory allowed one, was slower: DESIGN.md section 3):
//   * activations: the raw fp32 (128 + span)-row WINDOW of a K-block (32 channels = one 128-byte row) arrives by
//     cp.async (rows outside the array zero-filled); the producer then applies the leaky-ReLU prologue, splits hi/lo and
//     rewrites each row IN PLACE as [hi: 32 ch bf16 | lo: 32 ch bf16] in the K-major SWIZZLE_128B layout (row r at
//     r*128 B, 16-B chunk c at (c ^ (r & 7))), and arrives on the stage's full barrier.  A tap is the same window read
//     from a row offset: the A operand comes from registers (wgmma with A in registers), loaded per thread from the
//     swizzled image at any row, so a k-tap conv stages its input once;
//   * weights: pre-split, pre-swizzled images written at voice-load time, one cp.async.bulk (TMA) per tap image.
//     RESIDENT when the layer has at most two K-blocks (then all of the n-tile's images take no more shared memory than
//     two ring stages would): fetched once per CTA, before pdl_wait(), on a barrier of their own.  Otherwise each ring
//     stage holds one K-block's taps, counted in bytes on the stage's full barrier;
//   * MMA: wgmma.mma_async m64nNTk16 (B from shared memory by descriptor), six per (tap, K-block) and warpgroup, one
//     commit group per tap; the A fragments are double-buffered across taps (the next tap's load while this tap's MMAs
//     run, wait_group 1).  The issue order per accumulator is (K-block, tap, K step, hi*hi, lo*hi, hi*lo), so every
//     output keeps its bits.  Once a step's MMAs have retired, the MMA warpgroups arrive on the stage's empty barrier,
//     before the epilogue, so the producer refills it while they store;
//   * staged epilogue operands: on tiles wider than 32 columns, where they fit beside the ring at the same tile width
//     and CTAs per SM, the producers
//     also fetch each tile's residual and accumulated output (16-byte cp.async into one SWIZZLE_128B image per 32
//     columns, rows past the array zero-filled) while the MMA warpgroups run the tile's MMAs.  They complete on a
//     barrier of their own (cp.async.mbarrier.arrive), and the MMA warpgroups release the buffer on another once they
//     hold the operands in registers, before they store;
//   * epilogue: bias / gate / ReLU / residual / scale / accumulate straight from the accumulator registers; a column
//     pair is one 8-byte access where the output layout allows it.  Staged launches read the operands from shared
//     memory; the others issue a group of pairs' global reads before any of them stores (on tiles wider than 32
//     columns the first group's before the tile's last K-block runs its MMAs).
// Registers (setmaxnreg): 32-column tiles run 2 CTAs per SM at 80 registers per thread, the producer dropping to 40 and
// the MMA warpgroups rising to 96; wider tiles run one CTA per SM at 128, split 32 (two producer warpgroups) / 224.
// -Xptxas -v: no spills at NT = 32; 24 / 44 bytes of spill stores / loads at NT >= 64 (loop-invariant values, reloaded
// from L1).
// Every mbarrier wait carries a watchdog that traps instead of hanging the GPU.
#include "tc_common.cuh"
#include <algorithm>
#include <stdlib.h>
#include <string.h>

namespace sb200 {

int g_conv_tc_grid_cap = 0;

int wg_num_sms() {
    static int n = 0;
    if (!n) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
            cudaGetLastError();
        if (n <= 0) n = 132;
    }
    return n;
}

namespace {

using namespace tcx;

struct TcLaunch {
    int nt;          // columns per CTA tile (multiple of 32, <= 128)
    int wnt;         // rows of a weight IMAGE (the voice's tile width); nt == wnt, or a part of it (a multiple of 32 rows that
                     // divides it: every part keeps the image's swizzle, 32 % 8 == 0)
    int win;         // window rows (multiple of 8)
    int ntiles_m, ntiles_n;
    int grid;        // CTAs: a multiple of ntiles_n, at most ntiles_m * ntiles_n
    int resident;    // 1: every weight image of the CTA's n-tile stays in shared memory; 0: one K-block per ring stage
    int pairs;       // 1: a column pair may be one 8-byte access to res / y0 / y1 (aligned, no gate)
    int stage;       // 1: the producers stage each tile's residual / accumulated output in shared memory (needs pairs)
};

constexpr int TC_CONSUMERS = 256;       // two MMA warpgroups: tile rows [0, 64) and [64, 128)
constexpr int TC_STAGES = 2;
// full[TC_STAGES], empty[TC_STAGES], resident weights, staging full / free.  They live in the 1024 bytes of alignment
// slack (before the aligned base when it leaves room, else after the data), so they take no shared memory of their own.
constexpr int TC_BAR_BYTES = 64;

// Staged epilogue operand: 128 rows x nt fp32, one 16 KB SWIZZLE_128B image per 32 columns.  Element (r, col) at
// sw128(slab col / 32, r, (col % 32) / 4) + 4 (col % 4): the epilogue's float2 reads (rows g / g + 8, columns 8p + 2c)
// of a warp hit distinct banks, where a linear [128][nt] tile would be 4-way conflicted.
__device__ __forceinline__ uint32_t stg_addr(uint32_t base, int row, int col) {
    return sw128(base + (uint32_t)(col >> 5) * 16384u, row, (col >> 2) & 7) + 4u * (uint32_t)(col & 3);
}
// v, through a move the compiler cannot hoist out of a loop
__device__ __forceinline__ uint32_t opaque(uint32_t v) {
    asm volatile("mov.b32 %0, %0;" : "+r"(v));
    return v;
}

// Roles and register split per tile width.  32-column tiles run 2 CTAs per SM (their shared memory would allow more;
// registers decide) with one producer warpgroup: 80 registers at launch -> producer 40 / MMA warpgroups 96.  Wider tiles
// run one CTA per SM, and there the conversion of one warpgroup alone sets the pace of layers with short MMAs (the
// 64-channel ResBlocks), so two producer warpgroups share each window: 128 -> 32 / 224.
template <int NT> struct TcRoles {
    static constexpr int ctas = NT == 32 ? 2 : 1;
    static constexpr int producers = NT == 32 ? 128 : 256;   // window and weight loads, in-place conversion
    static constexpr int threads = TC_CONSUMERS + producers;
    static constexpr int launch = (65536 / (threads * ctas)) & ~7;
    static constexpr int producer_regs = NT == 32 ? 40 : 32;
    static constexpr int consumer_regs = ((launch * threads - producer_regs * producers) / TC_CONSUMERS) & ~7;
};

template <int NT>
__global__ void __launch_bounds__(TcRoles<NT>::threads, TcRoles<NT>::ctas) conv_tc_kernel(const ConvArgs a, const TcLaunch L) {
    constexpr int NPROD = TcRoles<NT>::producers;
    pdl_trigger();
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const int nkb = a.cin / 32, S = TC_STAGES;
    const bool acc_any = a.acc0 || a.acc1;
    const bool stage = NT > 32 && L.stage;                       // the planner stages wider tiles only
    const uint32_t a_buf = (uint32_t)L.win * 128u;               // one window image
    const uint32_t w_tap = (uint32_t)NT * 128u;                  // one tap of a weight image ([hi|lo] rows)
    const uint32_t w_kb = (uint32_t)a.ntaps * w_tap;             // the taps of one K-block
    const uint32_t w_bytes = L.resident ? (uint32_t)nkb * w_kb : (uint32_t)S * w_kb;
    const uint32_t stg_op = 128u * NT * 4u;                      // one staged epilogue operand
    const uint32_t raw = smem_u32(smem_raw), A0 = (raw + 1023u) & ~1023u, W0 = A0 + S * a_buf;
    const uint32_t SRES = W0 + w_bytes;                          // staged residual
    const uint32_t SACC = SRES + (stage && a.res ? stg_op : 0u);   // staged accumulated output
    const uint32_t data_end = SACC + (stage && acc_any ? stg_op : 0u);
    const uint32_t FULL = A0 - raw >= (uint32_t)TC_BAR_BYTES ? raw : data_end;   // full[s]: stage s converted (and its
                                                                                  // weights landed)
    const uint32_t EMPTY = FULL + 8u * TC_STAGES;                // empty[s]: both MMA warpgroups done reading stage s
    const uint32_t WRES = EMPTY + 8u * TC_STAGES;                // resident weights landed
    const uint32_t SFULL = WRES + 8u;                            // a tile's epilogue operands landed
    const uint32_t SFREE = SFULL + 8u;                           // the MMA warpgroups hold them in registers
    const int tid = threadIdx.x;
    const int n_tile = (int)blockIdx.x % L.ntiles_n, m_first = (int)blockIdx.x / L.ntiles_n;
    const int m_step = (int)gridDim.x / L.ntiles_n;
    const int nsteps = (L.ntiles_m - m_first + m_step - 1) / m_step * nkb;   // step j: m-tile m_first + j / nkb * m_step,
                                                                             // K-block j % nkb, ring stage j % S

    if (tid == 0) {
        for (int s = 0; s < S; s++) {
            mbar_init(FULL + 8u * s, NPROD + (L.resident ? 0 : 1));   // + the weights' expect_tx arrival
            mbar_init(EMPTY + 8u * s, TC_CONSUMERS);
        }
        mbar_init(WRES, 1);
        mbar_init(SFULL, NPROD);                                  // one cp.async arrival per producer thread
        mbar_init(SFREE, TC_CONSUMERS);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (tid >= TC_CONSUMERS) {
        // ============================= producer warpgroup(s): loads and in-place conversion =============================
        setmaxnreg_dec<TcRoles<NT>::producer_regs>();
        const int ptid = tid - TC_CONSUMERS;
        // K-block kb, tap t of the n-tile: rows [part * NT, part * NT + NT) of image (n-tile of the voice, kb, t)
        const int vf = L.wnt / NT;
        const size_t w_image = (size_t)L.wnt * 128u;
        const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(a.wtc) + (size_t)(n_tile / vf) * nkb * a.ntaps * w_image +
                              (size_t)(n_tile % vf) * w_tap;
        // images [kb0 * ntaps, (kb0 + nkb_) * ntaps) to dst, completion on bar
        auto issue_w = [&](int kb0, int nkb_, uint32_t dst, uint32_t bar) {
            if (ptid == 0) {
                mbar_expect_tx(bar, (uint32_t)nkb_ * w_kb);
                for (int i = 0; i < nkb_ * a.ntaps; i++)
                    bulk_g2s(dst + i * w_tap, wsrc + (size_t)(kb0 * a.ntaps + i) * w_image, w_tap, bar);
            }
        };
        // window of step j: raw fp32 rows, linear (row r at r * 128 B)
        auto issue_a = [&](int j, int s) {
            const int kb = j % nkb, rbase = (m_first + j / nkb * m_step) * 128 + a.min_off;
            for (int idx = ptid; idx < L.win * 8; idx += NPROD) {
                const int gr = rbase + (idx >> 3);
                const bool ok = gr >= 0 && gr < a.rows_in;
                const float* src = ok ? a.x + (size_t)gr * a.ldx + kb * 32 + (idx & 7) * 4 : a.x;
                cp_async16(A0 + s * a_buf + (uint32_t)idx * 16u, src, ok ? 16u : 0u);
            }
            cp_async_commit();
        };
        // epilogue operands of the CTA's tile t, once the MMA warpgroups have taken tile t - 1's: 16-byte pieces of the
        // residual and of the accumulated output (columns < split from y0 when acc0, >= split from y1 when acc1), rows
        // past the array and sides that are not accumulated zero-filled; completion on SFULL
        // A thread keeps one 16-byte column piece and walks the rows (NT = 96: 240 of the 256 threads, 10 rows a pass).
        // Its per-thread values are recomputed per tile from an opaque copy of ptid: the producers' 32 / 40 registers do
        // not hold them across the window loop.
        constexpr int CPR = NT / 4, RSTEP = NPROD / CPR;     // pieces per row; rows per pass
        auto issue_stage = [&](int t) {
            if (t > 0) mbar_wait<false>(SFREE, (uint32_t)((t - 1) & 1));
            const int pt = (int)opaque((uint32_t)ptid);
            if (pt < RSTEP * CPR) {
                const int col = 4 * (pt % CPR), nb = n_tile * NT + col;
                const bool lo_side = nb < a.split;
                const bool rd_res = a.res && nb < a.cout, rd_acc = (lo_side ? a.acc0 : a.acc1) && nb < a.cout;
                const float* acc_src = lo_side ? a.y0 + nb : a.y1 + (nb - a.split);
                const int ld_acc = lo_side ? a.ldy0 : a.ldy1;
                for (int r = pt / CPR; r < 128; r += RSTEP) {
                    const int q = (m_first + t * m_step) * 128 + r;
                    const size_t orow = (size_t)q * a.orow_mul + a.orow_add;
                    const bool ok_res = rd_res && q < a.rows_q, ok_acc = rd_acc && q < a.rows_q;
                    if (a.res) cp_async16(stg_addr(SRES, r, col), ok_res ? a.res + nb + orow * a.ldres : a.x, ok_res ? 16u : 0u);
                    if (acc_any) cp_async16(stg_addr(SACC, r, col), ok_acc ? acc_src + orow * ld_acc : a.x, ok_acc ? 16u : 0u);
                }
            }
            cp_async_commit();
            cp_async_mbar_arrive(SFULL);
        };

        // weights are constants: fetched before the predecessor finishes
        if (L.resident) issue_w(0, nkb, W0, WRES);
        else issue_w(0, 1, W0, FULL);
        pdl_wait();

        // Step j refills stage j % 2 once the MMA warpgroups have released it (step j - 2), and loads and converts it
        // while they run step j - 1.  Tile t's epilogue operands are issued at step t * nkb + 1, after that step's window
        // (so they never hold it up), when tile t - 1's epilogue has just taken its operands: they land while tile t's
        // MMAs run.  With one K-block per tile, the last tile's go out after the loop.
        for (int j = 0; j < nsteps; j++) {
            const int s = j & 1;
            if (j >= S) mbar_wait<false>(EMPTY + 8u * s, (uint32_t)((j / S - 1) & 1));
            if (!L.resident && j > 0) issue_w(j % nkb, 1, W0 + s * w_kb, FULL + 8u * s);
            issue_a(j, s);
            if (stage && j > 0 && (j - 1) % nkb == 0) {
                issue_stage((j - 1) / nkb);
                cp_async_wait<1>();              // the window; the staged operands complete on SFULL
            } else {
                cp_async_wait<0>();
            }
            named_bar_sync(1, NPROD);            // every producer's part of the window has landed
            // in-place conversion, 32-byte pieces (8 channels); the four lanes of a row sit in one warp: all read, then
            // write.  Odd rows take their two 16-byte chunks in the opposite order (bank-conflict-free quarter-warps).
            const uint32_t img = A0 + s * a_buf;
            const int npiece = L.win * 4;
            const float slope = a.in_slope;
            for (int base = 0; base < npiece; base += NPROD) {
                const int idx = base + ptid;
                const bool live = idx < npiece;
                const uint32_t odd = (uint32_t)(idx >> 2) & 1u;
                float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
                if (live) {
                    const float4 t0 = lds128(img + (uint32_t)idx * 32u + odd * 16u);
                    const float4 t1 = lds128(img + (uint32_t)idx * 32u + 16u - odd * 16u);
                    v0 = odd ? t1 : t0;
                    v1 = odd ? t0 : t1;
                }
                __syncwarp();
                if (live) {
                    const int r = idx >> 2, cc = idx & 3;
                    float e[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
                    if (slope != 1.f) {
#pragma unroll
                        for (int i = 0; i < 8; i++) e[i] = fmaxf(e[i], e[i] * slope);   // leaky ReLU, 0 < slope < 1
                    }
                    uint4 hi, lo;
                    hi.x = split2(e[0], e[1], lo.x);
                    hi.y = split2(e[2], e[3], lo.y);
                    hi.z = split2(e[4], e[5], lo.z);
                    hi.w = split2(e[6], e[7], lo.w);
                    const uint4 first = odd ? lo : hi, second = odd ? hi : lo;
                    sts128u(sw128(img, r, cc + 4 * (int)odd), first);
                    sts128u(sw128(img, r, cc + 4 - 4 * (int)odd), second);
                }
            }
            mbar_arrive(FULL + 8u * s);
        }
        if (stage && nkb == 1) issue_stage(nsteps - 1);
        cp_async_wait<0>();
        return;
    }

    // ================================ two MMA warpgroups: fragments, wgmma, epilogue ================================
    setmaxnreg_inc<TcRoles<NT>::consumer_regs>();
    pdl_wait();
    const int warp = tid >> 5, lane = tid & 31;
    const int wg = warp >> 2, g = lane >> 2, c = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + g;       // tile rows r0 and r0 + 8 of this thread
    float acc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; i++) acc[i] = 0.f;

    const int n0 = n_tile * NT;
    const bool gate = a.act == ACT_GATE;
    const bool grouped = L.pairs && !gate;
    // Grouped epilogue: both columns of a pair on one side of the split (split is even), the per-element rule of the
    // general path 8 bytes at a time.  A group of the thread's pairs issues all its global reads before any of them
    // stores: the compiler may not move a load above a store to a buffer that could alias it, so interleaved, every
    // pair would wait for a memory round trip of its own.  On tiles wider than 32 columns, the first group's reads go out
    // before the tile's last K-block runs its MMAs, and each later group's before the previous group stores.  Staged
    // launches (L.stage) take a group's operands from the staging buffer the producers filled during the MMAs instead.
    constexpr int NP = NT / 8, G = NT == 32 ? 4 : 8, NG = 2 * NP / G;   // pairs per row; pairs per group; groups
    constexpr bool EARLY = NT > 32;     // at 2 CTAs per SM (96 registers), one group's reads at a time, after the MMAs
    const bool early = EARLY && grouped && !stage;
    bool live[2], valid[2];
    const float* bias[2];
    size_t orow0[2];
    auto load_group = [&](int k0, float2 (&rv)[G], float2 (&dv)[G]) {
#pragma unroll
        for (int i = 0; i < G; i++) {
            const int h = (k0 + i) / NP, nb = n0 + 8 * ((k0 + i) % NP) + 2 * c;
            rv[i] = dv[i] = make_float2(0.f, 0.f);
            if (!live[h] || nb >= a.cout || !valid[h]) continue;
            const bool lo_side = nb < a.split;
            if (a.res) rv[i] = *reinterpret_cast<const float2*>(a.res + orow0[h] * a.ldres + nb);
            if (lo_side ? a.acc0 : a.acc1)
                dv[i] = *reinterpret_cast<const float2*>(lo_side ? a.y0 + orow0[h] * a.ldy0 + nb
                                                                 : a.y1 + orow0[h] * a.ldy1 + (nb - a.split));
        }
    };
    // stg_addr(base, r0 + 8h, 8p + 2c) = base + thread part + (h, p, g >> 1) part.  The thread part and g >> 1 pass
    // through an opaque move per tile (`opaque`), so the compiler computes each pair's address where it is read instead
    // of keeping all of them in registers across the tile loop.
    const uint32_t stg_thread = (uint32_t)r0 * 128u + ((uint32_t)((c >> 1) ^ (g & 1)) << 4) + 8u * (uint32_t)(c & 1);
    auto lds_group = [&](int k0, uint32_t thr, uint32_t gh, float2 (&rv)[G], float2 (&dv)[G]) {
#pragma unroll
        for (int i = 0; i < G; i++) {
            const int h = (k0 + i) / NP, p = (k0 + i) % NP;
            const uint32_t off = thr + (uint32_t)(p >> 2) * 16384u + (uint32_t)h * 1024u + (((uint32_t)(p & 3) ^ gh) << 5);
            if (a.res) rv[i] = lds64(SRES + off);
            if (acc_any) dv[i] = lds64(SACC + off);
        }
    };
    auto store_group = [&](int k0, const float2 (&rv)[G], const float2 (&dv)[G]) {
#pragma unroll
        for (int i = 0; i < G; i++) {
            const int h = (k0 + i) / NP, p = (k0 + i) % NP, nb = n0 + 8 * p + 2 * c;
            if (!live[h] || nb >= a.cout) continue;
            float o[2] = {acc[4 * p + 2 * h], acc[4 * p + 2 * h + 1]};
            if (bias[h]) { o[0] += bias[h][nb]; o[1] += bias[h][nb + 1]; }
            if (a.act == ACT_RELU) { o[0] = fmaxf(o[0], 0.f); o[1] = fmaxf(o[1], 0.f); }
            const bool lo_side = nb < a.split;
            const int accum = lo_side ? a.acc0 : a.acc1;
            if (accum && !valid[h]) continue;
            float2 m = make_float2(0.f, 0.f);
            if (a.res && valid[h]) { m.x = rv[i].x * a.scale; m.y = rv[i].y * a.scale; }
            if (accum && valid[h]) { m.x += dv[i].x; m.y += dv[i].y; }
            *reinterpret_cast<float2*>(lo_side ? a.y0 + orow0[h] * a.ldy0 + nb : a.y1 + orow0[h] * a.ldy1 + (nb - a.split)) =
                valid[h] ? make_float2(fmaf(o[0], a.scale, m.x), fmaf(o[1], a.scale, m.y)) : make_float2(0.f, 0.f);
        }
    };

    for (int j = 0; j < nsteps; j++) {
        const int s = j & 1, kb = j % nkb;
        const int m_tile = m_first + j / nkb * m_step;
        const bool last_kb = kb == nkb - 1;
        float2 rv[2][G], dv[2][G];
        auto rows_of_tile = [&]() {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int q = m_tile * 128 + r0 + 8 * h;
                live[h] = q < a.rows_q;
                valid[h] = false;
                bias[h] = live[h] ? conv_row(a, q, valid[h]) : nullptr;
                orow0[h] = (size_t)q * a.orow_mul + a.orow_add;
            }
        };
        if (early && last_kb) {
            rows_of_tile();
            load_group(0, rv[0], dv[0]);
        }
        mbar_wait<false>(FULL + 8u * s, (uint32_t)((j >> 1) & 1));
        if (L.resident && j == 0) mbar_wait<false>(WRES, 0);
        const uint32_t img = A0 + s * a_buf;
        const uint32_t wst = L.resident ? W0 + kb * w_kb : W0 + s * w_kb;
        auto load_frag = [&](int t, uint32_t (&ah)[2][4], uint32_t (&al)[2][4]) {
            const int R0 = r0 + a.tap_off[t] - a.min_off, R1 = R0 + 8;
#pragma unroll
            for (int ks = 0; ks < 2; ks++) {
                ah[ks][0] = lds32(sw128(img, R0, 2 * ks) + 4u * c);
                ah[ks][1] = lds32(sw128(img, R1, 2 * ks) + 4u * c);
                ah[ks][2] = lds32(sw128(img, R0, 2 * ks + 1) + 4u * c);
                ah[ks][3] = lds32(sw128(img, R1, 2 * ks + 1) + 4u * c);
                al[ks][0] = lds32(sw128(img, R0, 4 + 2 * ks) + 4u * c);
                al[ks][1] = lds32(sw128(img, R1, 4 + 2 * ks) + 4u * c);
                al[ks][2] = lds32(sw128(img, R0, 5 + 2 * ks) + 4u * c);
                al[ks][3] = lds32(sw128(img, R1, 5 + 2 * ks) + 4u * c);
            }
        };
        auto mma_tap = [&](int t, const uint32_t (&ah)[2][4], const uint32_t (&al)[2][4]) {
            const uint32_t wimg = wst + t * w_tap;
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < 2; ks++) {                // two K = 16 steps inside the 64-byte hi half
                const uint64_t dwh = sw128_desc(wimg + 32u * ks);
                const uint64_t dwl = sw128_desc(wimg + 64u + 32u * ks);   // lo half starts at byte 64
                wgmma_rs<WG_BF16, NT>(acc, ah[ks], dwh);
                wgmma_rs<WG_BF16, NT>(acc, al[ks], dwh);
                wgmma_rs<WG_BF16, NT>(acc, ah[ks], dwl);
            }
            wg_commit();
        };
        // even taps use fragment set 0, odd taps set 1; after a tap is issued, wait_group 1 retires the tap before it,
        // whose set the next tap reloads.  The issue order per accumulator is (tap, K step, hi*hi, lo*hi, hi*lo).
        uint32_t ah0[2][4], al0[2][4], ah1[2][4], al1[2][4];
        acc_fence<NT / 2>(acc);
        for (int t = 0; t < a.ntaps; t += 2) {
            load_frag(t, ah0, al0);
            mma_tap(t, ah0, al0);
            wg_wait1();
            if (t + 1 < a.ntaps) {
                load_frag(t + 1, ah1, al1);
                mma_tap(t + 1, ah1, al1);
                wg_wait1();
            }
        }
        wg_wait0();
        acc_fence<NT / 2>(acc);
        mbar_arrive(EMPTY + 8u * s);                    // stage s fully read: the producer may refill it
        if (!last_kb) continue;

        // ===================== epilogue: thread owns rows r0, r0 + 8 and column pairs 8p + 2c =====================
        if (grouped && stage) {
            rows_of_tile();
            mbar_wait<false>(SFULL, (uint32_t)((j / nkb) & 1));
            const uint32_t thr = opaque(stg_thread), gh = opaque((uint32_t)g >> 1);
#pragma unroll
            for (int k = 0; k < NG; k++) {
                lds_group(k * G, thr, gh, rv[0], dv[0]);
                if (k == NG - 1) mbar_arrive(SFREE);    // the producers may stage the next tile
                store_group(k * G, rv[0], dv[0]);
            }
        } else if (grouped) {
            if (!EARLY) {
                rows_of_tile();
                load_group(0, rv[0], dv[0]);
            }
#pragma unroll
            for (int k = 0; k < NG; k++) {
                const int b = EARLY ? k & 1 : 0;
                if (EARLY && k + 1 < NG) load_group((k + 1) * G, rv[b ^ 1], dv[b ^ 1]);
                if (!EARLY && k > 0) load_group(k * G, rv[0], dv[0]);
                store_group(k * G, rv[b], dv[b]);
            }
        } else {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int q = m_tile * 128 + r0 + 8 * h;
                if (q >= a.rows_q) continue;
                bool valid;
                const float* bias = conv_row(a, q, valid);
                const size_t orow0 = (size_t)q * a.orow_mul + a.orow_add;
#pragma unroll
                for (int p = 0; p < NT / 8; p++) {
                    const int nb = n0 + 8 * p + 2 * c;      // bias / weight column of the pair's first element
                    if (nb >= a.cout) continue;
                    float o[2] = {acc[4 * p + 2 * h], acc[4 * p + 2 * h + 1]};
                    if (bias) { o[0] += bias[nb]; o[1] += bias[nb + 1]; }
                    if (gate) {
                        // the pair (2k, 2k+1) gives output column k
                        a.y0[orow0 * a.ldy0 + (nb >> 1)] = valid ? tanhf(o[0]) * (1.f / (1.f + expf(-o[1]))) * a.scale : 0.f;
                        continue;
                    }
                    if (a.act == ACT_RELU) { o[0] = fmaxf(o[0], 0.f); o[1] = fmaxf(o[1], 0.f); }
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const int n = nb + e;
                        const bool lo_side = n < a.split;
                        const int accum = lo_side ? a.acc0 : a.acc1;
                        if (accum && !valid) continue;      // accumulated buffers keep their zeros in gap rows
                        float m = 0.f;
                        if (a.res && valid) m = a.res[orow0 * a.ldres + n] * a.scale;
                        float* dst = lo_side ? a.y0 + orow0 * a.ldy0 + n : a.y1 + orow0 * a.ldy1 + (n - a.split);
                        if (accum && valid) m += *dst;
                        *dst = valid ? fmaf(o[e], a.scale, m) : 0.f;
                    }
                }
            }
        }
#pragma unroll
        for (int i = 0; i < NT / 2; i++) acc[i] = 0.f;
    }
}

// Two window stages; every K-block's images when resident (nkb <= TC_STAGES: never more than the ring's two stages),
// else two stages; `staged` epilogue operands.  The barriers sit in the alignment slack.
size_t smem_bytes(const ConvArgs& a, int nt, int win, bool resident, int staged) {
    const size_t w_kb = (size_t)a.ntaps * nt * 128;
    return (size_t)TC_STAGES * win * 128 + (resident ? (size_t)(a.cin / 32) : (size_t)TC_STAGES) * w_kb +
           (size_t)staged * 128 * nt * 4;
}

template <int NT> void allow_smem() {
    static PerDeviceOnce once;
    once.run([] { cudaFuncSetAttribute(conv_tc_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024); });
}

template <int NT> int occupancy(size_t smem) {
    allow_smem<NT>();
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, conv_tc_kernel<NT>, TcRoles<NT>::threads, smem) != cudaSuccess) {
        cudaGetLastError();
        n = 0;
    }
    return n;
}

// CTAs of conv_tc_kernel<nt> with `smem` bytes of dynamic shared memory that fit on one SM: the occupancy API's answer,
// cached per (nt, smem KB) -- every plan's smem is a multiple of 1024, so the KB is exact.  Without a
// device, the kernel's register bound (TcRoles::ctas) and that of the 228 KB of shared memory per SM (1 KB of it
// reserved per CTA).
int ctas_per_sm(int nt, size_t smem) {
    static int cache[4][256];
    int& slot = cache[nt / 32 - 1][std::min<size_t>(smem >> 10, 255)];
    int n = __atomic_load_n(&slot, __ATOMIC_RELAXED);
    if (n > 0) return n;
    switch (nt) {
        case 32: n = occupancy<32>(smem); break;
        case 64: n = occupancy<64>(smem); break;
        case 96: n = occupancy<96>(smem); break;
        default: n = occupancy<128>(smem); break;
    }
    if (n > 0) {
        __atomic_store_n(&slot, n, __ATOMIC_RELAXED);
        return n;
    }
    const int by_regs = nt == 32 ? TcRoles<32>::ctas : TcRoles<128>::ctas;
    return std::max(1, std::min(by_regs, (int)((228u * 1024u) / (smem + 1024))));
}

bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }
bool aligned16(const void* p, int ld) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0 && ld % 4 == 0; }

// Epilogue operands the producers can stage in 16-byte pieces: 0 (nothing to read, gate, or misaligned), 1 or 2.
int staged_operands(const ConvArgs& a, const TcLaunch& L) {
    const bool acc = a.acc0 || a.acc1;
    if (!L.pairs || (!a.res && !acc) || a.split % 4) return 0;
    if (a.res && !aligned16(a.res, a.ldres)) return 0;
    if ((a.acc0 && !aligned16(a.y0, a.ldy0)) || (a.acc1 && !aligned16(a.y1, a.ldy1))) return 0;
    return (a.res ? 1 : 0) + (acc ? 1 : 0);
}

bool plan(const ConvArgs& a, TcLaunch& L, size_t& smem) {
    if (!a.wtc || a.tc_nt <= 0 || a.tc_nt > 128 || a.tc_nt % 32) return false;
    L.wnt = a.tc_nt;
    L.win = (128 + a.span + 7) & ~7;
    const int mt = (a.rows_q + 127) / 128;
    // The widest part of an image whose two ring stages fit; on small launches (a single utterance) the narrowest part
    // that still leaves no more tiles than SMs, so that more SMs share the work.  Tile width changes no summation order:
    // an utterance comes out bit-identical whether it is synthesised alone or in a batch.
    L.nt = 0;
    for (int nt = a.tc_nt; nt >= 32; nt -= 32)
        if (a.tc_nt % nt == 0 && smem_bytes(a, nt, L.win, false, 0) <= WG_SMEM_BUDGET) { L.nt = nt; break; }
    if (!L.nt) return false;
    if (a.cout % a.tc_nt == 0)
        for (int nt = 32; nt < L.nt; nt += 32)
            if (L.nt % nt == 0 && mt * (a.cout / nt) <= wg_num_sms()) { L.nt = nt; break; }
    L.ntiles_m = mt;
    L.ntiles_n = (a.cout + L.nt - 1) / L.nt;
    L.resident = a.cin / 32 <= TC_STAGES;
    L.pairs = a.act != ACT_GATE && a.split % 2 == 0 && aligned8(a.y0) && aligned8(a.y1) &&
              a.ldy0 % 2 == 0 && a.ldy1 % 2 == 0 && (!a.res || (aligned8(a.res) && a.ldres % 2 == 0));
    smem = smem_bytes(a, L.nt, L.win, L.resident, 0) + 1024;
    // Staged epilogue operands only where they fit beside the ring at the same tile width and CTAs per SM, and only on
    // tiles wider than 32 columns: two 32-column CTAs per SM with staging take 227 of the SM's 228 KB of shared memory,
    // which leaves the smallest L1 carve-out, and the 32-channel ResBlocks ran 3-7 % slower staged (DESIGN.md section 3).
    const int nst = staged_operands(a, L);
    const size_t staged = smem_bytes(a, L.nt, L.win, L.resident, nst) + 1024;
    L.stage = L.nt > 32 && nst > 0 && staged - 1024 <= WG_SMEM_BUDGET && ctas_per_sm(L.nt, staged) == ctas_per_sm(L.nt, smem);
    if (L.stage) smem = staged;
    // Persistent grid: every CTA that fits at once, rounded down to whole m-tiles (a CTA keeps its n-tile); a launch of
    // no more tiles than that runs one tile per CTA.
    int grid = wg_num_sms() * ctas_per_sm(L.nt, smem);
    if (g_conv_tc_grid_cap > 0) grid = std::min(grid, g_conv_tc_grid_cap);
    L.grid = std::min(std::max(L.ntiles_n, grid / L.ntiles_n * L.ntiles_n), L.ntiles_m * L.ntiles_n);
    return true;
}

template <int NT> void launch_nt(const ConvArgs& a, const TcLaunch& L, size_t smem, cudaStream_t st) {
    allow_smem<NT>();
    launch_pdl(conv_tc_kernel<NT>, dim3(L.grid), dim3(TcRoles<NT>::threads), smem, st, a, L);
}

uint16_t bf16_rn_host(float f) {
    uint32_t b; memcpy(&b, &f, 4);
    b += 0x7fffu + ((b >> 16) & 1u);
    return (uint16_t)(b >> 16);
}
float bf16_to_float_host(uint16_t h) {
    uint32_t b = (uint32_t)h << 16; float f; memcpy(&f, &b, 4); return f;
}

}  // namespace

// planning only (no launch): the configuration the launcher would choose; see sb200_debug_plan
bool conv_tc_plan_info(const ConvArgs& a, int* out, int* staging_bytes) {
    TcLaunch L{}; size_t smem = 0;
    if (a.cin % 32 || a.cout % 32 || a.ntaps > SB_MAX_TAPS || !plan(a, L, smem)) return false;
    const int v[16] = {L.nt, L.wnt, L.ntiles_m, L.ntiles_n, TC_STAGES, (int)smem, L.win, L.grid, L.resident,
                       ctas_per_sm(L.nt, smem), 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 16; i++) out[i] = v[i];
    if (staging_bytes) *staging_bytes = L.stage ? staged_operands(a, L) * 128 * L.nt * 4 : 0;
    return true;
}

// plans ONCE and launches; false (nothing launched) when the shape is not supported
bool try_launch_conv_tc(const ConvArgs& a, cudaStream_t st) {
    if (a.cin % 32 || a.cout % 32 || a.ntaps > SB_MAX_TAPS) return false;
    if ((a.ldx & 3) || (reinterpret_cast<uintptr_t>(a.x) & 15)) return false;     // 16-byte cp.async window rows
    TcLaunch L; size_t smem;
    if (!plan(a, L, smem)) return false;
    switch (L.nt) {
        case 32: launch_nt<32>(a, L, smem, st); break;
        case 64: launch_nt<64>(a, L, smem, st); break;
        case 96: launch_nt<96>(a, L, smem, st); break;
        default: launch_nt<128>(a, L, smem, st); break;
    }
    g_launch_count++;
    check_launch("conv_tc");
    return true;
}

// Host-side weight image builder: [n-tile][K-block][tap] images of nt rows x 128 B, row n =
// [hi: 32 ch bf16 | lo: 32 ch bf16] in the K-major SWIZZLE_128B layout (16-B chunk c at (c ^ (n & 7))).
// Sizes are in floats (4-byte units) because the voice arena is a float arena.
size_t conv_tc_weight_floats(int cin, int cout, int ntaps, int nt) {
    const int ntiles = (cout + nt - 1) / nt;
    return (size_t)ntiles * (cin / 32) * ntaps * nt * 32;
}

void conv_tc_build_weights(const float* wt /*[ntaps][cin][ldw]*/, int ldw, int cin, int cout, int ntaps, int nt,
                           float* out) {
    const int ntiles = (cout + nt - 1) / nt;
    const int nkb = cin / 32;
    uint16_t* o16 = reinterpret_cast<uint16_t*>(out);
    size_t o = 0;   // in bf16 elements
    for (int j = 0; j < ntiles; j++)
        for (int kb = 0; kb < nkb; kb++)
            for (int t = 0; t < ntaps; t++) {
                uint16_t* img = o16 + o;
                for (int n = 0; n < nt; n++)
                    for (int c = 0; c < 32; c++) {
                        const int col = j * nt + n;
                        const float v = col < cout ? wt[((size_t)t * cin + kb * 32 + c) * ldw + col] : 0.f;
                        const uint16_t h = bf16_rn_host(v);
                        const uint16_t l = bf16_rn_host(v - bf16_to_float_host(h));
                        const int ch = c >> 3, e = c & 7;                        // 16-B chunk (8 bf16) and element
                        img[(size_t)n * 64 + (size_t)((ch ^ (n & 7)) << 3) + e] = h;
                        img[(size_t)n * 64 + (size_t)(((ch + 4) ^ (n & 7)) << 3) + e] = l;
                    }
                o += (size_t)nt * 64;
            }
}

}  // namespace sb200
