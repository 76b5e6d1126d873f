// wgmma implicit-GEMM Conv1d in error-compensated TF32 ("3xTF32") with CHUNK-FLUSHED accumulation, sm_90a.
//
// Used for the contractions whose result reaches the duration predictor: text-encoder qkv / o / ffn / proj and the
// duration predictor's 1x1 convs (what onnxruntime's MLAS SGEMM computes inside `session.run`,
// piper/src/lib.rs:362-379).  ceil(exp(logw)) is a cliff (SURVEY fact 4), so these layers need fp32-class accuracy:
//   * operands are split  v = hi + lo,  hi = v with the low 13 mantissa bits cleared (exactly a tf32 number),
//     lo = tf32_rn(v - hi); three MMAs accumulate  hi*hi + lo*hi + hi*lo  (the dropped lo*lo term is 2^-22);
//   * the tensor core's fp32 accumulation loses accuracy as the number of accumulating MMAs grows.  The K loop is
//     therefore cut into chunks of 64 channels (1x1 convs) or 32 channels x k taps; each chunk accumulates into a
//     fresh register accumulator that is then added into a round-to-nearest fp32 running sum.
//     tools/emu_tc_accuracy.py: max error of a K = 2304 contraction 2.5e-6 vs 5.4e-6 for the fp32 FMA chain of
//     conv_simt.cu and 8.4e-5 without the flush.
//
// One CTA = one 128-row x NT-column tile (NT = 96 / 64 / 32), two warpgroups (rows 0-63 / 64-127), a two-stage ring
// over 32-channel K-blocks:
//   * activations: the raw fp32 (128 + span)-row window arrives by cp.async straight into the K-major SWIZZLE_128B
//     layout (32 fp32 = one 128-byte row, rows / columns outside the array zero-filled); all threads rewrite it as the
//     hi image in place and write the lo image beside it (same swizzled offsets: the conversion is element-wise).
//     The A operand comes from registers (wgmma with A in registers), loaded from any row offset: a tap is a shift.
//   * weights: hi / lo images pre-split at voice-load time, one cp.async.bulk (TMA) per image, mbarrier completion.
//   * epilogue: bias / ReLU / residual / scale / accumulate (or a transposed store) from the running sums.
//
// GM = 1 ("grouped GEMM", the two contractions of the relative-position attention): the B operand is not a pre-split
// weight image but a second ACTIVATION matrix (K for Q.K^T, V^T for P.V), loaded and split like A; tiles come from a
// host-built table (one entry per (utterance, head, m-tile pair, n-tile) with its own K extent), so ragged batches need
// no padding.  A CTA takes one m-tile of a table entry.  A K extent that ends inside a 32-column K-block (48-wide heads:
// Q.K^T has K = 48) zero-fills the rest of that block in BOTH operands: the columns beyond are the next head's
// activations, not zeros.  48-wide heads also give P.V its 48-column tiles (m64n48k8).
#include "tc_common.cuh"
#include <stdlib.h>
#include <string.h>

namespace sb200 {

namespace {

using namespace tcx;

constexpr int TF_THREADS = 256;
constexpr int TF_STAGES = 2;

struct TfLaunch {
    int nth;         // columns of a tile: 96 / 64 / 32 (grouped GEMM also 48)
    int wnth;        // rows of a weight IMAGE (tf_nth_for); nth == wnth, or 32 on small launches: the CTA then takes a 32-row
                     // part of the hi image and of the lo image (32 % 8 == 0 keeps the swizzle)
    int win;         // window rows (multiple of 8)
    int ntiles_m, ntiles_n;
    int chunk_kb;    // K-blocks per flush chunk
};

// GM = 1 operands: A [a_rows][a_cols] and B [b_rows][b_cols] (rows = output columns), K along the columns
struct TfOperands {
    const float* a; int a_rows, a_cols, lda;
    const float* b; int b_rows, b_cols, ldb;
    const TfTile* tiles;
};

__device__ __forceinline__ float tf32_rn(float v) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return __uint_as_float(r);
}

template <int GM, int NT>
__global__ void __launch_bounds__(TF_THREADS, 1) conv_tf_kernel(const ConvArgs a, const TfLaunch L, const TfOperands G) {
    pdl_trigger();
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int ntaps = GM ? 1 : a.ntaps;
    const uint32_t a_img = (uint32_t)L.win * 128u;               // one image (hi or lo) of a window
    const uint32_t w_img = (uint32_t)NT * 128u;                  // one image (hi or lo) of a tap
    const uint32_t w_buf = (uint32_t)ntaps * 2u * w_img;
    const uint32_t A0 = smem_u32(smem), W0 = A0 + TF_STAGES * 2 * a_img;   // [stage][hi | lo], [stage][tap][hi | lo]
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + TF_STAGES * (2 * a_img + w_buf));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    TfTile T{};
    int h = 0, m_tile = 0, n_tile = 0, nkb = a.cin / 32;
    if (GM) {
        T = G.tiles[blockIdx.x >> 1];
        h = (int)blockIdx.x & 1;
        nkb = T.nkb;
    } else {
        m_tile = (int)blockIdx.x / L.ntiles_n;
        n_tile = (int)blockIdx.x % L.ntiles_n;
    }
    if (tid == 0) {
        for (int s = 0; s < TF_STAGES; s++) mbar_init(smem_u32(&bars[s]), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // conv form: weight stage kb = (hi, lo) image pairs of every tap, rows [part * NT, +NT) of the voice's images
    const int vf = L.wnth / NT;
    const size_t src_img = (size_t)L.wnth * 128u;
    const uint8_t* wsrc = GM ? nullptr : reinterpret_cast<const uint8_t*>(a.wtf) + (size_t)(n_tile / vf) * nkb * ntaps * 2 * src_img +
                                         (size_t)(n_tile % vf) * w_img;
    auto issue_w = [&](int kb, int s) {
        if (tid == 0) {
            const uint32_t bar = smem_u32(&bars[s]);
            mbar_expect_tx(bar, w_buf);
            for (int t = 0; t < ntaps; t++) {
                const uint8_t* st = wsrc + (size_t)(kb * ntaps + t) * 2 * src_img;
                bulk_g2s(W0 + s * w_buf + t * 2 * w_img, st, w_img, bar);
                bulk_g2s(W0 + s * w_buf + t * 2 * w_img + w_img, st + src_img, w_img, bar);
            }
        }
    };
    // rows [row0, row0 + nrows) x columns [col0, col0 + 32) of a [rows][cols] matrix -> swizzled raw image
    auto load_rows = [&](uint32_t img, const float* base, int ld, int rows, int cols, int row0, int col0, int nrows) {
        for (int idx = tid; idx < nrows * 8; idx += TF_THREADS) {
            const int r = idx >> 3, ch = idx & 7;
            const int gr = row0 + r, gc = col0 + ch * 4;
            const int nval = gr >= 0 && gr < rows ? min(max(cols - gc, 0), 4) : 0;
            cp_async16(sw128(img, r, ch), nval ? base + (size_t)gr * ld + gc : base, (uint32_t)nval * 4u);
        }
    };
    auto issue_a = [&](int kb, int s) {
        const uint32_t img = A0 + s * 2 * a_img;
        if (GM) {
            load_rows(img, G.a, G.lda, G.a_rows, min(G.a_cols, T.a_col0 + T.kcols), T.a_row0[h], T.a_col0 + kb * 32, 128);
            load_rows(W0 + s * w_buf, G.b, G.ldb, G.b_rows, min(G.b_cols, T.b_col0 + T.kcols), T.b_row0, T.b_col0 + kb * 32, NT);
        } else {
            load_rows(img, a.x, a.ldx, a.rows_in, a.cin, m_tile * 128 + a.min_off, kb * 32, L.win);
        }
        cp_async_commit();
    };
    // hi = v with 13 low mantissa bits cleared (in place), lo = tf32_rn(v - hi) at the same offset of the next image
    auto split_image = [&](uint32_t hi_img, uint32_t lo_img, int n16, float slope) {
        for (int idx = tid; idx < n16; idx += TF_THREADS) {
            float4 v = lds128(hi_img + (uint32_t)idx * 16u);
            if (slope != 1.f) {
                v.x = fmaxf(v.x, v.x * slope); v.y = fmaxf(v.y, v.y * slope);
                v.z = fmaxf(v.z, v.z * slope); v.w = fmaxf(v.w, v.w * slope);
            }
            uint4 hi, lo;
            hi.x = __float_as_uint(v.x) & 0xffffe000u; hi.y = __float_as_uint(v.y) & 0xffffe000u;
            hi.z = __float_as_uint(v.z) & 0xffffe000u; hi.w = __float_as_uint(v.w) & 0xffffe000u;
            lo.x = __float_as_uint(tf32_rn(v.x - __uint_as_float(hi.x)));
            lo.y = __float_as_uint(tf32_rn(v.y - __uint_as_float(hi.y)));
            lo.z = __float_as_uint(tf32_rn(v.z - __uint_as_float(hi.z)));
            lo.w = __float_as_uint(tf32_rn(v.w - __uint_as_float(hi.w)));
            sts128u(hi_img + (uint32_t)idx * 16u, hi);
            sts128u(lo_img + (uint32_t)idx * 16u, lo);
        }
    };

    if (!GM) issue_w(0, 0);                             // weights are constants: fetched before the predecessor finishes
    pdl_wait();
    issue_a(0, 0);

    const int wg = warp >> 2, g = lane >> 2, c = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + g;       // tile rows r0 and r0 + 8 of this thread
    float acc[NT / 2], run[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; i++) { acc[i] = 0.f; run[i] = 0.f; }

    for (int kb = 0; kb < nkb; kb++) {
        const int s = kb & 1;
        if (kb + 1 < nkb) {
            if (!GM) issue_w(kb + 1, s ^ 1);
            issue_a(kb + 1, s ^ 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const uint32_t ahi = A0 + s * 2 * a_img, alo = ahi + a_img;
        const uint32_t wst = W0 + s * w_buf;
        split_image(ahi, alo, L.win * 8, GM ? 1.f : a.in_slope);
        if (GM) split_image(wst, wst + w_img, NT * 8, 1.f);
        if (GM) fence_async_smem();
        __syncthreads();
        if (!GM) mbar_wait(smem_u32(&bars[s]), (uint32_t)((kb >> 1) & 1));
        for (int t = 0; t < ntaps; t++) {
            const int R0 = r0 + (GM ? 0 : a.tap_off[t] - a.min_off), R1 = R0 + 8;
            const uint32_t whi = wst + t * 2 * w_img, wlo = whi + w_img;
#pragma unroll
            for (int half = 0; half < 2; half++) {      // two K = 8 steps per register load
                uint32_t fh[2][4], fl[2][4];
#pragma unroll
                for (int u = 0; u < 2; u++) {
                    const int ks = 2 * half + u;
                    fh[u][0] = lds32(sw128(ahi, R0, 2 * ks) + 4u * c);
                    fh[u][1] = lds32(sw128(ahi, R1, 2 * ks) + 4u * c);
                    fh[u][2] = lds32(sw128(ahi, R0, 2 * ks + 1) + 4u * c);
                    fh[u][3] = lds32(sw128(ahi, R1, 2 * ks + 1) + 4u * c);
                    fl[u][0] = lds32(sw128(alo, R0, 2 * ks) + 4u * c);
                    fl[u][1] = lds32(sw128(alo, R1, 2 * ks) + 4u * c);
                    fl[u][2] = lds32(sw128(alo, R0, 2 * ks + 1) + 4u * c);
                    fl[u][3] = lds32(sw128(alo, R1, 2 * ks + 1) + 4u * c);
                }
                acc_fence<NT / 2>(acc);
                wg_fence();
#pragma unroll
                for (int u = 0; u < 2; u++) {
                    const int ks = 2 * half + u;
                    const uint64_t dwh = sw128_desc(whi + 32u * ks), dwl = sw128_desc(wlo + 32u * ks);
                    wgmma_rs<WG_TF32, NT>(acc, fh[u], dwh);
                    wgmma_rs<WG_TF32, NT>(acc, fl[u], dwh);
                    wgmma_rs<WG_TF32, NT>(acc, fh[u], dwl);
                }
                wg_commit();
                wg_wait0();
                acc_fence<NT / 2>(acc);
            }
        }
        if (kb % L.chunk_kb == L.chunk_kb - 1 || kb == nkb - 1) {   // chunk finished: flush into the running sums
#pragma unroll
            for (int i = 0; i < NT / 2; i++) { run[i] += acc[i]; acc[i] = 0.f; }
        }
        __syncthreads();                                // stage s fully read: the next iteration refills it
    }

    // ===================== epilogue: thread owns rows r0, r0 + 8 and column pairs 8j + 2c =====================
#pragma unroll
    for (int hh = 0; hh < 2; hh++) {
        const int row = r0 + 8 * hh;
        if (GM) {
            // grouped GEMM: out = acc * scale (+ res), rows of this m-tile that belong to the utterance only
            if (row >= T.rows_valid[h]) continue;
            float* dst = a.y0 + T.out_off[h] + (size_t)row * a.ldy0;
            const float* rsrc = a.res ? a.res + T.out_off[h] + (size_t)row * a.ldres : nullptr;
#pragma unroll
            for (int j = 0; j < NT / 8; j++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int n = 8 * j + 2 * c + e;
                    dst[n] = fmaf(run[4 * j + 2 * hh + e], a.scale, rsrc ? rsrc[n] : 0.f);
                }
            continue;
        }
        const int q = m_tile * 128 + row;
        if (q >= a.rows_q) continue;
        bool valid;
        const float* bias = conv_row(a, q, valid);
        const size_t orow = (size_t)q + a.orow_add;
#pragma unroll
        for (int j = 0; j < NT / 8; j++)
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int n = n_tile * NT + 8 * j + 2 * c + e;
                float o = run[4 * j + 2 * hh + e] + (bias ? bias[n] : 0.f);
                if (a.act == ACT_RELU) o = fmaxf(o, 0.f);
                if (a.yt && n >= a.yt_col0) {
                    // transposed output (V of the fused q/k/v projection: the P.V contraction wants keys contiguous)
                    a.yt[(size_t)(n - a.yt_col0) * a.ldyt + q] = valid ? o * a.scale : 0.f;
                    if (!a.yt_keep) continue;
                }
                if (a.acc0 && !valid) continue;         // accumulated buffers keep their zeros in gap rows
                float m = 0.f;
                if (a.res && valid) m = a.res[orow * a.ldres + n] * a.scale;
                if (a.acc0 && valid) m += a.y0[orow * a.ldy0 + n];
                a.y0[orow * a.ldy0 + n] = valid ? fmaf(o, a.scale, m) : 0.f;
            }
    }
}

// Column tile.  k-tap layers (ffn): 96 columns; 1x1 layers: 64 columns.  Images are built at this width.
int tf_nth_for(int cout, int ntaps) {
    if (ntaps == 1 && cout % 64 == 0) return 64;
    if (cout % 96 == 0) return 96;
    if (cout % 64 == 0) return 64;
    if (cout % 32 == 0) return 32;
    return 0;
}

size_t smem_bytes(int win, int ntaps, int nth) {
    return (size_t)TF_STAGES * (2 * (size_t)win * 128 + (size_t)ntaps * 2 * nth * 128) + TF_STAGES * 8;
}

bool plan(const ConvArgs& a, TfLaunch& L, size_t& smem) {
    if (!a.wtf || a.cin % 32 || a.cout % 32 || a.ntaps < 1 || a.ntaps > SB_MAX_TAPS) return false;
    if (a.act == ACT_GATE || a.split < a.cout || a.orow_mul != 1) return false;
    if ((a.ldx & 3) || (reinterpret_cast<uintptr_t>(a.x) & 15)) return false;
    L.nth = L.wnth = tf_nth_for(a.cout, a.ntaps);
    if (!L.nth) return false;
    L.win = (128 + a.span + 7) & ~7;
    if (smem_bytes(L.win, a.ntaps, 32) > WG_SMEM_BUDGET) return false;
    L.ntiles_m = (a.rows_q + 127) / 128;
    // Small launches (a single utterance), or a weight stage too large for two stages: 32-column parts of the images.
    // Tile width changes no summation order.
    if (L.wnth > 32 && (L.ntiles_m * (a.cout / 32) <= wg_num_sms() || smem_bytes(L.win, a.ntaps, L.wnth) > WG_SMEM_BUDGET))
        L.nth = 32;
    L.ntiles_n = a.cout / L.nth;
    L.chunk_kb = a.ntaps == 1 ? 2 : 1;
    smem = smem_bytes(L.win, a.ntaps, L.nth) + 1024;
    return true;
}

template <int GM, int NT> void launch_nt(dim3 grid, size_t smem, cudaStream_t st, const ConvArgs& a, const TfLaunch& L,
                                         const TfOperands& G) {
    static PerDeviceOnce once;
    once.run([] { cudaFuncSetAttribute(conv_tf_kernel<GM, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024); });
    launch_pdl(conv_tf_kernel<GM, NT>, grid, dim3(TF_THREADS), smem, st, a, L, G);
}

template <int GM> void launch_any(int nth, dim3 grid, size_t smem, cudaStream_t st, const ConvArgs& a, const TfLaunch& L,
                                  const TfOperands& G) {
    switch (nth) {
        case 32: launch_nt<GM, 32>(grid, smem, st, a, L, G); break;
        case 64: launch_nt<GM, 64>(grid, smem, st, a, L, G); break;
        default: launch_nt<GM, 96>(grid, smem, st, a, L, G); break;
    }
}

// the grouped GEMM also takes 48-column tiles (P.V of 48-wide attention heads)
void launch_gemm_any(int nth, dim3 grid, size_t smem, cudaStream_t st, const ConvArgs& a, const TfLaunch& L,
                     const TfOperands& G) {
    if (nth == 48) launch_nt<1, 48>(grid, smem, st, a, L, G);
    else launch_any<1>(nth, grid, smem, st, a, L, G);
}

uint32_t tf32_rn_host(float f) {        // round to nearest, ties away from zero (cvt.rna.tf32.f32)
    uint32_t b; memcpy(&b, &f, 4);
    if ((b & 0x7f800000u) == 0x7f800000u) return b;
    b += 0x1000u;
    return b & 0xffffe000u;
}

}  // namespace

// planning only (no launch): the configuration the launcher would choose; see sb200_debug_plan
bool conv_tf_plan_info(const ConvArgs& a, int* out) {
    TfLaunch L{}; size_t smem = 0;
    if (!plan(a, L, smem)) return false;
    const int v[16] = {L.nth, L.wnth, L.ntiles_m, L.ntiles_n, TF_STAGES, L.chunk_kb, (int)smem, L.win, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 16; i++) out[i] = v[i];
    return true;
}

// plans ONCE and launches; false (nothing launched) when the shape is not supported
bool try_launch_conv_tf(const ConvArgs& a, cudaStream_t st) {
    TfLaunch L; size_t smem;
    if (!plan(a, L, smem)) return false;
    launch_any<0>(L.nth, dim3(L.ntiles_m * L.ntiles_n), smem, st, a, L, TfOperands{});
    g_launch_count++;
    check_launch("conv_tf");
    return true;
}

bool gemm_tf_supported(const TfGemm& g) {
    if (g.nth != 96 && g.nth != 64 && g.nth != 48 && g.nth != 32) return false;
    auto al = [](const void* p, int ld) { return p == nullptr || ((reinterpret_cast<uintptr_t>(p) & 15) == 0 && (ld & 3) == 0); };
    return al(g.a, g.lda) && al(g.b, g.ldb);
}

void launch_gemm_tf(const TfGemm& g, cudaStream_t st) {
    if (g.ntiles <= 0) return;
    ConvArgs a{};
    a.in_slope = 1.f; a.ntaps = 1; a.cin = 32; a.cout = g.nth;
    a.y0 = g.y; a.ldy0 = g.ldy; a.res = g.res; a.ldres = g.ldy; a.scale = g.scale; a.split = g.nth; a.orow_mul = 1;
    TfLaunch L{};
    L.nth = L.wnth = g.nth; L.win = 128; L.ntiles_m = 2 * g.ntiles; L.ntiles_n = 1; L.chunk_kb = 2;
    const TfOperands G{g.a, g.a_rows, g.a_cols, g.lda, g.b, g.b_rows, g.b_cols, g.ldb, g.tiles};
    launch_gemm_any(g.nth, dim3(2 * g.ntiles), smem_bytes(128, 1, g.nth) + 1024, st, a, L, G);
    g_launch_count++;
    check_launch("gemm_tf");
}

// Host-side weight image builder: [n-tile][K-block][tap] stages; a stage = hi image (nth rows x 128 B) followed by the
// lo image; row n = 32 channels fp32 of output column n, K-major SWIZZLE_128B (16-byte chunk c at c ^ (n & 7)).
// hi = tf32_rn(w), lo = tf32_rn(w - hi).  Sizes in floats.
size_t conv_tf_weight_floats(int cin, int cout, int ntaps) {
    const int nth = tf_nth_for(cout, ntaps);
    if (!nth || cin % 32) return 0;
    return (size_t)(cout / nth) * (cin / 32) * ntaps * nth * 64;
}

void conv_tf_build_weights(const float* wt /*[ntaps][cin][ldw]*/, int ldw, int cin, int cout, int ntaps, float* out) {
    const int nth = tf_nth_for(cout, ntaps);
    const int ntiles = cout / nth, nkb = cin / 32;
    uint32_t* o32 = reinterpret_cast<uint32_t*>(out);
    size_t o = 0;
    for (int j = 0; j < ntiles; j++)
        for (int kb = 0; kb < nkb; kb++)
            for (int t = 0; t < ntaps; t++) {
                uint32_t* hi = o32 + o;
                uint32_t* lo = hi + (size_t)nth * 32;
                for (int n = 0; n < nth; n++)
                    for (int c = 0; c < 32; c++) {
                        const float v = wt[((size_t)t * cin + kb * 32 + c) * ldw + j * nth + n];
                        const uint32_t hb = tf32_rn_host(v);
                        float hf; memcpy(&hf, &hb, 4);
                        const uint32_t lb = tf32_rn_host(v - hf);
                        const size_t pos = (size_t)n * 32 + (size_t)(((c >> 2) ^ (n & 7)) << 2) + (c & 3);
                        hi[pos] = hb;
                        lo[pos] = lb;
                    }
                o += (size_t)nth * 64;
            }
}

}  // namespace sb200
