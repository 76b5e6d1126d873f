// fp32 CUDA-core implicit-GEMM Conv1d over time-major activations (see common.cuh for the op).
//
// This is the correctness reference for every dense contraction on the path (text-encoder 1x1 /
// k3 convs, duration-predictor 1x1s, WaveNet k5 convs, HiFi-GAN k3..k11 dilated convs and the
// polyphase ConvTranspose1d), i.e. what onnxruntime's MLAS im2col+SGEMM does on the reference
// side of `session.run` (piper/src/lib.rs:362-379).  The wgmma kernel (conv_tc.cu) implements
// the same ConvArgs contract for the big ResBlock / WaveNet contractions.
//
// Tiling: CTA = 256 threads, BM x BN output tile, K loop over (32-channel chunk, tap).
//   * the activation WINDOW (BM + span rows x 32 channels) is staged once per chunk in shared
//     memory and re-used by every tap (a k-tap conv reads its input once, not k times);
//   * weight tiles [32 x BN] stream through a cp.async double buffer;
//   * each thread owns TM x TN accumulators; both operands are read with 128-bit LDS.
#include "common.cuh"
#include <stdio.h>

namespace sb200 {

unsigned long long g_launch_count = 0;

namespace {

constexpr int BK = 32;
constexpr int AS_STRIDE = 36;   // floats; 144 B rows: 16 B aligned, conflict-free for LDS.128/STS.128

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async16_zfill(void* smem, const void* gmem, bool ok) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(ok ? 16u : 0u));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::); }

template <int VW> struct Vec;
template <> struct Vec<4> { using T = float4; };
template <> struct Vec<2> { using T = float2; };

template <int BM, int TX, int VW, int NV>
__global__ void __launch_bounds__(256, 2) conv_simt_kernel(const ConvArgs a) {
    pdl_trigger(); pdl_wait();
    constexpr int TY = 256 / TX;
    constexpr int TM = BM / TY;
    constexpr int TN = VW * NV;
    constexpr int BN = TX * TN;
    constexpr int CSTRIDE = TX * VW;   // column distance between a thread's vectors
    using V = typename Vec<VW>::T;

    extern __shared__ __align__(16) float smem[];
    const int win = BM + a.span;
    // With no leaky-ReLU prologue (in_slope == 1: encoder / duration-predictor GEMMs) the window of the NEXT
    // 32-channel chunk is prefetched with cp.async into a second buffer while the current chunk is computed; a
    // synchronous load exposed a full memory latency per chunk (every iteration for the k = 1 projections).
    const bool pfa = a.in_slope == 1.f;
    float* As0 = smem;
    float* Bs = smem + 2 * win * AS_STRIDE;

    const int tid = threadIdx.x;
    const int tx = tid % TX, ty = tid / TX;
    const int q0 = blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; i++)
#pragma unroll
        for (int j = 0; j < TN; j++) acc[i][j] = 0.f;

    const int nchunks = a.cin / BK;
    const int nit = nchunks * a.ntaps;

    auto issue_b = [&](int it, int buf) {
        const int chunk = it / a.ntaps, t = it - chunk * a.ntaps;
        const float* src = a.w + ((size_t)(t * a.cin + chunk * BK)) * a.ldw + n0;
        float* dst = Bs + buf * (BK * BN);
        constexpr int NCH = BK * BN / 4;
        for (int c = tid; c < NCH; c += 256) {
            const int kk = c / (BN / 4), n4 = c - kk * (BN / 4);
            cp_async16(dst + kk * BN + n4 * 4, src + (size_t)kk * a.ldw + n4 * 4);
        }
        cp_async_commit();
    };

    auto issue_a = [&](int chunk) {           // async window load of `chunk` (joins the next committed group)
        float* dstA = As0 + (chunk & 1) * (win * AS_STRIDE);
        const int c0 = chunk * BK;
        const int rbase = q0 + a.min_off;
        for (int idx = tid; idx < win * 8; idx += 256) {
            const int r = idx >> 3, c4 = idx & 7;
            const int gr = rbase + r;
            const bool ok = gr >= 0 && gr < a.rows_in;
            cp_async16_zfill(dstA + r * AS_STRIDE + c4 * 4, ok ? a.x + (size_t)gr * a.ldx + c0 + c4 * 4 : a.x, ok);
        }
    };
    if (pfa) issue_a(0);
    issue_b(0, 0);
    for (int it = 0; it < nit; it++) {
        const int chunk = it / a.ntaps, t = it - chunk * a.ntaps;
        const int buf = it & 1;
        float* As = As0 + (pfa ? (chunk & 1) * (win * AS_STRIDE) : 0);
        if (t == 0 && !pfa) {
            __syncthreads();   // everyone is done reading the previous window
            const int c0 = chunk * BK;
            const int rbase = q0 + a.min_off;
            for (int idx = tid; idx < win * 8; idx += 256) {
                const int r = idx >> 3, c4 = idx & 7;
                const int gr = rbase + r;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (gr >= 0 && gr < a.rows_in)
                    v = *reinterpret_cast<const float4*>(a.x + (size_t)gr * a.ldx + c0 + c4 * 4);
                const float s = a.in_slope;
                v.x = v.x > 0.f ? v.x : v.x * s;
                v.y = v.y > 0.f ? v.y : v.y * s;
                v.z = v.z > 0.f ? v.z : v.z * s;
                v.w = v.w > 0.f ? v.w : v.w * s;
                *reinterpret_cast<float4*>(As + r * AS_STRIDE + c4 * 4) = v;
            }
        }
        cp_async_wait_all();
        __syncthreads();       // weights(it) + window visible; compute(it-1) finished everywhere
        if (it + 1 < nit) {
            if (pfa && t + 1 == a.ntaps) issue_a(chunk + 1);     // buffer (chunk+1)&1 was last read in chunk-1: all done
            issue_b(it + 1, buf ^ 1);
        }

        const float* Ab = As + (ty + a.tap_off[t] - a.min_off) * AS_STRIDE;
        const float* Bb = Bs + buf * (BK * BN) + tx * VW;
#pragma unroll
        for (int k4 = 0; k4 < BK / 4; k4++) {
            float4 av[TM];
#pragma unroll
            for (int i = 0; i < TM; i++)
                av[i] = *reinterpret_cast<const float4*>(Ab + (i * TY) * AS_STRIDE + k4 * 4);
#pragma unroll
            for (int kk = 0; kk < 4; kk++) {
                float bv[TN];
#pragma unroll
                for (int v = 0; v < NV; v++) {
                    V b = *reinterpret_cast<const V*>(Bb + (k4 * 4 + kk) * BN + v * CSTRIDE);
                    if constexpr (VW == 4) { bv[v * 4] = b.x; bv[v * 4 + 1] = b.y; bv[v * 4 + 2] = b.z; bv[v * 4 + 3] = b.w; }
                    else { bv[v * 2] = b.x; bv[v * 2 + 1] = b.y; }
                }
#pragma unroll
                for (int i = 0; i < TM; i++) {
                    const float af = kk == 0 ? av[i].x : kk == 1 ? av[i].y : kk == 2 ? av[i].z : av[i].w;
#pragma unroll
                    for (int j = 0; j < TN; j++) acc[i][j] = fmaf(af, bv[j], acc[i][j]);
                }
            }
        }
    }

    // ---------------- epilogue ----------------
#pragma unroll
    for (int i = 0; i < TM; i++) {
        const int q = q0 + ty + i * TY;
        if (q >= a.rows_q) continue;
        bool valid;
        const float* bias = conv_row(a, q, valid);
        const size_t orow = (size_t)q * a.orow_mul + a.orow_add;
#pragma unroll
        for (int v = 0; v < NV; v++) {
            const int n = n0 + v * CSTRIDE + tx * VW;
            if (n >= a.cout) continue;
            float o[VW];
#pragma unroll
            for (int e = 0; e < VW; e++) o[e] = acc[i][v * VW + e] + (bias ? bias[n + e] : 0.f);
            if (a.act == ACT_GATE) {
                // columns are interleaved (tanh_j, sigmoid_j) pairs -> VW/2 outputs at column n/2
                float g[VW / 2];
#pragma unroll
                for (int e = 0; e < VW / 2; e++)
                    g[e] = valid ? tanhf(o[2 * e]) * (1.f / (1.f + expf(-o[2 * e + 1]))) * a.scale : 0.f;
                float* dst = a.y0 + orow * a.ldy0 + (n >> 1);
                if constexpr (VW == 4) *reinterpret_cast<float2*>(dst) = make_float2(g[0], g[1]);
                else dst[0] = g[0];
                continue;
            }
            if (a.act == ACT_RELU) {
#pragma unroll
                for (int e = 0; e < VW; e++) o[e] = fmaxf(o[e], 0.f);
            }
            if (a.res && valid) {
                const V r = *reinterpret_cast<const V*>(a.res + orow * a.ldres + n);
                if constexpr (VW == 4) { o[0] += r.x; o[1] += r.y; o[2] += r.z; o[3] += r.w; }
                else { o[0] += r.x; o[1] += r.y; }
            }
#pragma unroll
            for (int e = 0; e < VW; e++) o[e] *= a.scale;
            float* dst; int accum;
            if (n < a.split) { dst = a.y0 + orow * a.ldy0 + n; accum = a.acc0; }
            else { dst = a.y1 + orow * a.ldy1 + (n - a.split); accum = a.acc1; }
            if (accum) {
                if (!valid) continue;   // accumulated buffers keep their zeros in gap rows
                const V p = *reinterpret_cast<const V*>(dst);
                if constexpr (VW == 4) { o[0] += p.x; o[1] += p.y; o[2] += p.z; o[3] += p.w; }
                else { o[0] += p.x; o[1] += p.y; }
            } else if (!valid) {
#pragma unroll
                for (int e = 0; e < VW; e++) o[e] = 0.f;
            }
            if constexpr (VW == 4) *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
            else *reinterpret_cast<float2*>(dst) = make_float2(o[0], o[1]);
        }
    }
}

template <int BM, int TX, int VW, int NV>
void launch_cfg(const ConvArgs& a, cudaStream_t st) {
    constexpr int BN = TX * VW * NV;
    auto kern = conv_simt_kernel<BM, TX, VW, NV>;
    static PerDeviceOnce once;
    once.run([&] { cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024); });
    const size_t smem = ((size_t)2 * (BM + a.span) * AS_STRIDE + 2 * BK * BN) * sizeof(float);
    dim3 grid((a.rows_q + BM - 1) / BM, a.ldw / BN);
    launch_pdl(kern, dim3(grid), dim3(256), smem, st, a);
    g_launch_count++;
    check_launch("conv");
}

}  // namespace

int conv_simt_bn_for(int cout) {
    if (cout <= 32) return 32;
    if (cout % 128 == 0) return 128;
    if (cout % 192 == 0) return 192;   // 192 / 576 (encoder, duration predictor): 64 x 192 tiles, 4 x 12 per thread
                                       // (the 128 x 96 tiling with float2 columns ran the FP32 pipe at 47 %)
    if (cout % 96 == 0) return 96;
    if (cout % 64 == 0) return 64;
    return 128;   // padded
}

void launch_conv_simt(const ConvArgs& a, cudaStream_t st) {
    // the K loop walks whole 32-channel chunks: other widths would silently drop channels (voice.cu widens x_low's
    // 48-channel coupling halves to 96 for this reason too)
    if (a.cin % BK) throw_launch_error("conv_simt: input channels must be a multiple of 32");
    const int bn = conv_simt_bn_for(a.cout);
    switch (bn) {
        case 32: launch_cfg<256, 8, 4, 1>(a, st); break;
        case 64: launch_cfg<128, 16, 4, 1>(a, st); break;
        case 96: launch_cfg<128, 16, 2, 3>(a, st); break;
        case 192: launch_cfg<64, 16, 4, 3>(a, st); break;
        default: launch_cfg<128, 16, 4, 2>(a, st); break;
    }
}

}  // namespace sb200
