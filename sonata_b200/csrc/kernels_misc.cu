// Non-GEMM stages of the Piper/VITS path as sm_90a kernels: embedding, channel LayerNorm
// (warp-shuffle reductions), DDSConv depthwise stage, relative-position attention, the
// duration-predictor spline flow, the duration ceil/scan, the monotonic-alignment expansion
// (generate_path restated as a gather), conv_post+tanh and the Philox noise source.
// The reference executes all of these inside onnxruntime (piper/src/lib.rs:362-379); the
// arithmetic restated here follows oracle/vits_oracle.py function by function.
#include "common.cuh"
#include <algorithm>
#include <climits>
#include <math.h>

namespace sb200 {

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float gelu_exact(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

// ------------------------------------------------------------------ embedding
// oracle: text_encoder()  x = emb[ids] * sqrt(H)
__global__ void embed_kernel(const int* __restrict__ ids, const float* __restrict__ emb, float scale,
                             float* __restrict__ x, int rows, int H) {
    pdl_trigger(); pdl_wait();
    const int h4 = H / 4;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)rows * h4) return;
    const int r = (int)(i / h4), c = (int)(i % h4);
    const int id = ids[r];
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (id >= 0) {
        v = reinterpret_cast<const float4*>(emb + (size_t)id * H)[c];
        v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
    }
    reinterpret_cast<float4*>(x + (size_t)r * H)[c] = v;
}

// ------------------------------------------------------------------ channel LayerNorm (one warp per row)
// oracle: _layer_norm()  (eps = 1e-5, biased variance, two-pass)
template <int NV>
__global__ void __launch_bounds__(256) ln_kernel(const float* __restrict__ x, const float* __restrict__ res1,
                                                 const float* __restrict__ res2, const float* __restrict__ gamma,
                                                 const float* __restrict__ beta, float* __restrict__ out, int act,
                                                 RowMap map) {
    pdl_trigger(); pdl_wait();
    constexpr int C = NV * 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int r = blockIdx.x * 8 + warp;
    if (r >= map.rows) return;
    float* o = out + (size_t)r * C;
    if (!row_valid(map, r)) {
#pragma unroll
        for (int j = 0; j < NV; j++) o[lane + 32 * j] = 0.f;
        return;
    }
    float v[NV];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < NV; j++) {
        float t = x[(size_t)r * C + lane + 32 * j];
        if (res1) t += res1[(size_t)r * C + lane + 32 * j];
        v[j] = t;
        s += t;
    }
    const float mean = warp_sum(s) * (1.f / C);
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < NV; j++) { const float d = v[j] - mean; q += d * d; }
    const float rstd = rsqrtf(warp_sum(q) * (1.f / C) + 1e-5f);
#pragma unroll
    for (int j = 0; j < NV; j++) {
        const int c = lane + 32 * j;
        float y = (v[j] - mean) * rstd * gamma[c] + beta[c];
        if (act == 1) y = gelu_exact(y);
        if (res2) y += res2[(size_t)r * C + c];
        o[c] = y;
    }
}

// ------------------------------------------------------------------ DDSConv: depthwise conv + LN + GELU
// oracle: _dds()  y = gelu(LN(conv_sep(x)))
template <int NV>
__global__ void __launch_bounds__(256) dw_ln_gelu_kernel(const float* __restrict__ x, const float* __restrict__ wdw,
                                                         const float* __restrict__ bdw, int k, int dil,
                                                         const float* __restrict__ gamma,
                                                         const float* __restrict__ beta, float* __restrict__ out,
                                                         RowMap map) {
    pdl_trigger(); pdl_wait();
    constexpr int C = NV * 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int r = blockIdx.x * 8 + warp;
    if (r >= map.rows) return;
    float* o = out + (size_t)r * C;
    if (!row_valid(map, r)) {
#pragma unroll
        for (int j = 0; j < NV; j++) o[lane + 32 * j] = 0.f;
        return;
    }
    float v[NV];
#pragma unroll
    for (int j = 0; j < NV; j++) v[j] = bdw[lane + 32 * j];
    const int half = (k - 1) / 2;
    for (int t = 0; t < k; t++) {
        const int rr = r + (t - half) * dil;
        if (rr < 0 || rr >= map.rows) continue;   // gap rows hold zeros, so no per-segment test needed
#pragma unroll
        for (int j = 0; j < NV; j++) {
            const int c = lane + 32 * j;
            v[j] = fmaf(wdw[t * C + c], x[(size_t)rr * C + c], v[j]);
        }
    }
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < NV; j++) s += v[j];
    const float mean = warp_sum(s) * (1.f / C);
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < NV; j++) { const float d = v[j] - mean; q += d * d; }
    const float rstd = rsqrtf(warp_sum(q) * (1.f / C) + 1e-5f);
#pragma unroll
    for (int j = 0; j < NV; j++) {
        const int c = lane + 32 * j;
        o[c] = gelu_exact((v[j] - mean) * rstd * gamma[c] + beta[c]);
    }
}

// ------------------------------------------------------------------ relative-position attention
// oracle: _mha()   one CTA = (16 query rows, head, segment); 2*D threads.
//   scores[i][j] = (q_i/sqrt(D)).k_j + [|j-i|<=w] (q_i/sqrt(D)).E_k[j-i+w]
//   out_i = softmax(scores_i) . V + sum_{|d|<=w} p[i][i+d] E_v[d+w]
constexpr int ATT_QT = 16;

template <int D>
__global__ void __launch_bounds__(2 * D) attention_kernel(const float* __restrict__ qkv, int ldq,
                                                          const float* __restrict__ relk,
                                                          const float* __restrict__ relv, int window,
                                                          float* __restrict__ out, int ldo, int H,
                                                          const SegInfo* __restrict__ segs, int tpad) {
    pdl_trigger(); pdl_wait();
    const SegInfo sg = segs[blockIdx.z];
    const int T = sg.len;
    const int i0 = blockIdx.x * ATT_QT;
    if (i0 >= T) return;
    const int head = blockIdx.y;
    const int tid = threadIdx.x;
    constexpr int NT = 2 * D;
    const int nrel = 2 * window + 1;

    extern __shared__ __align__(16) float sm[];
    float* Qs = sm;                               // [QT][D]
    float* S = Qs + ATT_QT * D;                   // [QT][tpad]
    float* qE = S + ATT_QT * tpad;                // [QT][nrel]
    float* inv = qE + ATT_QT * nrel;              // [QT]
    float* Osum = inv + ATT_QT;                   // [4][QT][D] partial outputs of the four key-range quarters

    const float* qbase = qkv + (size_t)sg.off * ldq + head * D;
    const float* kbase = qbase + H;
    const float* vbase = qbase + 2 * H;
    const float qscale = rsqrtf((float)D);

    for (int idx = tid; idx < ATT_QT * D; idx += NT) {
        const int i = idx / D, c = idx % D;
        Qs[idx] = (i0 + i < T) ? qbase[(size_t)(i0 + i) * ldq + c] * qscale : 0.f;
    }
    __syncthreads();
    // relative-key logits
    for (int idx = tid; idx < ATT_QT * nrel; idx += NT) {
        const int i = idx / nrel, d = idx % nrel;
        float s = 0.f;
        for (int c = 0; c < D; c++) s = fmaf(Qs[i * D + c], relk[d * D + c], s);
        qE[idx] = s;
    }
    // scores: KPT keys per thread, all ATT_QT queries in registers.  Every Q value is a broadcast LDS that feeds one
    // FMA per key held by the thread: with one key per thread the phase issued one LDS.128 per four FMAs and was
    // bound by the load/store unit, not by the FP32 pipe.
    constexpr int KPT = 3;
    for (int j0 = tid * KPT; j0 < T; j0 += NT * KPT) {
        float acc[KPT][ATT_QT];
#pragma unroll
        for (int k = 0; k < KPT; k++)
#pragma unroll
            for (int i = 0; i < ATT_QT; i++) acc[k][i] = 0.f;
        const float4* kr[KPT];
#pragma unroll
        for (int k = 0; k < KPT; k++)
            kr[k] = reinterpret_cast<const float4*>(kbase + (size_t)min(j0 + k, T - 1) * ldq);
#pragma unroll 2
        for (int c4 = 0; c4 < D / 4; c4++) {
            float4 kv[KPT];
#pragma unroll
            for (int k = 0; k < KPT; k++) kv[k] = kr[k][c4];
#pragma unroll
            for (int i = 0; i < ATT_QT; i++) {
                const float4 qv = *reinterpret_cast<const float4*>(Qs + i * D + c4 * 4);
#pragma unroll
                for (int k = 0; k < KPT; k++) {
                    acc[k][i] = fmaf(qv.x, kv[k].x, acc[k][i]);
                    acc[k][i] = fmaf(qv.y, kv[k].y, acc[k][i]);
                    acc[k][i] = fmaf(qv.z, kv[k].z, acc[k][i]);
                    acc[k][i] = fmaf(qv.w, kv[k].w, acc[k][i]);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < KPT; k++)
            if (j0 + k < T) {
#pragma unroll
                for (int i = 0; i < ATT_QT; i++) S[i * tpad + j0 + k] = acc[k][i];
            }
    }
    __syncthreads();
    // add relative logits, softmax (one warp per query row, round-robin)
    const int warp = tid >> 5, lane = tid & 31;
    for (int i = warp; i < ATT_QT; i += NT / 32) {
        const int ia = i0 + i;
        if (ia >= T) { if (lane == 0) inv[i] = 0.f; continue; }
        float* Sr = S + i * tpad;
        if (lane < nrel) {
            const int j = ia + lane - window;
            if (j >= 0 && j < T) Sr[j] += qE[i * nrel + lane];
        }
        __syncwarp();
        float m = -INFINITY;
        for (int j = lane; j < T; j += 32) m = fmaxf(m, Sr[j]);
        m = warp_max(m);
        float s = 0.f;
        for (int j = lane; j < T; j += 32) { const float e = expf(Sr[j] - m); Sr[j] = e; s += e; }
        s = warp_sum(s);
        if (lane == 0) inv[i] = 1.f / s;
    }
    // zero the tail so the float4 loop below may over-read up to tpad
    for (int idx = tid; idx < ATT_QT * (tpad - T); idx += NT) {
        const int i = idx / (tpad - T), j = T + idx % (tpad - T);
        S[i * tpad + j] = 0.f;
    }
    __syncthreads();
    // P.V : thread = (quarter of the key range, channel PAIR): two channels per thread halve the broadcast LDS of the
    // probabilities per FMA (same load/store-unit argument as in the score phase)
    {
        const int part = tid / (D / 2), cp = tid % (D / 2);
        float acc[ATT_QT][2];
#pragma unroll
        for (int i = 0; i < ATT_QT; i++) { acc[i][0] = 0.f; acc[i][1] = 0.f; }
        const int nj4 = tpad / 4;
        for (int j4 = part; j4 < nj4; j4 += 4) {
            float2 vv[4];
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int j = j4 * 4 + e;
                vv[e] = j < T ? *reinterpret_cast<const float2*>(vbase + (size_t)j * ldq + cp * 2) : make_float2(0.f, 0.f);
            }
#pragma unroll
            for (int i = 0; i < ATT_QT; i++) {
                const float4 p = *reinterpret_cast<const float4*>(S + i * tpad + j4 * 4);
                acc[i][0] = fmaf(p.x, vv[0].x, acc[i][0]); acc[i][1] = fmaf(p.x, vv[0].y, acc[i][1]);
                acc[i][0] = fmaf(p.y, vv[1].x, acc[i][0]); acc[i][1] = fmaf(p.y, vv[1].y, acc[i][1]);
                acc[i][0] = fmaf(p.z, vv[2].x, acc[i][0]); acc[i][1] = fmaf(p.z, vv[2].y, acc[i][1]);
                acc[i][0] = fmaf(p.w, vv[3].x, acc[i][0]); acc[i][1] = fmaf(p.w, vv[3].y, acc[i][1]);
            }
        }
#pragma unroll
        for (int i = 0; i < ATT_QT; i++)
            *reinterpret_cast<float2*>(Osum + (part * ATT_QT + i) * D + cp * 2) = make_float2(acc[i][0], acc[i][1]);
    }
    __syncthreads();
    for (int idx = tid; idx < ATT_QT * D; idx += NT) {
        const int i = idx / D, c = idx % D;
        const int ia = i0 + i;
        if (ia >= T) continue;
        float o = (Osum[i * D + c] + Osum[(ATT_QT + i) * D + c]) + (Osum[(2 * ATT_QT + i) * D + c] + Osum[(3 * ATT_QT + i) * D + c]);
        for (int d = 0; d < nrel; d++) {
            const int j = ia + d - window;
            if (j >= 0 && j < T) o = fmaf(S[i * tpad + j], relv[d * D + c], o);
        }
        out[(size_t)(sg.off + ia) * ldo + head * D + c] = o * inv[i];
    }
}

// ------------------------------------------------------------------ relative-position softmax (tensor-core attention)
// Sits between the two grouped GEMMs of conv_tf.cu.  S[head][row][key] = (q.k)/sqrt(D) arrives from the first GEMM;
// one warp per (row, head) adds the relative-key logits on the |j - i| <= window band, takes the softmax over the
// utterance's keys IN PLACE, zero-fills the row up to the next multiple of 32 keys (the K extent of the second GEMM) and
// writes the relative-value term  orel[row][head*D + c] = sum_d p[i][i+d] E_v[d+w][c],  which the second GEMM adds as
// its residual.  The whole row lives in registers (NREG x 32 keys).  Lane l holds head channels l + 32k (k < ceil(D/32);
// 48-wide heads leave lanes 16-31 idle in the second).  The launcher picks NREG from the longest utterance of the job
// on this path; rows of longer utterances, which run on attention_kernel, are skipped.  oracle: _mha()
template <int D, int NREG>
__global__ void __launch_bounds__(256) attn_softmax_kernel(float* __restrict__ S, int Tp, const float* __restrict__ qkv,
                                                           int ldq, const float* __restrict__ relk,
                                                           const float* __restrict__ relv, int window,
                                                           float* __restrict__ orel, int ldo, int RX,
                                                           const SegInfo* __restrict__ segs,
                                                           const int* __restrict__ seg_of_gran, int gran) {
    pdl_trigger(); pdl_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q = blockIdx.x * 8 + warp;
    const int head = blockIdx.y;
    if (q >= RX) return;
    const SegInfo sg = segs[seg_of_gran[q / gran]];
    const int i = q - sg.off, T = sg.len;
    if (i < 0 || i >= T) return;                       // gap row
    if (T > 32 * NREG) return;                         // an utterance longer than the registers hold: on attention_kernel
    float* Sr = S + ((size_t)head * RX + q) * Tp;
    const int nrel = 2 * window + 1;
    constexpr int NV = (D + 31) / 32;
    auto has = [&](int k) { return D % 32 == 0 || lane + 32 * k < D; };
    const float qs = rsqrtf((float)D);
    float qv[NV];
#pragma unroll
    for (int k = 0; k < NV; k++) qv[k] = has(k) ? qkv[(size_t)q * ldq + head * D + lane + 32 * k] * qs : 0.f;
    float mine = 0.f;                                  // lane d keeps the logit of relative offset d - window
    for (int d = 0; d < nrel; d++) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < NV; k++) if (has(k)) s = fmaf(qv[k], relk[d * D + lane + 32 * k], s);
        s = warp_sum(s);
        if (lane == d) mine = s;
    }
    if (lane < nrel) {
        const int j = i + lane - window;
        if (j >= 0 && j < T) Sr[j] += mine;
    }
    __syncwarp();
    float s[NREG];
    float m = -INFINITY;
#pragma unroll
    for (int k = 0; k < NREG; k++) {
        const int j = lane + 32 * k;
        s[k] = j < T ? Sr[j] : -INFINITY;
        m = fmaxf(m, s[k]);
    }
    m = warp_max(m);
    float l = 0.f;
#pragma unroll
    for (int k = 0; k < NREG; k++) {
        const float e = (lane + 32 * k) < T ? expf(s[k] - m) : 0.f;
        s[k] = e;
        l += e;
    }
    l = warp_sum(l);
    const float inv = 1.f / l;
    const int Tz = (T + 31) & ~31;
#pragma unroll
    for (int k = 0; k < NREG; k++) {
        const int j = lane + 32 * k;
        if (j < Tz) Sr[j] = s[k] * inv;
    }
    __syncwarp();
    float pb = 0.f;
    if (lane < nrel) {
        const int j = i + lane - window;
        if (j >= 0 && j < T) pb = Sr[j];
    }
    float acc[NV];
#pragma unroll
    for (int k = 0; k < NV; k++) acc[k] = 0.f;
    for (int d = 0; d < nrel; d++) {
        const float p = __shfl_sync(0xffffffffu, pb, d);
#pragma unroll
        for (int k = 0; k < NV; k++) if (has(k)) acc[k] = fmaf(p, relv[d * D + lane + 32 * k], acc[k]);
    }
#pragma unroll
    for (int k = 0; k < NV; k++) if (has(k)) orel[(size_t)q * ldo + head * D + lane + 32 * k] = acc[k];
}

// ------------------------------------------------------------------ duration-predictor flow pieces
// oracle: _conv_flow_reverse()  h = pre(z0) + g
__global__ void flow_pre_kernel(const float* __restrict__ z, int zcol, const float* __restrict__ w,
                                const float* __restrict__ b, const float* __restrict__ g, float* __restrict__ h,
                                int C, RowMap map) {
    pdl_trigger(); pdl_wait();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)map.rows * C) return;
    const int r = (int)(i / C), c = (int)(i % C);
    h[i] = row_valid(map, r) ? fmaf(w[c], z[2 * r + zcol], b[c]) + g[i] : 0.f;
}

__device__ __forceinline__ float softplus_f(float x) { return x > 20.f ? x : log1pf(expf(x)); }

// oracle: _rqs_inverse()  (tails = linear, bound 5, min bin w/h 1e-3, min derivative 1e-3)
template <int NB>
__global__ void spline_kernel(const float* __restrict__ h29, int ldh, float* __restrict__ z, int tcol,
                              float inv_sqrt_filter, RowMap map) {
    pdl_trigger(); pdl_wait();
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= map.rows) return;
    if (!row_valid(map, r)) { z[2 * r + tcol] = 0.f; return; }
    const float x = z[2 * r + tcol];
    const float B = 5.0f;
    if (!(x >= -B && x <= B)) return;   // identity outside the tails
    const float* h = h29 + (size_t)r * ldh;
    float cw[NB + 1], ch[NB + 1], dv[NB + 1];
    // widths
    {
        float u[NB], m = -INFINITY, s = 0.f;
#pragma unroll
        for (int k = 0; k < NB; k++) { u[k] = h[k] * inv_sqrt_filter; m = fmaxf(m, u[k]); }
#pragma unroll
        for (int k = 0; k < NB; k++) { u[k] = expf(u[k] - m); s += u[k]; }
        float c = 0.f;
        cw[0] = -B;
#pragma unroll
        for (int k = 0; k < NB; k++) {
            const float wk = 1e-3f + (1.f - 1e-3f * NB) * (u[k] / s);
            c += wk;
            cw[k + 1] = 2.f * B * c + (-B);
        }
        cw[NB] = B;
    }
    {
        float u[NB], m = -INFINITY, s = 0.f;
#pragma unroll
        for (int k = 0; k < NB; k++) { u[k] = h[NB + k] * inv_sqrt_filter; m = fmaxf(m, u[k]); }
#pragma unroll
        for (int k = 0; k < NB; k++) { u[k] = expf(u[k] - m); s += u[k]; }
        float c = 0.f;
        ch[0] = -B;
#pragma unroll
        for (int k = 0; k < NB; k++) {
            const float hk = 1e-3f + (1.f - 1e-3f * NB) * (u[k] / s);
            c += hk;
            ch[k + 1] = 2.f * B * c + (-B);
        }
        ch[NB] = B;
    }
    {
        const float cst = logf(expf(1.f - 1e-3f) - 1.f);
        dv[0] = 1e-3f + softplus_f(cst);
        dv[NB] = dv[0];
#pragma unroll
        for (int k = 1; k < NB; k++) dv[k] = 1e-3f + softplus_f(h[2 * NB + k - 1]);
    }
    int bin = -1;
#pragma unroll
    for (int k = 0; k <= NB; k++) {
        const float loc = (k == NB) ? ch[k] + 1e-6f : ch[k];
        bin += (x >= loc) ? 1 : 0;
    }
    bin = min(max(bin, 0), NB - 1);
    float in_cw = 0, in_w = 0, in_ch = 0, in_h = 0, in_d = 0, in_d1 = 0;
#pragma unroll
    for (int k = 0; k < NB; k++)
        if (k == bin) {
            in_cw = cw[k]; in_w = cw[k + 1] - cw[k];
            in_ch = ch[k]; in_h = ch[k + 1] - ch[k];
            in_d = dv[k]; in_d1 = dv[k + 1];
        }
    const float delta = in_h / in_w;
    const float t = x - in_ch;
    const float e = in_d + in_d1 - 2.f * delta;
    const float a = t * e + in_h * (delta - in_d);
    const float b = in_h * in_d - t * e;
    const float c = -delta * t;
    // At the top of a bin disc = h^2 d_{k+1}^2 exactly, but in fp32 it is the difference of two O(4 h^2 delta^2) terms and
    // can round below zero, where sqrtf gives NaN (the fp32 graph does).  Clamped, the root is the fp64 answer to within
    // the condition of the inverse (DESIGN.md section 4).
    const float disc = fmaxf(b * b - 4.f * a * c, 0.f);
    const float root = (2.f * c) / (-b - sqrtf(disc));
    // the exact inverse of an input in [-B, B] lies in [-B, B]; in fp32 the root of an end bin can overshoot B by up to
    // ~1.4e-4 (hundreds of ulp, saturated and sigma-10 logits), which the next flow would take as its identity tail
    z[2 * r + tcol] = fminf(fmaxf(root * in_w + in_cw, -B), B);
}

// z[r][0..1] = eps[r][0..1] * noise_w of r's segment   (oracle: sdp_reverse  z = eps_w * noise_w).  A segment whose
// noise_w is 0 gets exact zeros, as a call without noise does (eps * 0 would give -0 for a negative draw).
__global__ void scale_copy2_kernel(const float* __restrict__ eps, const float* __restrict__ s,
                                   const int* __restrict__ seg_of_gran, float* __restrict__ z, RowMap map) {
    pdl_trigger(); pdl_wait();
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= map.rows) return;
    const float sr = (eps != nullptr && row_valid(map, r)) ? s[seg_of_gran[r / map.gran]] : 0.f;
    const bool v = sr != 0.f;
    z[2 * r] = v ? eps[2 * r] * sr : 0.f;
    z[2 * r + 1] = v ? eps[2 * r + 1] * sr : 0.f;
}

// ------------------------------------------------------------------ durations: ceil + inclusive scan
// oracle: sdp_reverse() tail (ElementwiseAffine^-1) + durations()
// The scan runs in 64 bits and cum / y_len saturate at INT_MAX: a duration past 2^31 - 1 frames (or a NaN / inf one)
// must reach the host as an overlong frame count, which it rejects, not wrap into a plausible one.
// Optional per-id controls, at the id level like logw (null: none):
//   dur_scale  : the predicted count is ceil((exp(logw) * length_scale) * s); the product is rounded in that order, so
//                s = 1 gives the bits of a call without scales
//   dur_frames : a value >= 0 replaces the count (no ceil involved); -1 keeps the predicted one
//   fit        : the target fit's factor u (fit.cu), multiplied in after s as one more f32 multiply
// logw is written for every id either way.
__device__ __forceinline__ int sat_int(long long v) { return (int)min(v, (long long)INT_MAX); }

__global__ void __launch_bounds__(256) durations_kernel(const float* __restrict__ z, float m0, float logs0,
                                                        const float* __restrict__ length_scales,
                                                        const SegInfo* __restrict__ segs,
                                                        const float* __restrict__ dur_scale,
                                                        const int* __restrict__ dur_frames,
                                                        const float* __restrict__ fit,
                                                        float* __restrict__ logw, int* __restrict__ cum,
                                                        int* __restrict__ y_len) {
    pdl_trigger(); pdl_wait();
    const SegInfo sg = segs[blockIdx.x];
    const float length_scale = length_scales[blockIdx.x];
    __shared__ long long warp_tot[8];
    __shared__ long long carry_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry_s = 0;
    __syncthreads();
    const float einv = expf(-logs0);
    for (int base = 0; base < sg.len; base += 256) {
        const int i = base + tid;
        long long w = 0;
        if (i < sg.len) {
            const int row = sg.off + i;
            const float lw = dur_logw(z, row, m0, einv);
            logw[row] = lw;
            float wf = dur_weight(lw, length_scale, dur_scale, row);
            if (fit) wf = wf * fit[row];
            w = dur_count(wf);
            if (dur_frames) {
                const int f = dur_frames[row];
                if (f >= 0) w = f;
            }
        }
        long long s = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long t = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += t;
        }
        if (lane == 31) warp_tot[warp] = s;
        __syncthreads();
        long long pre = carry_s;
        for (int k = 0; k < warp; k++) pre += warp_tot[k];
        if (i < sg.len) cum[sg.off + i] = sat_int(pre + s);
        __syncthreads();
        if (tid == 255) carry_s = pre + s;
        __syncthreads();
    }
    if (tid == 0) y_len[blockIdx.x] = sat_int(max(carry_s, 1LL));
}

// ------------------------------------------------------------------ alignment expansion (one warp per frame)
// oracle: expand()   frame j takes token i iff cum[i-1] <= j < cum[i]
__global__ void __launch_bounds__(256) expand_kernel(const float* __restrict__ stats, int ldst, int I,
                                                     const int* __restrict__ cum, const float* __restrict__ eps,
                                                     const float* __restrict__ noise_scales, float* __restrict__ zp,
                                                     const FrameSeg* __restrict__ fsegs,
                                                     const int* __restrict__ ftile_seg, RowMap ymap) {
    pdl_trigger(); pdl_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int r = blockIdx.x * 8 + warp;
    if (r >= ymap.rows) return;
    float* o = zp + (size_t)r * I;
    if (!row_valid(ymap, r)) {
        for (int c = lane; c < I; c += 32) o[c] = 0.f;
        return;
    }
    const int seg = ftile_seg[r / ymap.gran];
    const FrameSeg fs = fsegs[seg];
    // a segment whose noise_scale is 0 takes the no-noise branch (no `eps * 0` term, which could be -0)
    const float noise_scale = eps ? noise_scales[seg] : 0.f;
    const int j = r - fs.off;
    const int* cm = cum + fs.xoff;
    int lo = 0, hi = fs.xlen;          // first i with cm[i] > j
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cm[mid] > j) hi = mid; else lo = mid + 1;
    }
    if (lo >= fs.xlen) {               // only when sum(w_ceil) == 0 and y_len was clamped to 1
        for (int c = lane; c < I; c += 32) o[c] = (eps && noise_scale != 0.f) ? eps[(size_t)r * I + c] * noise_scale : 0.f;
        return;
    }
    const float* st = stats + (size_t)(fs.xoff + lo) * ldst;
    for (int c = lane; c < I; c += 32) {
        float v = st[c];
        if (eps && noise_scale != 0.f) v += eps[(size_t)r * I + c] * expf(st[I + c]) * noise_scale;
        o[c] = v;
    }
}

// ------------------------------------------------------------------ conv_post + tanh (C -> 1, k = 7)
// oracle: decoder() tail.  HBM-bound in principle (read 4*C bytes, write 4 bytes per sample); the first version (one
// sample per thread, 7*C scalar shared-memory loads each) was bound by shared-memory wavefronts at 0.70 ms on C2 against
// a 0.3 ms HBM floor.  Here a CTA stages 512 rows CHANNEL-MAJOR (xs[c][row], leaky-relu applied) and every thread
// produces FOUR consecutive samples: per channel three 128-bit loads bring the 12 staged rows its 4 x 7 taps touch, so a
// staged value is read ~once instead of seven times.  Layout: 16-byte unit u (4 rows) of channel c lives at unit
// (u ^ ((c >> 2) & 7)) -- with that XOR both the transposing stores of the load phase (8 channel groups x 4 rows per
// warp) and the unit-strided 128-bit loads of the compute phase are bank-conflict free.  256 threads: all of them load
// (four independent 128-bit loads in flight each), pairs of lanes split the channels of one 4-sample group.
template <int C>
__global__ void __launch_bounds__(256) conv_post_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                        float* __restrict__ wav, const FrameSeg* __restrict__ fsegs,
                                                        const int* __restrict__ ftile_seg, int U, RowMap map, int vec_ok) {
    pdl_trigger(); pdl_wait();
    constexpr int NT = 256, ROWS = 512, LEAD = 4, SR = ROWS + 8;   // staged rows r0-4 .. r0+515
    constexpr int S = 544;                               // floats per channel row: 136 units, a multiple of 8 units >= SR/4 + 7
    extern __shared__ __align__(16) float sm[];
    float* xs = sm;                       // [C][S]
    float* ws = xs + C * S;               // [C][8]: taps 0..6 of channel c, then 0
    const int tid = threadIdx.x;
    const int r0 = blockIdx.x * ROWS;
    for (int i = tid; i < C * 8; i += NT) {
        const int c = i >> 3, t = i & 7;
        ws[i] = t < 7 ? w[t * C + c] : 0.f;
    }
    constexpr int NF4 = SR * (C / 4);
    for (int base = tid; base < NF4; base += NT * 4) {    // four independent 128-bit loads in flight per thread
        float4 v[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int i = base + k * NT;
            const int rr = i / (C / 4), c4 = i % (C / 4);
            const int gr = r0 - LEAD + rr;
            v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (i < NF4 && gr >= 0 && gr < map.rows) v[k] = reinterpret_cast<const float4*>(x + (size_t)gr * C)[c4];
        }
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int i = base + k * NT;
            if (i >= NF4) continue;
            const int rr = i / (C / 4), c4 = i % (C / 4);
            const int pos = (((rr >> 2) ^ (c4 & 7)) << 2) | (rr & 3);
            float* d = xs + (size_t)(c4 * 4) * S + pos;
            d[0] = v[k].x > 0.f ? v[k].x : 0.01f * v[k].x;
            d[S] = v[k].y > 0.f ? v[k].y : 0.01f * v[k].y;
            d[2 * S] = v[k].z > 0.f ? v[k].z : 0.01f * v[k].z;
            d[3 * S] = v[k].w > 0.f ? v[k].w : 0.01f * v[k].w;
        }
    }
    __syncthreads();
    // thread pair (2g, 2g+1) owns the four rows r0 + 4g ..; each lane of the pair sums half of the channels
    const int g = tid >> 1, half = tid & 1;
    const int r = r0 + 4 * g;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const int u0 = g + 1;                                     // staged unit of the group's own four rows
#pragma unroll 4
    for (int k = 0; k < C / 2; k++) {
        const int c = half * (C / 2) + k;
        const int sw = (c >> 2) & 7;
        const float* xc = xs + (size_t)c * S;
        const float4 a = *reinterpret_cast<const float4*>(xc + (((u0 - 1) ^ sw) << 2));
        const float4 b = *reinterpret_cast<const float4*>(xc + ((u0 ^ sw) << 2));
        const float4 d = *reinterpret_cast<const float4*>(xc + (((u0 + 1) ^ sw) << 2));
        const float4 w0 = *reinterpret_cast<const float4*>(ws + c * 8);
        const float4 w1 = *reinterpret_cast<const float4*>(ws + c * 8 + 4);
        const float v[12] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, d.x, d.y, d.z, d.w};
        const float wt[7] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z};
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int t = 0; t < 7; t++) acc[j] = fmaf(v[j + 1 + t], wt[t], acc[j]);
    }
#pragma unroll
    for (int j = 0; j < 4; j++) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], 1);
    if (half != 0 || r >= map.rows || !row_valid(map, r)) return;     // a group of four rows never straddles a segment end
    const FrameSeg fs = fsegs[ftile_seg[r / map.gran]];
    float* dst = wav + fs.out_off + (long long)(r - (long long)fs.off * U);
    const float o0 = tanhf(acc[0]), o1 = tanhf(acc[1]), o2 = tanhf(acc[2]), o3 = tanhf(acc[3]);
    if (vec_ok) *reinterpret_cast<float4*>(dst) = make_float4(o0, o1, o2, o3);
    else { dst[0] = o0; dst[1] = o1; dst[2] = o2; dst[3] = o3; }
}

// ------------------------------------------------------------------ f32 -> i16 with per-utterance peak normalisation
// crates/audio/ops/src/samples.rs:51-75 (`to_i16_vec`): scale = 32767 / max(|x|_max, f32::EPSILON);
// y = trunc(clamp(x * scale, -32768, 32767)).  Bit-exact with the host version (same fp32 operations in the same
// order); halves the device->host bytes of a synthesis result.  `PcmPost` folds in what the reference does to a
// chunk before that conversion: trimming the overlap frames of a streamed chunk (piper/src/lib.rs:811-826),
// crossfade(42) (samples.rs:144-157; the sine table is computed by the host so both sides use the same floats) and
// the linear volume gain of AudioOutputConfig (synth/src/lib.rs:84-86).  Every segment (blockIdx.y) has its own
// PcmPost, so one launch converts the chunks of many streams, each normalised to its own peak.  A segment is read
// through pcm_seg / pcm_value (common.cuh).

__global__ void i16_absmax_kernel(const float* __restrict__ wav, const FrameSeg* __restrict__ fsegs,
                                  const PcmPost* __restrict__ posts, int hop, unsigned* __restrict__ maxbits) {
    pdl_trigger(); pdl_wait();
    const PcmSeg s = pcm_seg(wav, fsegs[blockIdx.y], posts + blockIdx.y, hop);
    float m = 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < s.n; i += (long long)gridDim.x * blockDim.x)
        m = fmaxf(m, fabsf(pcm_value(s, i)));
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(maxbits + blockIdx.y, __float_as_uint(m));   // non-negative floats
                                                                                                  // order like their bits
}

// FMT: PCM_I16 stores the 16-bit sample; PCM_MULAW / PCM_ALAW store the G.711 byte of that same sample (common.cuh),
// so an encoded result is the i16 result encoded, at half its bytes.
template <int FMT> struct PcmOut { using T = uint8_t; };
template <> struct PcmOut<PCM_I16> { using T = short; };
template <int FMT>
__global__ void i16_convert_kernel(const float* __restrict__ wav, const FrameSeg* __restrict__ fsegs,
                                   const PcmPost* __restrict__ posts, int hop, const unsigned* __restrict__ maxbits,
                                   typename PcmOut<FMT>::T* __restrict__ out) {
    pdl_trigger(); pdl_wait();
    const FrameSeg fs = fsegs[blockIdx.y];
    const PcmSeg s = pcm_seg(wav, fs, posts + blockIdx.y, hop);
    typename PcmOut<FMT>::T* y = out + fs.out_off;
    const float amax = fmaxf(__uint_as_float(maxbits[blockIdx.y]), 1.1920928955078125e-07f);
    const float scale = posts[blockIdx.y].fixed_scale ? 32767.0f : __fdiv_rn(32767.0f, amax);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < s.n; i += (long long)gridDim.x * blockDim.x) {
        const float v = fminf(fmaxf(__fmul_rn(pcm_value(s, i), scale), -32768.0f), 32767.0f);
        const short q = (short)(int)v;             // truncating cast
        if constexpr (FMT == PCM_I16) y[i] = q;
        else if constexpr (FMT == PCM_MULAW) y[i] = g711_ulaw(q);
        else y[i] = g711_alaw(q);
    }
}

// ------------------------------------------------------------------ polyphase resampling (scipy's resample_poly)
// Output j of a segment of n inputs is  y[j] = sum_i x[i] * h[j*down + H - i*up]  over 0 <= i < n with the tap index in
// [0, 2H], evaluated as ONE fmaf chain in ascending i starting from 0.  With t = j*down + H, phase p = t % up and
// i_max = t / up, input i_max - k meets tap h[p + k*up] = taps[p][k].  The chain depends on j, n and the ratio only, so
// a sample comes out with the same bits whatever buffer, batch or block split it is computed in.  A block computes runs
// of RS_OUTS consecutive outputs: it stages the input span of the run in shared memory, read through pcm_value (the
// segment's trim, crossfade and gain), then each thread evaluates its outputs from there, the taps of one output being
// contiguous in the phase-major table.
// A stream's segment continues an input sequence: its samples are inputs c .. c + n of the stream, the h inputs before
// them come from `hist`, and it writes outputs j0 .. j0 + n_out.  Block 0 of the segment also stores the stream's last
// h_out inputs into `hist_out` (a different buffer, so no block reads what another writes).  Outputs are only emitted
// once every input they read has arrived (or the stream has ended), so the chain of output j is the same as over the
// whole stream in one buffer.
__device__ __forceinline__ float rs_input(const ResampleSeg& r, const PcmSeg& s, long long g) {
    return g < r.c ? r.hist[g - (r.c - r.h)] : pcm_value(s, g - r.c);
}
__global__ void resample_kernel(const float* __restrict__ wav, const FrameSeg* __restrict__ fsegs,
                                const PcmPost* __restrict__ posts, int hop, const ResampleSeg* __restrict__ segs,
                                float* __restrict__ out) {
    extern __shared__ float xs[];
    pdl_trigger(); pdl_wait();
    const ResampleSeg r = segs[blockIdx.y];
    const PcmSeg s = pcm_seg(wav, fsegs[blockIdx.y], posts + blockIdx.y, hop);
    float* y = out + r.out_off;
    if (r.up == 0) {
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < s.n; i += (long long)gridDim.x * blockDim.x)
            y[i] = pcm_value(s, i);
        return;
    }
    const long long N = r.c + s.n;            // inputs of the stream so far
    if (blockIdx.x == 0 && r.hist_out)
        for (int q = threadIdx.x; q < r.h_out; q += blockDim.x) r.hist_out[q] = rs_input(r, s, N - r.h_out + q);
    const int up = r.up, down = r.down, H2 = 2 * r.H, K = r.K;
    for (long long a = (long long)blockIdx.x * RS_OUTS; a < r.n_out; a += (long long)gridDim.x * RS_OUTS) {
        const long long j_a = r.j0 + a, j_b = r.j0 + min(a + RS_OUTS, r.n_out);
        const long long i_lo = max(0ll, (j_a * down + r.H) / up - (K - 1));
        const long long i_hi = min(((j_b - 1) * down + r.H) / up, N - 1);
        for (int q = threadIdx.x; q <= (int)(i_hi - i_lo); q += blockDim.x) xs[q] = rs_input(r, s, i_lo + q);
        __syncthreads();
        for (long long j = j_a + threadIdx.x; j < j_b; j += blockDim.x) {
            const long long t = j * down + r.H, im = t / up;
            const int p = (int)(t - im * up);
            const int kmax = (int)min((long long)((H2 - p) / up), im);      // i >= 0
            const int kmin = (int)max(0ll, im - (N - 1));                     // i < N
            const float* h = r.taps + p * K;
            const float* x = xs + (int)(im - i_lo);
            float acc = 0.f;
            for (int k = kmax; k >= kmin; k--) acc = fmaf(x[-k], __ldg(h + k), acc);
            y[j - r.j0] = acc;
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------ integrated loudness (ITU-R BS.1770-4, one channel)
// One block per segment.  The K-weighting cascade is the only sequential part: (1) every chunk of S samples is filtered
// from zero state by one thread, which keeps the chunk's end state and peak; (2) thread 0 chains the states,
// s_{c+1} = A^S s_c + e_c, giving every chunk its true initial state; (3) every full chunk is filtered again from it and
// its sum of y^2, in sample order, is q_c; (4) block j (samples [jS, jS + 4S)) has z_j = (q_j + .. + q_{j+3}) / 4S and
// the absolute and relative gates run over the z_j in a fixed tree order; (5) the gain g = min(10^((T - L)/20), 1/peak)
// scales the segment in place.  Filter, energies and gates are double.  Chunking, chains and reduction orders depend on
// the segment's samples and S only, so L, g and the output are the same bits in any batch.
constexpr int LD_THREADS = 256;

// Samples [i0, i1) of x through the cascade from state s (updated), returning the sum of y^2 in sample order.
__device__ __forceinline__ double kweight_run(const float* __restrict__ x, long long i0, long long i1, const double* k,
                                              double* s, float* peak) {
    double s1 = s[0], s2 = s[1], t1 = s[2], t2 = s[3], e = 0.0;
    float m = 0.f;
    auto step = [&](float xf) {
        m = fmaxf(m, fabsf(xf));
        const double v = (double)xf;
        const double y1 = fma(k[0], v, s1);
        s1 = fma(k[1], v, fma(-k[3], y1, s2));
        s2 = fma(k[2], v, -k[4] * y1);
        const double y = fma(k[5], y1, t1);
        t1 = fma(k[6], y1, fma(-k[8], y, t2));
        t2 = fma(k[7], y1, -k[9] * y);
        e = fma(y, y, e);
    };
    // the lanes of a warp read chunks S samples apart: 16 loads issued together wait for memory once, not 16 times
    constexpr int V = 16;
    long long i = i0;
    for (; i + V <= i1; i += V) {
        float xv[V];
#pragma unroll
        for (int u = 0; u < V; u++) xv[u] = x[i + u];
#pragma unroll
        for (int u = 0; u < V; u++) step(xv[u]);
    }
    for (; i < i1; i++) step(x[i]);
    s[0] = s1; s[1] = s2; s[2] = t1; s[3] = t2;
    *peak = m;
    return e;
}

// Fixed-order tree sum over the block (every thread gets the total).
__device__ __forceinline__ double ld_block_sum(double v, double* red) {
    __syncthreads();
    red[threadIdx.x] = v;
    for (int w = LD_THREADS / 2; w > 0; w >>= 1) {
        __syncthreads();
        if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    }
    __syncthreads();
    return red[0];
}

__device__ __forceinline__ double ld_block_loudness(double z) { return -0.691 + 10.0 * log10(z); }

// One step of the state chain: s <- A^S s + e, each row summed in a fixed order.
__device__ __forceinline__ void ld_chain_step(const double* AS, const double* e, double* s) {
    double t[4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
        double a = e[r];
#pragma unroll
        for (int q = 0; q < 4; q++) a = fma(AS[4 * r + q], s[q], a);
        t[r] = a;
    }
#pragma unroll
    for (int r = 0; r < 4; r++) s[r] = t[r];
}

// z_j of block j, whose four steps' energies are q[0], q[stride], q[2 stride], q[3 stride]; blk = 4S.
__device__ __forceinline__ double ld_block_z(const double* q, long long stride, double blk) {
    return (((q[0] + q[stride]) + q[2 * stride]) + q[3 * stride]) / blk;
}

// The gated integrated loudness of the nb blocks whose step energies are q[c * stride] (block j: steps j .. j + 3):
// the absolute gate at -70 LUFS, the relative gate 10 LU under the mean of the blocks that pass it, each sum taken per
// thread in stride order and then over the block in a fixed tree order.  -inf when no block passes.  Every thread of
// the block calls it and gets the result.
__device__ __forceinline__ double ld_gates(const double* q, long long stride, long long nb, double blk, double* red) {
    double sum = 0.0, cnt = 0.0;
    for (long long j = threadIdx.x; j < nb; j += LD_THREADS) {
        const double z = ld_block_z(q + stride * j, stride, blk);
        if (ld_block_loudness(z) > -70.0) { sum += z; cnt += 1.0; }
    }
    sum = ld_block_sum(sum, red);
    cnt = ld_block_sum(cnt, red);
    double L = -INFINITY;
    if (cnt > 0.0) {
        const double rel = ld_block_loudness(sum / cnt) - 10.0;
        double sum2 = 0.0, cnt2 = 0.0;
        for (long long j = threadIdx.x; j < nb; j += LD_THREADS) {
            const double z = ld_block_z(q + stride * j, stride, blk), l = ld_block_loudness(z);
            if (l > -70.0 && l > rel) { sum2 += z; cnt2 += 1.0; }
        }
        sum2 = ld_block_sum(sum2, red);
        cnt2 = ld_block_sum(cnt2, red);
        if (cnt2 > 0.0) L = ld_block_loudness(sum2 / cnt2);
    }
    return L;
}

__global__ void __launch_bounds__(LD_THREADS) loudness_kernel(float* __restrict__ wav, const LoudSeg* __restrict__ segs,
                                                              double* __restrict__ scratch, double* __restrict__ lufs,
                                                              float* __restrict__ gain) {
    __shared__ double red[LD_THREADS];
    pdl_trigger(); pdl_wait();
    const LoudSeg& G = segs[blockIdx.x];
    const long long n = G.n, S = G.S;
    float* x = wav + G.off;
    double* sc = scratch + (long long)LD_SCRATCH * G.c0;
    double k[10];
#pragma unroll
    for (int i = 0; i < 10; i++) k[i] = G.k[i];
    const long long nch = (n + S - 1) / S, nfull = n / S;
    // (1) zero-state end states and peaks
    float peak = 0.f;
    for (long long c = threadIdx.x; c < nch; c += LD_THREADS) {
        double s[4] = {0.0, 0.0, 0.0, 0.0};
        float m;
        kweight_run(x, c * S, min(n, (c + 1) * S), k, s, &m);
        double* d = sc + LD_SCRATCH * c;
        d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; d[3] = s[3];
        peak = fmaxf(peak, m);
    }
    __syncthreads();
    // (2) initial states, in place of the end states
    if (threadIdx.x == 0) {
        double s[4] = {0.0, 0.0, 0.0, 0.0};
        for (long long c = 0; c + 1 < nch; c++) {
            double* d = sc + LD_SCRATCH * c;
            const double e[4] = {d[0], d[1], d[2], d[3]};
            d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; d[3] = s[3];
            ld_chain_step(G.AS, e, s);
        }
        if (nch > 0) {
            double* d = sc + LD_SCRATCH * (nch - 1);
            d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; d[3] = s[3];
        }
    }
    __syncthreads();
    // (3) energy of every full chunk from its true initial state
    for (long long c = threadIdx.x; c < nfull; c += LD_THREADS) {
        double* d = sc + LD_SCRATCH * c;
        double s[4] = {d[0], d[1], d[2], d[3]};
        float m;
        d[4] = kweight_run(x, c * S, (c + 1) * S, k, s, &m);
    }
    // peak of the segment (fmaxf of |x|, as i16_absmax_kernel)
    peak = warp_max(peak);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = (double)peak;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = 0.f;
        for (int w = 0; w < LD_THREADS / 32; w++) m = fmaxf(m, (float)red[w]);
        red[LD_THREADS - 1] = (double)m;
    }
    __syncthreads();
    peak = (float)red[LD_THREADS - 1];
    // (4) gates over the nb blocks
    const long long nb = n >= 4 * S ? (n - 4 * S) / S + 1 : 0;
    const double L = ld_gates(sc + 4, LD_SCRATCH, nb, 4.0 * (double)S, red);
    // (5) the gain, never taking the peak above full scale
    float g = 1.f;
    if (!isnan(G.target) && L > -INFINITY && peak > 0.f) {
        g = (float)fmin(exp10(((double)G.target - L) / 20.0), 1.0 / (double)peak);
        while (__fmul_rn(peak, g) > 1.f) g = nextafterf(g, 0.f);
    }
    if (threadIdx.x == 0) { lufs[blockIdx.x] = L; gain[blockIdx.x] = g; }
    if (g != 1.f)
        for (long long i = threadIdx.x; i < n; i += LD_THREADS) x[i] = __fmul_rn(x[i], g);
}

// ------------------------------------------------------------------ live loudness of a stream (one block per chunk)
// The chunk continues its meter's signal: the carried partial step (p samples) and the chunk's n samples are staged
// as one window, every step the window completes is filtered from zero state by one thread, thread 0 chains the states
// from the carried one, and each step's q is summed again from its true state, exactly as loudness_kernel does it.
// Then the readings at each step boundary the window reaches, the gains they give, and the ramp, scale and clamp of the
// chunk in place; the carry of the next chunk goes to the other buffer.
__global__ void __launch_bounds__(LD_THREADS) loudness_stream_kernel(const LoudStreamSeg* __restrict__ segs) {
    __shared__ double red[LD_THREADS];
    pdl_trigger(); pdl_wait();
    const LoudStreamSeg& G = segs[blockIdx.x];
    const long long n = G.n, S = G.S, p = G.p, w = p + n, nc = w / S, m0 = G.m0;
    float* win = G.win;
    double k[10];
#pragma unroll
    for (int i = 0; i < 10; i++) k[i] = G.k[i];
    // (1) the window: the carried samples, then the chunk's
    const float* tail = reinterpret_cast<const float*>(G.cin + 4);
    for (long long i = threadIdx.x; i < w; i += LD_THREADS) win[i] = i < p ? tail[i] : G.y[i - p];
    if (threadIdx.x == 0) *G.clipped = 0ull;
    __syncthreads();
    // (2) zero-state end states of the completed steps
    for (long long c = threadIdx.x; c < nc; c += LD_THREADS) {
        double s[4] = {0.0, 0.0, 0.0, 0.0};
        float m;
        kweight_run(win, c * S, (c + 1) * S, k, s, &m);
        double* d = G.e + 8 * c;
        d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; d[3] = s[3];
    }
    __syncthreads();
    // (3) true initial states from the carried one; the state at the new last boundary is carried
    if (threadIdx.x == 0) {
        double s[4] = {G.cin[0], G.cin[1], G.cin[2], G.cin[3]};
        for (long long c = 0; c < nc; c++) {
            double* d = G.e + 8 * c;
            d[4] = s[0]; d[5] = s[1]; d[6] = s[2]; d[7] = s[3];
            ld_chain_step(G.AS, d, s);
        }
        G.cout[0] = s[0]; G.cout[1] = s[1]; G.cout[2] = s[2]; G.cout[3] = s[3];
    }
    __syncthreads();
    // (4) q of every completed step, and the samples past the last boundary into the carry
    for (long long c = threadIdx.x; c < nc; c += LD_THREADS) {
        const double* d = G.e + 8 * c;
        double s[4] = {d[4], d[5], d[6], d[7]};
        float m;
        G.q[m0 + c] = kweight_run(win, c * S, (c + 1) * S, k, s, &m);
    }
    float* tail_out = reinterpret_cast<float*>(G.cout + 4);
    for (long long i = nc * S + threadIdx.x; i < w; i += LD_THREADS) tail_out[i - nc * S] = win[i];
    __syncthreads();
    // (5) the reading and gain at every boundary m0 + 1 .. m0 + nc: the batch gates over blocks 0 .. m - 4 from m = 4
    // on, the provisional mean before it; a boundary without a reading keeps the gain
    const double amax = exp10((double)G.max_gain_db / 20.0);
    float a = G.a_cur;
    for (long long c = 1; c <= nc; c++) {
        const long long m = m0 + c;
        double L;
        if (m >= 4) {
            L = ld_gates(G.q, 1, m - 3, 4.0 * (double)S, red);
        } else {
            double sum = 0.0;
            for (long long j = 0; j < m; j++) sum += G.q[j];
            L = sum > 0.0 ? ld_block_loudness(sum / (double)(m * S)) : -INFINITY;
            if (L <= -70.0) L = -INFINITY;
        }
        if (L > -INFINITY) a = (float)fmin(exp10(((double)G.target - L) / 20.0), amax);
        if (threadIdx.x == 0) { G.lufs[c - 1] = L; G.gains[c - 1] = a; }
    }
    __syncthreads();
    // (6) each sample's gain, ramped over its step from the gain at the step's start to the one at its end; then the
    // clamp and the chunk's own gain
    const auto a_at = [&](long long m) { return m == m0 - 1 ? G.a_prev : m == m0 ? G.a_cur : G.gains[m - m0 - 1]; };
    unsigned long long clip = 0;
    const float vol = G.gain;
    for (long long i = threadIdx.x; i < n; i += LD_THREADS) {
        const long long t = m0 * S + p + i, m = t / S;
        float g;
        if (m == 0) {
            g = a_at(0);
        } else {
            const double a0 = (double)a_at(m - 1), a1 = (double)a_at(m);
            g = (float)__dadd_rn(a0, __ddiv_rn(__dmul_rn(__dsub_rn(a1, a0), (double)(t - m * S + 1)), (double)S));
        }
        float v = __fmul_rn(win[p + i], g);
        if (v > 1.f) { v = 1.f; clip++; }
        else if (v < -1.f) { v = -1.f; clip++; }
        G.y[i] = vol == 1.f ? v : __fmul_rn(v, vol);
    }
    if (clip) atomicAdd(G.clipped, clip);
}

// Frame-level input of a chunk pass: every row is a plain 16-byte copy of its segment's latent row or exact zeros, so a
// chunk's rows hold the same bits whatever else shares the pass.
__global__ void gather_rows_kernel(const GatherSeg* __restrict__ segs, const int* __restrict__ tile_seg, int gran, int c4,
                                   long long n4, float4* __restrict__ s) {
    pdl_trigger(); pdl_wait();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const int r = (int)(i / c4), c = (int)(i - (long long)r * c4);
    const GatherSeg g = segs[tile_seg[r / gran]];
    const int k = r - g.off;                   // >= 0: a segment's tiles start at its first row
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k < g.len) v = reinterpret_cast<const float4*>(g.src)[(g.lo + k) * c4 + c];
    s[i] = v;
}

// ------------------------------------------------------------------ Philox4x32-10 -> N(0,1)
// Four N(0,1) values from one Philox4x32-10 block of counter (c0..c3) under key (k0, k1), by Box-Muller
// (tests/noise_reference.py restates it on the host).
__device__ __forceinline__ void philox_normal4(unsigned c0, unsigned c1, unsigned c2, unsigned c3, unsigned k0,
                                               unsigned k1, float v[4]) {
#pragma unroll
    for (int r = 0; r < 10; r++) {
        philox_round(c0, c1, c2, c3, k0, k1);
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    const float u0 = ((float)c0 + 0.5f) * 2.3283064365386963e-10f;
    const float u1 = ((float)c1 + 0.5f) * 2.3283064365386963e-10f;
    const float u2 = ((float)c2 + 0.5f) * 2.3283064365386963e-10f;
    const float u3 = ((float)c3 + 0.5f) * 2.3283064365386963e-10f;
    const float r0 = sqrtf(-2.f * logf(u0)), r1 = sqrtf(-2.f * logf(u2));
    float s0, cs0, s1, cs1;
    sincosf(6.283185307179586f * u1, &s0, &cs0);
    sincosf(6.283185307179586f * u3, &s1, &cs1);
    v[0] = r0 * cs0; v[1] = r0 * s0; v[2] = r1 * cs1; v[3] = r1 * s1;
}

// Positional noise: quad i4 of the buffer is counter (i4, i4 >> 32, stream_id, stream_id >> 32) under the voice's key.
__global__ void randn_kernel(float* __restrict__ out, long long n, unsigned long long seed,
                             unsigned long long stream_id) {
    pdl_trigger(); pdl_wait();
    const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i4 * 4 >= n) return;
    float v[4];
    philox_normal4((unsigned)i4, (unsigned)(i4 >> 32), (unsigned)stream_id, (unsigned)(stream_id >> 32), (unsigned)seed,
                   (unsigned)(seed >> 32), v);
    for (int e = 0; e < 4; e++)
        if (i4 * 4 + e < n) out[i4 * 4 + e] = v[e];
}

// randn_kernel's buffer [rows][cols] with keyed draws for seeded segments.  The quad starting at row r, column c
// belongs to the segment of r's granule; when r is a valid row of a seeded segment it is counter (q, q >> 32, tag, 0)
// under key (seed, seed >> 32), q = ((r - off) * cols + c) / 4, off the segment's first row.  That draw depends on the
// seed, the tensor (tag), the row within the utterance and the column only, never on the batch around it.  Every other
// quad (gap rows, unseeded segments) gets randn_kernel's value at the same flat index.  cols is 2 at the id level
// (segments start on 64-row boundaries, so a quad never leaves its segment; the second row of the last quad of an odd
// length segment is a gap row that takes the keyed value, and no consumer reads it) and inter, a multiple of 4, at the
// frame level.
template <typename Seg>
__global__ void randn_seg_kernel(float* __restrict__ out, long long n, unsigned long long seed,
                                 unsigned long long stream_id, int cols, unsigned tag,
                                 const NoiseSeed* __restrict__ seeds, const Seg* __restrict__ segs,
                                 const int* __restrict__ seg_of_gran, RowMap map) {
    pdl_trigger(); pdl_wait();
    const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i4 * 4 >= n) return;
    const int r = (int)(i4 * 4 / cols), c = (int)(i4 * 4 - (long long)r * cols);
    unsigned c0 = (unsigned)i4, c1 = (unsigned)(i4 >> 32), c2 = (unsigned)stream_id, c3 = (unsigned)(stream_id >> 32);
    unsigned long long key = seed;
    if (row_valid(map, r)) {
        const int s = seg_of_gran[r / map.gran];
        const NoiseSeed ns = seeds[s];
        if (ns.seeded) {
            const unsigned long long q = ((unsigned long long)(r - segs[s].off) * (unsigned)cols + (unsigned)c) >> 2;
            c0 = (unsigned)q; c1 = (unsigned)(q >> 32); c2 = tag; c3 = 0u;
            key = ns.seed;
        }
    }
    float v[4];
    philox_normal4(c0, c1, c2, c3, (unsigned)key, (unsigned)(key >> 32), v);
    for (int e = 0; e < 4; e++)
        if (i4 * 4 + e < n) out[i4 * 4 + e] = v[e];
}

// speaker conditioning: one warp per row of the stacked 1x1 conditioning convs, one grid row (blockIdx.y) per speaker slot
__global__ void __launch_bounds__(256) cond_bias_kernel(const float* __restrict__ w, const float* __restrict__ base,
                                                        const float* __restrict__ emb_g, const int* __restrict__ sid,
                                                        int rows, int gin, float* __restrict__ out) {
    pdl_trigger(); pdl_wait();
    const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= rows) return;
    const float* g = emb_g + (size_t)(sid ? sid[blockIdx.y] : (int)blockIdx.y) * gin;
    out += (size_t)blockIdx.y * rows;
    float s = 0.f;
    for (int k = lane; k < gin; k += 32) s = fmaf(w[(size_t)r * gin + k], g[k], s);
    s = warp_sum(s);
    if (lane == 0) out[r] = base[r] + s;
}

// blended speaker embeddings: one thread per column k, one grid row (blockIdx.y) per slot; the slot's terms
// [off[slot], off[slot + 1]) are accumulated in their (canonical) order, g[k] = fmaf(w_i, emb_g[s_i][k], g[k]) from 0
__global__ void __launch_bounds__(128) blend_g_kernel(const float* __restrict__ emb_g, const int* __restrict__ off,
                                                      const BlendTerm* __restrict__ terms, int gin, float* __restrict__ g) {
    pdl_trigger(); pdl_wait();
    const int k = blockIdx.x * 128 + threadIdx.x;
    if (k >= gin) return;
    float acc = 0.f;
    for (int i = off[blockIdx.y]; i < off[blockIdx.y + 1]; i++) acc = fmaf(terms[i].w, emb_g[(size_t)terms[i].s * gin + k], acc);
    g[(size_t)blockIdx.y * gin + k] = acc;
}

template <typename K>
void set_smem(K kern, size_t bytes) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}

}  // namespace

// ====================================================================== launchers
void launch_embed(const int* ids_rows, const float* emb, float scale, float* x, int rows, int H, cudaStream_t st) {
    const long long n = (long long)rows * (H / 4);
    launch_pdl(embed_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, ids_rows, emb, scale, x, rows, H);
    g_launch_count++;
}

void launch_ln(const float* x, const float* res1, const float* res2, const float* gamma, const float* beta,
               float* out, int C, int act, RowMap map, cudaStream_t st) {
    const unsigned grid = (map.rows + 7) / 8;
    switch (C) {
        case 96: launch_pdl(ln_kernel<3>, dim3(grid), dim3(256), 0, st, x, res1, res2, gamma, beta, out, act, map); break;
        case 192: launch_pdl(ln_kernel<6>, dim3(grid), dim3(256), 0, st, x, res1, res2, gamma, beta, out, act, map); break;
        case 256: launch_pdl(ln_kernel<8>, dim3(grid), dim3(256), 0, st, x, res1, res2, gamma, beta, out, act, map); break;
        default: throw_launch_error("LayerNorm: unsupported channel count (96 / 192 / 256)");
    }
    g_launch_count++;
}

void launch_dw_ln_gelu(const float* x, const float* wdw, const float* bdw, int k, int dil, const float* gamma,
                       const float* beta, float* out, int C, RowMap map, cudaStream_t st) {
    const unsigned grid = (map.rows + 7) / 8;
    switch (C) {
        case 96: launch_pdl(dw_ln_gelu_kernel<3>, dim3(grid), dim3(256), 0, st, x, wdw, bdw, k, dil, gamma, beta, out, map); break;
        case 192: launch_pdl(dw_ln_gelu_kernel<6>, dim3(grid), dim3(256), 0, st, x, wdw, bdw, k, dil, gamma, beta, out, map); break;
        case 256: launch_pdl(dw_ln_gelu_kernel<8>, dim3(grid), dim3(256), 0, st, x, wdw, bdw, k, dil, gamma, beta, out, map); break;
        default: throw_launch_error("DDSConv: unsupported channel count (96 / 192 / 256)");
    }
    g_launch_count++;
}

static int att_tpad(int max_len) { return (max_len + 3) & ~3; }

size_t attention_smem_bytes(int max_len, int D) {
    const int tpad = att_tpad(max_len);
    return sizeof(float) * ((size_t)ATT_QT * D + (size_t)ATT_QT * tpad + ATT_QT * 32 + ATT_QT + 4 * ATT_QT * D);
}

void launch_attention(const float* qkv, int ldq, const float* relk, const float* relv, int window, float* out,
                      int ldo, int H, int heads, const SegInfo* segs, int nseg, int max_len, cudaStream_t st) {
    const int D = H / heads;
    const int tpad = att_tpad(max_len);
    const size_t smem = attention_smem_bytes(max_len, D);
    dim3 grid((max_len + ATT_QT - 1) / ATT_QT, heads, nseg);
    if (D == 96) {
        set_smem(attention_kernel<96>, smem);
        launch_pdl(attention_kernel<96>, dim3(grid), dim3(192), smem, st, qkv, ldq, relk, relv, window, out, ldo, H, segs, tpad);
    } else if (D == 48) {
        set_smem(attention_kernel<48>, smem);
        launch_pdl(attention_kernel<48>, dim3(grid), dim3(96), smem, st, qkv, ldq, relk, relv, window, out, ldo, H, segs, tpad);
    } else throw_launch_error("attention: unsupported head size (96 / 48)");
    g_launch_count++;
}

void launch_attn_softmax(float* S, int Tp, const float* qkv, int ldq, const float* relk, const float* relv, int window,
                         float* orel, int ldo, int H, int heads, int RX, const SegInfo* segs, const int* seg_of_gran,
                         int gran, int max_len, cudaStream_t st) {
    const int D = H / heads;
    dim3 grid((RX + 7) / 8, heads);
    if ((D != 96 && D != 48) || max_len > ATT_TC_MAX || 2 * window + 1 > 32) throw_launch_error("attn_softmax: unsupported head size / length");
    auto k = D == 96 ? (max_len <= 640 ? attn_softmax_kernel<96, 20> : attn_softmax_kernel<96, 40>)
                     : (max_len <= 640 ? attn_softmax_kernel<48, 20> : attn_softmax_kernel<48, 40>);
    launch_pdl(k, dim3(grid), dim3(256), 0, st, S, Tp, qkv, ldq, relk, relv, window, orel, ldo, RX, segs, seg_of_gran, gran);
    g_launch_count++;
}

void launch_flow_pre(const float* z, int zcol, const float* w, const float* b, const float* g, float* h, int C,
                     RowMap map, cudaStream_t st) {
    const long long n = (long long)map.rows * C;
    launch_pdl(flow_pre_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, z, zcol, w, b, g, h, C, map);
    g_launch_count++;
}

void launch_spline(const float* h29, int ldh, float* z, int tcol, int bins, float inv_sqrt_filter, RowMap map,
                   cudaStream_t st) {
    (void)bins;   // 10 bins is the only configuration Piper ships (SURVEY Appendix A)
    launch_pdl(spline_kernel<10>, dim3((map.rows + 127) / 128), dim3(128), 0, st, h29, ldh, z, tcol, inv_sqrt_filter, map);
    g_launch_count++;
}

void launch_scale_copy2(const float* eps, const float* s, const int* seg_of_gran, float* z, RowMap map, cudaStream_t st) {
    launch_pdl(scale_copy2_kernel, dim3((map.rows + 255) / 256), dim3(256), 0, st, eps, s, seg_of_gran, z, map);
    g_launch_count++;
}

void launch_durations(const float* z, float m0, float logs0, const float* length_scale, const SegInfo* segs, int nseg,
                      float* logw, int* cum, int* y_len, cudaStream_t st, const float* dur_scale, const int* dur_frames,
                      const float* fit) {
    launch_pdl(durations_kernel, dim3(nseg), dim3(256), 0, st, z, m0, logs0, length_scale, segs, dur_scale, dur_frames,
               fit, logw, cum, y_len);
    g_launch_count++;
}

void launch_expand(const float* stats, int ldst, int I, const int* cum, const float* eps, const float* noise_scale,
                   float* zp, const FrameSeg* fsegs, const int* ftile_seg, RowMap ymap, cudaStream_t st) {
    launch_pdl(expand_kernel, dim3((ymap.rows + 7) / 8), dim3(256), 0, st, stats, ldst, I, cum, eps, noise_scale, zp, fsegs, ftile_seg, ymap);
    g_launch_count++;
}

void launch_conv_post(const float* x, int C, const float* w, float* wav, const FrameSeg* fsegs,
                      const int* ftile_seg, int U, RowMap map, cudaStream_t st) {
    if (U % 4 != 0) throw_launch_error("conv_post: samples per frame must be a multiple of 4");
    const unsigned grid = (map.rows + 511) / 512;
    const size_t smem = sizeof(float) * ((size_t)C * 544 + (size_t)C * 8);
    const int vec_ok = (reinterpret_cast<uintptr_t>(wav) & 15) == 0;     // out_off is a multiple of U samples
    switch (C) {
        case 16: set_smem(conv_post_kernel<16>, smem); launch_pdl(conv_post_kernel<16>, dim3(grid), dim3(256), smem, st, x, w, wav, fsegs, ftile_seg, U, map, vec_ok); break;
        case 32: set_smem(conv_post_kernel<32>, smem); launch_pdl(conv_post_kernel<32>, dim3(grid), dim3(256), smem, st, x, w, wav, fsegs, ftile_seg, U, map, vec_ok); break;
        case 64: set_smem(conv_post_kernel<64>, smem); launch_pdl(conv_post_kernel<64>, dim3(grid), dim3(256), smem, st, x, w, wav, fsegs, ftile_seg, U, map, vec_ok); break;
        default: throw_launch_error("conv_post: unsupported channel count (16 / 32 / 64)");
    }
    g_launch_count++;
}

void launch_pcm(const float* wav, const FrameSeg* fsegs, const PcmPost* posts, int nseg, int hop, long long max_samples,
                unsigned* maxbits, int fmt, void* out, cudaStream_t st) {
    if (fmt != PCM_I16 && fmt != PCM_MULAW && fmt != PCM_ALAW) throw_launch_error("pcm: format is not i16 or G.711");
    if (nseg <= 0) return;
    cudaMemsetAsync(maxbits, 0, sizeof(unsigned) * nseg, st);
    int bx = (int)((max_samples + 256 * 8 - 1) / (256 * 8));
    if (bx < 1) bx = 1;
    if (bx > 1024) bx = 1024;
    dim3 grid(bx, nseg);
    launch_pdl(i16_absmax_kernel, dim3(grid), dim3(256), 0, st, wav, fsegs, posts, hop, maxbits);
    if (fmt == PCM_I16)
        launch_pdl(i16_convert_kernel<PCM_I16>, dim3(grid), dim3(256), 0, st, wav, fsegs, posts, hop, maxbits, (short*)out);
    else if (fmt == PCM_MULAW)
        launch_pdl(i16_convert_kernel<PCM_MULAW>, dim3(grid), dim3(256), 0, st, wav, fsegs, posts, hop, maxbits, (uint8_t*)out);
    else
        launch_pdl(i16_convert_kernel<PCM_ALAW>, dim3(grid), dim3(256), 0, st, wav, fsegs, posts, hop, maxbits, (uint8_t*)out);
    g_launch_count += 2;
}

// One thread per value: the G.711 byte of x[i] (sb200_debug_g711's device side).
__global__ void g711_kernel(const short* __restrict__ x, long long n, int fmt, uint8_t* __restrict__ out) {
    pdl_trigger(); pdl_wait();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        out[i] = fmt == PCM_MULAW ? g711_ulaw(x[i]) : g711_alaw(x[i]);
}
void launch_g711(const short* x, long long n, int fmt, uint8_t* out, cudaStream_t st) {
    if (n <= 0) return;
    const long long bx = std::min<long long>((n + 255) / 256, 4096);
    launch_pdl(g711_kernel, dim3((unsigned)bx), dim3(256), 0, st, x, n, fmt, out);
    g_launch_count++;
}

void launch_resample(const float* wav, const FrameSeg* fsegs, const PcmPost* posts, int hop, const ResampleSeg* segs,
                     int nseg, long long max_out, int smem_floats, float* out, cudaStream_t st) {
    if (nseg <= 0) return;
    const size_t smem = sizeof(float) * (size_t)smem_floats;
    if (smem > 48 * 1024) throw_launch_error("resample: input span exceeds 48 KB of shared memory");
    const long long bx = std::min<long long>(std::max<long long>((max_out + RS_OUTS - 1) / RS_OUTS, 1), 4096);
    launch_pdl(resample_kernel, dim3((unsigned)bx, nseg), dim3(256), smem, st, wav, fsegs, posts, hop, segs, out);
    g_launch_count++;
}

void launch_loudness(float* wav, const LoudSeg* segs, int nseg, double* scratch, double* lufs, float* gain, cudaStream_t st) {
    if (nseg <= 0) return;
    launch_pdl(loudness_kernel, dim3(nseg), dim3(LD_THREADS), 0, st, wav, segs, scratch, lufs, gain);
    g_launch_count++;
}

void launch_loudness_stream(const LoudStreamSeg* segs, int nseg, cudaStream_t st) {
    if (nseg == 0) return;
    launch_pdl(loudness_stream_kernel, dim3(nseg), dim3(LD_THREADS), 0, st, segs);
    g_launch_count++;
}

void launch_gather_rows(const GatherSeg* segs, const int* tile_seg, int gran, int rows, int cols, float* s, cudaStream_t st) {
    if (cols % 4 != 0) throw_launch_error("gather_rows: channel count must be a multiple of 4");
    const long long n4 = (long long)rows * (cols / 4);
    launch_pdl(gather_rows_kernel, dim3((unsigned)((n4 + 255) / 256)), dim3(256), 0, st, segs, tile_seg, gran, cols / 4, n4,
               reinterpret_cast<float4*>(s));
    g_launch_count++;
}

void launch_randn(float* out, long long n, unsigned long long seed, unsigned long long stream_id, cudaStream_t st) {
    const long long n4 = (n + 3) / 4;
    launch_pdl(randn_kernel, dim3((unsigned)((n4 + 255) / 256)), dim3(256), 0, st, out, n, seed, stream_id);
    g_launch_count++;
}

template <typename Seg>
static void randn_seg(float* out, int cols, unsigned tag, unsigned long long seed, unsigned long long stream_id,
                      const NoiseSeed* seeds, const Seg* segs, const int* seg_of_gran, RowMap map, cudaStream_t st) {
    const long long n = (long long)map.rows * cols, n4 = (n + 3) / 4;
    launch_pdl(randn_seg_kernel<Seg>, dim3((unsigned)((n4 + 255) / 256)), dim3(256), 0, st, out, n, seed, stream_id, cols,
               tag, seeds, segs, seg_of_gran, map);
    g_launch_count++;
}
void launch_randn_seeded(float* out, int cols, unsigned tag, unsigned long long seed, unsigned long long stream_id,
                         const NoiseSeed* seeds, const SegInfo* segs, const int* seg_of_gran, RowMap map, cudaStream_t st) {
    randn_seg(out, cols, tag, seed, stream_id, seeds, segs, seg_of_gran, map, st);
}
void launch_randn_seeded(float* out, int cols, unsigned tag, unsigned long long seed, unsigned long long stream_id,
                         const NoiseSeed* seeds, const FrameSeg* segs, const int* seg_of_gran, RowMap map, cudaStream_t st) {
    randn_seg(out, cols, tag, seed, stream_id, seeds, segs, seg_of_gran, map, st);
}

void launch_cond_bias(const float* w, const float* base, const float* emb_g, const int* sid, int nslots, int rows, int gin,
                      float* out, cudaStream_t st) {
    launch_pdl(cond_bias_kernel, dim3((rows + 7) / 8, nslots), dim3(256), 0, st, w, base, emb_g, sid, rows, gin, out);
    g_launch_count++;
}

void launch_blend_g(const float* emb_g, const int* off, const BlendTerm* terms, int nslots, int gin, float* g,
                    cudaStream_t st) {
    launch_pdl(blend_g_kernel, dim3((gin + 127) / 128, nslots), dim3(128), 0, st, emb_g, off, terms, gin, g);
    g_launch_count++;
}

}  // namespace sb200
