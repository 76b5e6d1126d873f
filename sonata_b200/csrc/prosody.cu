// Pitch and tempo by caller-chosen ratios, on the decoder's waveform at the voice's own rate (DESIGN.md section 4,
// "Pitch and tempo").  Stage 1 stretches time by alpha = pitch / tempo with WSOLA (Verhelst & Roelands, ICASSP 1993):
// frames of N = 2 Hs samples, Hann-windowed and overlap-added at a hop of Hs, each taken from the input near
// a_k = round(k Hs / alpha) at the offset in [-D, D] that best continues the previous frame.  Stage 2 resamples by the
// pitch ratio with a Blackman-windowed sinc.  Offsets are an argmax over exact integer scores of the signal quantised
// to 16 bits, so they are the same numbers on any machine; the waveform stages are f32 with a fixed evaluation order,
// so an utterance has the same bits in any batch.
#include "engine.h"
#include <algorithm>
#include <climits>
#include <cmath>

namespace sb200 {

// ------------------------------------------------------------------ host: checks and the plan
namespace {
bool prosody_asked(float v) { return !std::isnan(v) && v != 1.f; }
}  // namespace

bool check_prosody(const float* pitch, const float* tempo, size_t B) {
    bool any = false;
    for (size_t b = 0; b < B; b++) {
        if (pitch && prosody_asked(pitch[b])) {
            if (!(std::isfinite(pitch[b]) && pitch[b] >= 0.5f && pitch[b] <= 2.f))
                throw Error(19, "utterance " + std::to_string(b) + ": pitch ratio " + std::to_string(pitch[b]) +
                                    " is not a finite value in [0.5, 2] (NaN or 1: none)");
            any = true;
        }
        if (tempo && prosody_asked(tempo[b])) {
            if (!(std::isfinite(tempo[b]) && tempo[b] >= 0.25f && tempo[b] <= 4.f))
                throw Error(19, "utterance " + std::to_string(b) + ": tempo ratio " + std::to_string(tempo[b]) +
                                    " is not a finite value in [0.25, 4] (NaN or 1: none)");
            any = true;
        }
    }
    return any;
}

ProsodyShape prosody_shape(int rate, long long n, float pitch, float tempo) {
    if (rate < 1000 || rate > 48000)
        throw Error(19, "prosody: no frame sizes for a rate of " + std::to_string(rate) + " Hz (1000 .. 48000)");
    ProsodyShape s{};
    s.Hs = rate / 100; s.N = 2 * s.Hs; s.D = rate / 160;
    const float p = prosody_asked(pitch) ? pitch : 1.f, t = prosody_asked(tempo) ? tempo : 1.f;
    s.p = (double)p; s.alpha = (double)p / (double)t;
    s.stretch = p != t; s.pitch = p != 1.f;
    s.n1 = s.stretch ? (long long)std::floor((double)n * s.alpha + 0.5) : n;
    s.n2 = s.pitch ? (long long)std::floor((double)s.n1 / s.p + 0.5) : s.n1;
    if (s.n1 > INT_MAX || s.n2 > INT_MAX) throw Error(19, "prosody: the stretched utterance is unreasonably long");
    s.F = s.stretch ? (int)((s.n1 + s.Hs - 1) / s.Hs) : 0;
    return s;
}

// ------------------------------------------------------------------ kernel 1: the offset chain
// One block per segment walks its frames in order.  For frame k it stages q around where the previous frame would
// continue (c = a_{k-1} + delta_{k-1} + Hs) and around a_k, every thread scores lags l, l + blockDim, .. as 64-bit
// integer dot products, and the block takes the argmax with the tie rule (smaller |delta|, then the negative one).
constexpr int PR_THREADS = 288;   // 9 warps: the 2 D + 1 = 275 lags of a 22 050 Hz voice, one each

__device__ __forceinline__ int pr_quant(const float* __restrict__ x, long long n, long long i) {
    if (i < 0 || i >= n) return 0;
    return (int)__fmul_rn(fminf(fmaxf(x[i], -1.f), 1.f), 32767.f);      // truncating cast
}
__device__ __forceinline__ bool pr_better(long long s1, int d1, long long s0, int d0) {
    if (s1 != s0) return s1 > s0;
    const int a1 = abs(d1), a0 = abs(d0);
    return a1 != a0 ? a1 < a0 : d1 < d0;
}

__global__ void __launch_bounds__(PR_THREADS)
prosody_offsets_kernel(const float* __restrict__ wav, const ProsodySeg* __restrict__ segs, int* __restrict__ offsets) {
    extern __shared__ int pq[];
    __shared__ long long ws[PR_THREADS / 32];
    __shared__ int wd[PR_THREADS / 32];
    pdl_trigger(); pdl_wait();
    const ProsodySeg g = segs[blockIdx.x];
    if (!g.stretch || g.F == 0) return;
    const float* x = wav + g.in_off;
    int* out = offsets + g.d_off;
    const int Hs = g.Hs, N = 2 * Hs, D = g.D, L = 2 * D + 1;
    int* ref = pq;
    int* cand = pq + N;
    if (threadIdx.x == 0) out[0] = 0;
    long long a_prev = 0;
    int d_prev = 0;
    for (int k = 1; k < g.F; k++) {
        const long long a = prosody_analysis(Hs, g.alpha, k), c = a_prev + d_prev + Hs;
        for (int i = threadIdx.x; i < N; i += PR_THREADS) ref[i] = pr_quant(x, g.n, c + i);
        for (int i = threadIdx.x; i < N + 2 * D; i += PR_THREADS) cand[i] = pr_quant(x, g.n, a - D + i);
        __syncthreads();
        long long best = LLONG_MIN;      // a thread without a lag loses to every score
        int bd = 0;
        for (int l = threadIdx.x; l < L; l += PR_THREADS) {
            const int* cj = cand + l;
            long long acc = 0;
#pragma unroll 8
            for (int i = 0; i < N; i++) acc += (long long)ref[i] * cj[i];
            if (pr_better(acc, l - D, best, bd)) { best = acc; bd = l - D; }
        }
        for (int o = 16; o > 0; o >>= 1) {
            const long long s2 = __shfl_xor_sync(0xffffffffu, best, o);
            const int d2 = __shfl_xor_sync(0xffffffffu, bd, o);
            if (pr_better(s2, d2, best, bd)) { best = s2; bd = d2; }
        }
        if ((threadIdx.x & 31) == 0) { ws[threadIdx.x >> 5] = best; wd[threadIdx.x >> 5] = bd; }
        __syncthreads();
        best = ws[0]; bd = wd[0];
        for (int w = 1; w < PR_THREADS / 32; w++)
            if (pr_better(ws[w], wd[w], best, bd)) { best = ws[w]; bd = wd[w]; }
        if (threadIdx.x == 0) out[k] = bd;
        a_prev = a; d_prev = bd;
    }
}

// ------------------------------------------------------------------ kernel 2: overlap-add
// s[m] = w[r] x[a_k + d_k + r] + w[r + Hs] x[a_{k-1} + d_{k-1} + r + Hs] with k = m / Hs, r = m - k Hs and the periodic
// Hann window w[i] = 0.5 - 0.5 cos(2 pi i / N) (w[r] + w[r + Hs] = 1): two rounded products and one rounded sum.  A
// segment with neither stage is copied; one with the pitch stage only is left to the pitch kernel.
__device__ __forceinline__ float pr_window(int i, int N) { return (float)(0.5 - 0.5 * cospi(2.0 * (double)i / (double)N)); }

__global__ void prosody_ola_kernel(const float* __restrict__ wav, const ProsodySeg* __restrict__ segs,
                                   const int* __restrict__ offsets, float* __restrict__ s, float* __restrict__ y) {
    pdl_trigger(); pdl_wait();
    const ProsodySeg g = segs[blockIdx.y];
    const float* x = wav + g.in_off;
    const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, step = (long long)gridDim.x * blockDim.x;
    if (!g.stretch) {
        if (!g.pitch)
            for (long long i = i0; i < g.n; i += step) y[g.y_off + i] = x[i];
        return;
    }
    float* out = g.pitch ? s + g.s_off : y + g.y_off;
    const int* dl = offsets + g.d_off;
    const int Hs = g.Hs, N = 2 * Hs;
    for (long long m = i0; m < g.n1; m += step) {
        const int k = (int)(m / Hs), r = (int)(m - (long long)k * Hs);
        const long long p1 = prosody_analysis(Hs, g.alpha, k) + dl[k] + r;
        const long long p0 = prosody_analysis(Hs, g.alpha, k - 1) + (k > 0 ? dl[k - 1] : 0) + r + Hs;
        const float x1 = p1 >= 0 && p1 < g.n ? x[p1] : 0.f, x0 = p0 >= 0 && p0 < g.n ? x[p0] : 0.f;
        out[m] = __fadd_rn(__fmul_rn(pr_window(r, N), x1), __fmul_rn(pr_window(r + Hs, N), x0));
    }
}

// ------------------------------------------------------------------ kernel 3: pitch resampling
// y[j] = sum_i s[i] h(j p - i) over the i in [0, n1) with |j p - i| < W, one fmaf chain in ascending i.
// h(u) = c sinc(c u) (0.42 + 0.5 cos(pi u / W) + 0.08 cos(2 pi u / W)), c = min(1, 1 / p), W = 16 / c.  The position j p
// and the phases are double: sin(pi c u) and cos(pi u / W) are evaluated once at the first tap and rotated by the
// constant per-tap angle after it; a tap is rounded to f32 as (sin(pi c u) * window) / (pi u).  A block stages the input
// span of PP_OUTS consecutive outputs in shared memory.  The chain of output j depends on j, p and n1 alone.
__global__ void __launch_bounds__(PP_OUTS)
prosody_pitch_kernel(const float* __restrict__ wav, const float* __restrict__ s, const ProsodySeg* __restrict__ segs,
                     float* __restrict__ y) {
    __shared__ float xs[PP_SPAN];
    pdl_trigger(); pdl_wait();
    const ProsodySeg g = segs[blockIdx.y];
    if (!g.pitch) return;
    const float* in = g.stretch ? s + g.s_off : wav + g.in_off;
    float* out = y + g.y_off;
    const double pi = 3.14159265358979323846, p = g.p, c = p > 1.0 ? 1.0 / p : 1.0, W = 16.0 / c;
    double sdc, cdc, sdw, cdw;            // the per-tap rotations: pi c and pi / W
    sincospi(c, &sdc, &cdc);
    sincospi(1.0 / W, &sdw, &cdw);
    for (long long a = (long long)blockIdx.x * PP_OUTS; a < g.n2; a += (long long)gridDim.x * PP_OUTS) {
        const long long jb = min(a + (long long)PP_OUTS, g.n2);
        const long long lo = max(0ll, (long long)floor((double)a * p - W) + 1);
        const long long hi = min(g.n1 - 1, (long long)ceil((double)(jb - 1) * p + W) - 1);
        for (int q = threadIdx.x; q <= (int)(hi - lo); q += PP_OUTS) xs[q] = in[lo + q];
        __syncthreads();
        const long long j = a + threadIdx.x;
        if (j < jb) {
            const double pos = (double)j * p;
            const long long i0 = max(lo, (long long)floor(pos - W) + 1), i1 = min(hi, (long long)ceil(pos + W) - 1);
            double u = pos - (double)i0, su, cu, sw, cw;
            sincospi(c * u, &su, &cu);
            sincospi(u / W, &sw, &cw);
            float acc = 0.f;
            for (long long i = i0; i <= i1; i++) {
                const double win = 0.42 + 0.5 * cw + 0.08 * (2.0 * cw * cw - 1.0);
                const float h = u == 0.0 ? (float)(c * win) : (float)(su * win) / (float)(pi * u);
                acc = fmaf(xs[i - lo], h, acc);
                const double su2 = su * cdc - cu * sdc, sw2 = sw * cdw - cw * sdw;      // one tap on: u - 1
                cu = cu * cdc + su * sdc; su = su2;
                cw = cw * cdw + sw * sdw; sw = sw2;
                u -= 1.0;
            }
            out[j] = acc;
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------ launchers
namespace {
unsigned grid_for(long long n, int per_block) {
    return (unsigned)std::min<long long>(std::max<long long>((n + per_block - 1) / per_block, 1), 4096);
}
}  // namespace

void launch_prosody_offsets(const float* wav, const ProsodySeg* segs, int nseg, int smem_ints, int* offsets,
                            cudaStream_t st) {
    if (nseg <= 0) return;
    const size_t smem = sizeof(int) * (size_t)smem_ints;
    if (smem > 48 * 1024) throw_launch_error("prosody: frame staging exceeds 48 KB of shared memory");
    launch_pdl(prosody_offsets_kernel, dim3(nseg), dim3(PR_THREADS), smem, st, wav, segs, offsets);
    g_launch_count++;
}

void launch_prosody_ola(const float* wav, const ProsodySeg* segs, int nseg, long long max_out, const int* offsets,
                        float* s, float* y, cudaStream_t st) {
    if (nseg <= 0) return;
    launch_pdl(prosody_ola_kernel, dim3(grid_for(max_out, 1024), nseg), dim3(256), 0, st, wav, segs, offsets, s, y);
    g_launch_count++;
}

void launch_prosody_pitch(const float* wav, const float* s, const ProsodySeg* segs, int nseg, long long max_out, float* y,
                          cudaStream_t st) {
    if (nseg <= 0) return;
    launch_pdl(prosody_pitch_kernel, dim3(grid_for(max_out, PP_OUTS), nseg), dim3(PP_OUTS), 0, st, wav, s, segs, y);
    g_launch_count++;
}

// ------------------------------------------------------------------ the launches of a plan
void ProsodyPlan::add(const ProsodyShape& sh, long long in_off, long long n) {
    ProsodySeg g{};
    g.in_off = in_off; g.n = n; g.n1 = sh.n1; g.n2 = sh.n2;
    g.F = sh.F; g.Hs = sh.Hs; g.D = sh.D; g.stretch = sh.stretch; g.pitch = sh.pitch; g.alpha = sh.alpha; g.p = sh.p;
    g.y_off = y_total; y_total += sh.n2;
    g.d_off = d_total; d_total += sh.F;
    if (sh.stretch && sh.pitch) { g.s_off = s_total; s_total += sh.n1; }
    max_ola = std::max(max_ola, sh.stretch ? sh.n1 : sh.pitch ? 0 : n);
    if (sh.stretch) {
        smem_ints = std::max(smem_ints, 2 * sh.N + 2 * sh.D);
        // per frame step: 2 D + 1 lags of N multiply-adds; the frames staged (N + N + 2 D samples) and the sums written
        stretch_flops += 2.0 * (sh.F > 0 ? sh.F - 1 : 0) * (2.0 * sh.D + 1.0) * sh.N + 3.0 * (double)sh.n1;
        stretch_bytes += 4.0 * ((sh.F > 0 ? sh.F - 1 : 0) * (2.0 * sh.N + 2.0 * sh.D) + 3.0 * (double)sh.n1 + sh.F);
        steps += sh.F > 0 ? sh.F - 1 : 0;
    } else if (!sh.pitch) {
        stretch_bytes += 8.0 * (double)n;
    }
    if (sh.pitch) {
        const double taps = 2.0 * 16.0 * std::max(1.0, sh.p) + 1.0;
        max_pitch = std::max(max_pitch, sh.n2);
        pitch_flops += 2.0 * (double)sh.n2 * taps;
        pitch_bytes += 4.0 * ((double)sh.n1 + (double)sh.n2);
    }
    segs.push_back(g);
    shapes.push_back(sh);
}

}  // namespace sb200
