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

__device__ __forceinline__ int pr_quant(const float* __restrict__ x, long long x0, long long n, long long i) {
    if (i < 0 || i >= n) return 0;
    return (int)__fmul_rn(fminf(fmaxf(x[i - x0], -1.f), 1.f), 32767.f);      // truncating cast
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
    if (!g.stretch || g.k1 <= g.k0) return;
    const float* x = wav + g.in_off;
    int* out = offsets + g.d_off - g.d0;      // out[k]: frame k's delta
    const int Hs = g.Hs, N = 2 * Hs, D = g.D, L = 2 * D + 1;
    int* ref = pq;
    int* cand = pq + N;
    if (g.k0 == 0 && threadIdx.x == 0) out[0] = 0;
    // the frame before the first one computed: frame 0 (delta 0, at 0) or the last one an earlier pass computed
    const int k_first = max(g.k0, 1);
    long long a_prev = prosody_analysis(Hs, g.alpha, k_first - 1);
    int d_prev = k_first == 1 ? 0 : out[k_first - 1];
    for (int k = k_first; k < g.k1; k++) {
        const long long a = prosody_analysis(Hs, g.alpha, k), c = a_prev + d_prev + Hs;
        for (int i = threadIdx.x; i < N; i += PR_THREADS) ref[i] = pr_quant(x, g.x0, g.n, c + i);
        for (int i = threadIdx.x; i < N + 2 * D; i += PR_THREADS) cand[i] = pr_quant(x, g.x0, g.n, a - D + i);
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
    // out[m - ob]: stretched sample m
    float* out = g.pitch ? s + g.s_off : y + g.y_off;
    const long long ob = g.pitch ? g.s0 : g.m0;
    const int* dl = offsets + g.d_off - g.d0;
    const int Hs = g.Hs, N = 2 * Hs;
    for (long long m = g.m0 + i0; m < g.m1; m += step) {
        const int k = (int)(m / Hs), r = (int)(m - (long long)k * Hs);
        const long long p1 = prosody_analysis(Hs, g.alpha, k) + dl[k] + r;
        const long long p0 = prosody_analysis(Hs, g.alpha, k - 1) + (k > 0 ? dl[k - 1] : 0) + r + Hs;
        const float x1 = p1 >= 0 && p1 < g.n ? x[p1 - g.x0] : 0.f, x0 = p0 >= 0 && p0 < g.n ? x[p0 - g.x0] : 0.f;
        out[m - ob] = __fadd_rn(__fmul_rn(pr_window(r, N), x1), __fmul_rn(pr_window(r + Hs, N), x0));
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
    // in[i - ib]: stretched sample i
    const float* in = g.stretch ? s + g.s_off : wav + g.in_off;
    const long long ib = g.stretch ? g.s0 : g.x0;
    float* out = y + g.y_off - g.j0;
    const double pi = 3.14159265358979323846, p = g.p, c = p > 1.0 ? 1.0 / p : 1.0, W = 16.0 / c;
    double sdc, cdc, sdw, cdw;            // the per-tap rotations: pi c and pi / W
    sincospi(c, &sdc, &cdc);
    sincospi(1.0 / W, &sdw, &cdw);
    for (long long a = g.j0 + (long long)blockIdx.x * PP_OUTS; a < g.j1; a += (long long)gridDim.x * PP_OUTS) {
        const long long jb = min(a + (long long)PP_OUTS, g.j1);
        const long long lo = max(0ll, (long long)floor((double)a * p - W) + 1);
        const long long hi = min(g.n1 - 1, (long long)ceil((double)(jb - 1) * p + W) - 1);
        for (int q = threadIdx.x; q <= (int)(hi - lo); q += PP_OUTS) xs[q] = in[lo + q - ib];
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

// ------------------------------------------------------------------ a stream's chunk pass: staging and carry
// Staging writes each segment's input window (the history, then the chunk after its post-path), the stretched history
// and the two deltas before its first frame; the carry copies the tails the next pass reads into the stream's other
// buffers, so no block reads what another writes.
__global__ void prosody_stage_kernel(const float* __restrict__ src, const FrameSeg* __restrict__ fsegs,
                                     const PcmPost* __restrict__ posts, int hop, const ProsodySeg* __restrict__ segs,
                                     const ProsodyCarry* __restrict__ cs, float* __restrict__ wav, float* __restrict__ s,
                                     int* __restrict__ offsets) {
    pdl_trigger(); pdl_wait();
    const ProsodySeg g = segs[blockIdx.y];
    const ProsodyCarry c = cs[blockIdx.y];
    const PcmSeg x = pcm_seg(src, fsegs[c.chunk], posts + c.chunk, hop);
    float* w = wav + g.in_off;
    const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, step = (long long)gridDim.x * blockDim.x;
    for (long long i = i0; i < c.h_in + x.n; i += step) w[i] = i < c.h_in ? c.in_hist[i] : pcm_value(x, i - c.h_in);
    for (long long i = i0; i < c.h_s; i += step) s[g.s_off + i] = c.s_hist[i];
    if (g.stretch && i0 < 2) offsets[g.d_off + i0] = c.d_hist[i0];
}

__global__ void prosody_carry_kernel(const float* __restrict__ wav, const float* __restrict__ s,
                                     const int* __restrict__ offsets, const ProsodySeg* __restrict__ segs,
                                     const ProsodyCarry* __restrict__ cs) {
    pdl_trigger(); pdl_wait();
    const ProsodySeg g = segs[blockIdx.y];
    const ProsodyCarry c = cs[blockIdx.y];
    const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, step = (long long)gridDim.x * blockDim.x;
    for (long long i = i0; i < c.in_keep; i += step) c.in_next[i] = wav[g.in_off + c.in_from + i];
    for (long long i = i0; i < c.s_keep; i += step) c.s_next[i] = s[g.s_off + c.s_from + i];
    if (g.stretch && i0 < 2) c.d_next[i0] = offsets[g.d_off + c.d_from + i0];
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

void launch_prosody_stage(const float* src, const FrameSeg* fsegs, const PcmPost* posts, int hop, const ProsodySeg* segs,
                          const ProsodyCarry* cs, int nseg, long long max_in, float* wav, float* s, int* offsets,
                          cudaStream_t st) {
    if (nseg <= 0) return;
    launch_pdl(prosody_stage_kernel, dim3(grid_for(max_in, 1024), nseg), dim3(256), 0, st, src, fsegs, posts, hop, segs,
               cs, wav, s, offsets);
    g_launch_count++;
}

void launch_prosody_carry(const float* wav, const float* s, const int* offsets, const ProsodySeg* segs,
                          const ProsodyCarry* cs, int nseg, long long max_keep, cudaStream_t st) {
    if (nseg <= 0) return;
    launch_pdl(prosody_carry_kernel, dim3(grid_for(max_keep, 1024), nseg), dim3(256), 0, st, wav, s, offsets, segs, cs);
    g_launch_count++;
}

// ------------------------------------------------------------------ the launches of a plan
void ProsodyPlan::add(const ProsodyShape& sh, long long in_off, long long n) {
    ProsodySeg g{};
    g.in_off = in_off; g.n = n; g.n1 = sh.n1; g.n2 = sh.n2;
    g.F = sh.F; g.Hs = sh.Hs; g.D = sh.D; g.stretch = sh.stretch; g.pitch = sh.pitch; g.alpha = sh.alpha; g.p = sh.p;
    g.k1 = sh.F; g.m1 = sh.n1; g.j1 = sh.n2;      // the whole utterance: every other window field 0
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

// ------------------------------------------------------------------ streams
namespace {
double pitch_radius(double p) { return 16.0 / (p > 1.0 ? 1.0 / p : 1.0); }     // W, as the pitch kernel computes it
}  // namespace

void prosody_stream_init(ProsodyStream& ps, int rate, float pitch, float tempo) {
    check_prosody(&pitch, &tempo, 1);
    if (!prosody_asked(pitch) && !prosody_asked(tempo))
        throw Error(19, "a prosody stream needs a pitch or a tempo ratio other than 1 (NaN or 1: none)");
    ps.sh = prosody_shape(rate, 0, pitch, tempo);
    ps.rate = rate; ps.pitch = pitch; ps.tempo = tempo;
    const ProsodyShape& s = ps.sh;
    const int pitch_tail = s.pitch ? 2 * (int)std::ceil(pitch_radius(s.p)) + 4 : 0;
    // The offset chain of the next frame and the overlap-add of the stretched samples after the last emitted one read
    // inputs from min(a_{K-2} + Hs, a_{K-1}) - D on, and the next frame is not ready: fewer than
    // max(ceil(2 Hs / alpha), Hs) + 2 D + N of them are held.
    ps.cap_in = s.stretch ? (int)std::max<double>(std::ceil(2.0 * s.Hs / s.alpha), s.Hs) + 2 * s.D + s.N + 4 : pitch_tail;
    ps.cap_s = s.stretch ? pitch_tail : 0;
}

ProsodyStream* create_prosody_stream(Voice* v, int device, int rate, float pitch, float tempo) {
    std::unique_ptr<ProsodyStream> ps(new ProsodyStream());
    prosody_stream_init(*ps, rate, pitch, tempo);
    ps->v = v; ps->device = device;
    SB_CUDA(cudaSetDevice(device));
    const size_t side = (size_t)ps->cap_in + ps->cap_s + 2;      // floats, floats, two ints
    void* mem = nullptr;
    SB_CUDA(cudaMalloc(&mem, 2 * side * 4));
    ps->mem = mem;
    SB_CUDA(cudaMemset(mem, 0, 2 * side * 4));                   // delta_{-2} = delta_{-1} = 0 (unused) before frame 0
    for (int b = 0; b < 2; b++) {
        float* base = static_cast<float*>(mem) + b * side;
        ps->in_hist[b] = base; ps->s_hist[b] = base + ps->cap_in;
        ps->d_hist[b] = reinterpret_cast<int*>(base + ps->cap_in + ps->cap_s);
    }
    return ps.release();
}

ProsodyStream::~ProsodyStream() {
    if (!mem) return;
    cudaSetDevice(device);
    cudaFree(mem);
}

ProsodyStep prosody_stream_step(const ProsodyStream& ps, long long n_in, bool last) {
    const ProsodyShape& sh = ps.sh;
    const ProsodyCounts& c = ps.c;
    ProsodyStep t{};
    const long long C = c.consumed + n_in;
    t.n_in = n_in;
    t.x0 = c.consumed - c.h_in; t.s0 = c.stretched - c.h_s;
    t.k0 = (int)c.frames; t.m0 = c.stretched; t.j0 = c.emitted;
    auto a = [&](long long k) { return prosody_analysis(sh.Hs, sh.alpha, k); };
    long long K = c.frames, S, J;
    if (last) {
        const ProsodyShape e = prosody_shape(ps.rate, C, ps.pitch, ps.tempo);
        K = e.F; S = e.n1; J = e.n2;
    } else {
        S = C;
        if (sh.stretch) {
            // frame k is ready once its offset search and its overlap-add read only inputs that have arrived, with the
            // continuation point bounded by delta_{k-1} <= D; a stretched sample once it lies below the n1 of any
            // longer input
            while (std::max(a(K - 1) + sh.D + sh.Hs + sh.N, a(K) + sh.D + sh.N) <= C) K++;
            S = std::min(K * sh.Hs, (long long)std::floor((double)C * sh.alpha + 0.5));
        }
        J = S;
        if (sh.pitch) {
            const double W = pitch_radius(sh.p);
            J = c.emitted;
            while ((long long)std::ceil((double)J * sh.p + W) <= S) J++;
        }
    }
    if (K < c.frames || S < c.stretched || J < c.emitted || K > INT_MAX)
        throw Error(19, "internal: a prosody stream would go back");
    t.k1 = (int)K; t.m1 = S; t.j1 = J;
    ProsodyCounts& nx = t.next;
    nx.consumed = C; nx.frames = K; nx.stretched = S; nx.emitted = J;
    // the tails the next pass reads: none after the last chunk
    long long in_from = C, s_from = S;
    if (!last) {
        const long long pitch_from =
            sh.pitch ? std::min(S, std::max(0ll, (long long)std::floor((double)J * sh.p - pitch_radius(sh.p)) + 1)) : S;
        if (sh.stretch) {
            in_from = K == 0 ? 0 : std::max(0ll, std::min(a(K - 2) + sh.Hs, a(K - 1)) - sh.D);
            in_from = std::min(in_from, C);
            s_from = pitch_from;
        } else {
            in_from = pitch_from;        // the stretched signal is the input itself
        }
    }
    t.in_from = in_from; t.s_from = s_from;
    nx.h_in = (int)(C - in_from);
    nx.h_s = sh.stretch && sh.pitch ? (int)(S - s_from) : 0;
    if (in_from < t.x0 || s_from < t.s0 || nx.h_in > ps.cap_in || nx.h_s > ps.cap_s)
        throw Error(19, "internal: a prosody stream's history exceeds its buffers");
    return t;
}

void ProsodyPlan::add_stream(const ProsodyStream& ps, const ProsodyStep& t) {
    const ProsodyShape& sh = ps.sh;
    ProsodySeg g{};
    g.Hs = sh.Hs; g.D = sh.D; g.stretch = sh.stretch; g.pitch = sh.pitch; g.alpha = sh.alpha; g.p = sh.p;
    const long long nx = ps.c.h_in + t.n_in;
    g.in_off = in_total; in_total += nx;
    g.x0 = t.x0; g.n = t.next.consumed;
    g.n1 = t.m1; g.n2 = t.j1; g.F = t.k1;
    g.k0 = t.k0; g.k1 = t.k1; g.m0 = t.m0; g.m1 = t.m1; g.j0 = t.j0; g.j1 = t.j1;
    g.y_off = y_total; y_total += t.j1 - t.j0;
    const long long frames = t.k1 - t.k0, stretched = t.m1 - t.m0, outs = t.j1 - t.j0;
    max_in = std::max(max_in, nx);
    max_keep = std::max<long long>(max_keep, std::max({t.next.h_in, t.next.h_s, 2}));
    if (sh.stretch) {
        g.d0 = t.k0 - 2; g.d_off = d_total; d_total += 2 + frames;
        if (sh.pitch) { g.s0 = t.s0; g.s_off = s_total; s_total += ps.c.h_s + stretched; }
        max_ola = std::max(max_ola, stretched);
        smem_ints = std::max(smem_ints, 2 * sh.N + 2 * sh.D);
        stretch_flops += 2.0 * frames * (2.0 * sh.D + 1.0) * sh.N + 3.0 * (double)stretched;
        stretch_bytes += 4.0 * (frames * (2.0 * sh.N + 2.0 * sh.D) + 3.0 * (double)stretched + frames);
        steps += frames;
    }
    stretch_bytes += 4.0 * (2.0 * nx + t.next.h_in + t.next.h_s);      // staging and carry
    if (sh.pitch) {
        const double taps = 2.0 * pitch_radius(sh.p) + 1.0;
        max_pitch = std::max(max_pitch, outs);
        pitch_flops += 2.0 * (double)outs * taps;
        pitch_bytes += 4.0 * ((double)(sh.stretch ? stretched : t.n_in) + (double)outs);
    }
    segs.push_back(g);
}

ProsodyCarry prosody_carry(const ProsodyStream& ps, const ProsodyStep& t, int chunk) {
    ProsodyCarry c{};
    c.chunk = chunk;
    c.h_in = ps.c.h_in; c.h_s = ps.c.h_s;
    c.in_keep = t.next.h_in; c.s_keep = t.next.h_s;
    c.in_from = t.in_from - t.x0; c.s_from = t.s_from - t.s0; c.d_from = t.k1 - t.k0;
    c.in_hist = ps.in_hist[ps.cur]; c.s_hist = ps.s_hist[ps.cur]; c.d_hist = ps.d_hist[ps.cur];
    c.in_next = ps.in_hist[1 - ps.cur]; c.s_next = ps.s_hist[1 - ps.cur]; c.d_next = ps.d_hist[1 - ps.cur];
    return c;
}

void launch_prosody_stream_stretch(const ProsodyPlan& p, const ProsodySeg* segs, const ProsodyCarry* cs,
                                   const float* src, const FrameSeg* fsegs, const PcmPost* posts, int hop, float* x,
                                   float* s, int* offsets, float* y, cudaStream_t st) {
    const int n = (int)p.segs.size();
    launch_prosody_stage(src, fsegs, posts, hop, segs, cs, n, p.max_in, x, s, offsets, st);
    if (p.smem_ints) launch_prosody_offsets(x, segs, n, p.smem_ints, offsets, st);
    if (p.max_ola) launch_prosody_ola(x, segs, n, p.max_ola, offsets, s, y, st);
    launch_prosody_carry(x, s, offsets, segs, cs, n, p.max_keep, st);
}

void prosody_stream_advance(ProsodyStream& ps, const ProsodyStep& t, bool last) {
    ps.c = t.next;
    ps.cur ^= 1;
    ps.ended = last;
}

std::vector<long long> prosody_stream_plan(int rate, float pitch, float tempo, const long long* chunk_lens, size_t n) {
    ProsodyStream ps;
    prosody_stream_init(ps, rate, pitch, tempo);
    std::vector<long long> out(n);
    for (size_t k = 0; k < n; k++) {
        if (chunk_lens[k] < 0) throw Error(19, "chunk " + std::to_string(k) + ": negative length");
        const ProsodyStep t = prosody_stream_step(ps, chunk_lens[k], k + 1 == n);
        out[k] = t.j1 - t.j0;
        prosody_stream_advance(ps, t, k + 1 == n);
    }
    return out;
}

}  // namespace sb200
