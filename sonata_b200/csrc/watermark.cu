// Watermark: a keyed spread-spectrum mark added to every sample a marked voice delivers, at the delivered rate, and its
// batched detector (DESIGN.md section 4, "Watermark"; include/sonata_b200.h, sb200_voice_set_watermark).  The mark is
// two P-periodic +-1 chip sequences of the key, the second shifted by the payload, scaled per 10 ms block by the quieter
// of the block and the one before it, so silence stays silent.  The gains use only rounded double operations, so the
// kernel and tests/watermark_reference.py agree bit for bit.  Detection folds each clip modulo P, whitens the fold's
// spectrum and correlates it with both chip sequences in one CTA per clip.
#include "engine.h"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <memory>
#include <mutex>
#include <shared_mutex>

namespace sb200 {

void check_watermark(long long payload, float strength_db) {
    if (payload < 0 || payload >= WM_P)
        throw Error(19, "watermark: payload " + std::to_string(payload) + " is not in [0, 4096)");
    if (!(std::isfinite(strength_db) && strength_db >= -40.f && strength_db <= -10.f))
    {
        char v[32];
        snprintf(v, sizeof v, "%g", (double)strength_db);
        throw Error(19, std::string("watermark: strength_db ") + v + " is not a finite value in [-40, -10] dB");
    }
}

namespace {

// c_j[m]: bit 0 of word 0 of the Philox4x32-10 block of counter (m, j, 0, 0) under the key
__device__ __forceinline__ int wm_chip(unsigned long long key, int j, int m) {
    unsigned c0 = (unsigned)m, c1 = (unsigned)j, c2 = 0u, c3 = 0u, k0 = (unsigned)key, k1 = (unsigned)(key >> 32);
#pragma unroll
    for (int r = 0; r < 10; r++) {
        philox_round(c0, c1, c2, c3, k0, k1);
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return (c0 & 1u) ? 1 : -1;
}

__global__ void wm_chips_kernel(unsigned long long key, signed char* __restrict__ chips) {
    pdl_trigger(); pdl_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 2 * WM_P) chips[i] = (signed char)wm_chip(key, i / WM_P, i % WM_P);
}

// q[i] as the pitch stage quantises it (prosody.cu pr_quant)
__device__ __forceinline__ long long wm_quant(float x) {
    return (long long)(int)__fmul_rn(fminf(fmaxf(x, -1.f), 1.f), 32767.f);
}
__device__ __forceinline__ long long wm_quant(short x) { return (long long)x; }

// ------------------------------------------------------------------ the mark
// A CTA takes runs of WM_RUN blocks; each warp sums whole blocks (the run's and the one before it), then writes whole
// blocks, so a block's samples are read twice by the same warp, the second time from L1.
constexpr int WM_THREADS = 256, WM_WARPS = WM_THREADS / 32, WM_RUN = 32;

__global__ void __launch_bounds__(WM_THREADS)
watermark_kernel(const WatermarkSeg* __restrict__ segs, const float* __restrict__ x, float* __restrict__ y) {
    __shared__ long long S[WM_RUN + 1];
    __shared__ float a[WM_RUN];
    pdl_trigger(); pdl_wait();
    const WatermarkSeg g = segs[blockIdx.y];
    const long long n = g.n, blk = g.blk, K = (n + blk - 1) / blk;
    const float* xs = x + g.x_off;
    float* ys = y + g.y_off;
    const int h = g.h;
    // input i: the held samples, then the new ones
    const auto z = [&](long long i) { return i < h ? g.hold[i] : xs[i - h]; };
    if (!g.chips) {
        for (long long i = (long long)blockIdx.x * WM_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * WM_THREADS)
            ys[i] = z(i);
        return;
    }
    const signed char* __restrict__ chips = g.chips;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (blockIdx.x == 0) {
        // what the stream holds back, and the carry when this pass emits nothing
        for (long long i = n + threadIdx.x; i < h + g.m; i += WM_THREADS) g.hold_out[i - n] = z(i);
        if (g.s_out && K == 0 && threadIdx.x == 0) *g.s_out = g.s_in ? *g.s_in : 0;
    }
    for (long long k0 = (long long)blockIdx.x * WM_RUN; k0 < K; k0 += (long long)gridDim.x * WM_RUN) {
        const int nb = (int)min((long long)WM_RUN, K - k0);
        // S[r]: block k0 - 1 + r; block -1 is the stream's carried block, or block 0
        for (int r = warp; r <= nb; r += WM_WARPS) {
            if (k0 - 1 + r < 0 && g.s_in) {
                if (lane == 0) S[r] = *g.s_in;
                continue;
            }
            const long long k = max(k0 - 1 + r, 0LL), lo = k * blk, hi = min(lo + blk, n);
            long long s = 0;
            for (long long i = lo + lane; i < hi; i += 32) {
                const long long q = wm_quant(z(i));
                s += q * q;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) S[r] = s;
        }
        __syncthreads();
        if (threadIdx.x < nb) {
            const int r = threadIdx.x;
            const long long k = k0 + r;
            const double Lk = (double)min(blk, n - k * blk);
            const double Lp = k == 0 && g.s_in ? (double)blk : (double)min(blk, n - max(k - 1, 0LL) * blk);
            const double E = fmin(__ddiv_rn((double)S[r], Lp), __ddiv_rn((double)S[r + 1], Lk));
            a[r] = __double2float_rn(__ddiv_rn(__dmul_rn(g.alpha, __dsqrt_rn(__dmul_rn(E, 0.5))), 32767.0));
            if (g.s_out && k == K - 1) *g.s_out = S[r + 1];
        }
        __syncthreads();
        for (int r = warp; r < nb; r += WM_WARPS) {
            const long long lo = (k0 + r) * blk, hi = min(lo + blk, n);
            const float ar = a[r];
            for (long long i = lo + lane; i < hi; i += 32) {
                const long long p = g.pos0 + i;
                const int c = __ldg(&chips[p & (WM_P - 1)]) + __ldg(&chips[WM_P + ((p - g.payload) & (WM_P - 1))]);
                ys[i] = __fadd_rn(z(i), __fmul_rn(ar, (float)c));
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------ detection
// The fold: one CTA per tile of WM_FOLD periods of a clip, each thread WM_P / WM_FOLD_THREADS residues, int64 atomics
// into the clip's fold (integer sums, so the order does not matter).
constexpr int WM_FOLD = 16, WM_FOLD_THREADS = 1024, WM_FOLD_R = WM_P / WM_FOLD_THREADS;
struct FoldTile { long long off, n; int clip; };

template <typename T>
__global__ void __launch_bounds__(WM_FOLD_THREADS)
wm_fold_kernel(const T* __restrict__ x, const FoldTile* __restrict__ tiles, unsigned long long* __restrict__ F) {
    pdl_trigger(); pdl_wait();
    const FoldTile t = tiles[blockIdx.x];
    long long acc[WM_FOLD_R] = {};
    for (int p = 0; p < WM_FOLD; p++)
#pragma unroll
        for (int r = 0; r < WM_FOLD_R; r++) {
            const long long i = (long long)p * WM_P + r * WM_FOLD_THREADS + threadIdx.x;
            if (i < t.n) acc[r] += wm_quant(x[t.off + i]);
        }
    unsigned long long* f = F + (size_t)t.clip * WM_P;
#pragma unroll
    for (int r = 0; r < WM_FOLD_R; r++)
        if (acc[r]) atomicAdd(&f[r * WM_FOLD_THREADS + threadIdx.x], (unsigned long long)acc[r]);
}

constexpr int WM_FFT_THREADS = 1024;
__device__ __forceinline__ int wm_rev(int i) { return (int)(__brev((unsigned)i) >> 20); }     // 12-bit reversal

// In-place radix-2 FFT of x (bit-reversed in, natural order out), e^{-2 pi i / P} forward and the conjugate inverse,
// unscaled: formant.cu's shape at 12 bits, two butterflies per thread per stage.  Ends synchronised.
__device__ void wm_fft(double2* x, const double2* tw, bool inverse) {
#pragma unroll 1
    for (int s = 1; s <= 12; s++) {
        const int half = 1 << (s - 1);
        for (int b = threadIdx.x; b < WM_P / 2; b += WM_FFT_THREADS) {
            const int pos = b & (half - 1);
            const int i0 = ((b >> (s - 1)) << s) + pos, i1 = i0 + half;
            double2 w = tw[pos << (12 - s)];
            if (inverse) w.y = -w.y;
            const double2 u = x[i0], v = x[i1];
            const double vr = v.x * w.x - v.y * w.y, vi = v.x * w.y + v.y * w.x;
            x[i0] = make_double2(u.x + vr, u.y + vi);
            x[i1] = make_double2(u.x - vr, u.y - vi);
        }
        __syncthreads();
    }
}
__device__ void wm_twiddles(double2* tw) {
    for (int k = threadIdx.x; k < WM_P / 2; k += WM_FFT_THREADS) {
        double s, c;
        sincospi((double)k / (WM_P / 2), &s, &c);
        tw[k] = make_double2(c, -s);
    }
}
struct WmSmem {
    double2 x[WM_P];
    double2 tw[WM_P / 2];
    double2 red[WM_FFT_THREADS / 32];
    int idx[2][WM_FFT_THREADS / 32];
};

// FFT_P(c_j) into C[j] for j = blockIdx.x
__global__ void __launch_bounds__(WM_FFT_THREADS) wm_spectra_kernel(unsigned long long key, double2* __restrict__ C) {
    extern __shared__ __align__(16) unsigned char wm_raw[];
    WmSmem& sm = *reinterpret_cast<WmSmem*>(wm_raw);
    pdl_trigger(); pdl_wait();
    wm_twiddles(sm.tw);
    const int j = blockIdx.x;
    for (int m = threadIdx.x; m < WM_P; m += WM_FFT_THREADS) sm.x[wm_rev(m)] = make_double2(wm_chip(key, j, m), 0.0);
    __syncthreads();
    wm_fft(sm.x, sm.tw, false);
    for (int k = threadIdx.x; k < WM_P; k += WM_FFT_THREADS) C[(size_t)j * WM_P + k] = sm.x[k];
}

// Sum of v over the CTA, in every thread.  Ends synchronised.
__device__ double2 wm_sum(WmSmem& sm, double2 v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        v.x += __shfl_xor_sync(0xffffffffu, v.x, o);
        v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
    }
    if ((threadIdx.x & 31) == 0) sm.red[threadIdx.x >> 5] = v;
    __syncthreads();
    double2 t = make_double2(0.0, 0.0);
    for (int w = 0; w < WM_FFT_THREADS / 32; w++) { t.x += sm.red[w].x; t.y += sm.red[w].y; }
    __syncthreads();
    return t;
}
// (value, lag) pairs: the larger value, the smaller lag on ties
__device__ __forceinline__ void wm_best(double& v, int& o, double v2, int o2) {
    if (v2 > v || (v2 == v && o2 < o)) { v = v2; o = o2; }
}

// One CTA per clip: X = FFT(F), W = X / |X|, r0 + i r1 = IFFT(conj(W) (C0 + i C1)) / P (both r_j are real), then each
// r_j's peak and its z over the other P - 1 lags.
__global__ void __launch_bounds__(WM_FFT_THREADS)
wm_detect_kernel(const long long* __restrict__ F, const double2* __restrict__ C, WatermarkScore* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char wm_raw[];
    WmSmem& sm = *reinterpret_cast<WmSmem*>(wm_raw);
    pdl_trigger(); pdl_wait();
    wm_twiddles(sm.tw);
    const long long* f = F + (size_t)blockIdx.x * WM_P;
    for (int m = threadIdx.x; m < WM_P; m += WM_FFT_THREADS) sm.x[wm_rev(m)] = make_double2((double)f[m], 0.0);
    __syncthreads();
    wm_fft(sm.x, sm.tw, false);
    for (int k = threadIdx.x; k < WM_P; k += WM_FFT_THREADS) {
        const double2 X = sm.x[k], c0 = C[k], c1 = C[WM_P + k];
        const double mag = sqrt(X.x * X.x + X.y * X.y);
        const double wr = mag > 0.0 ? X.x / mag : 0.0, wi = mag > 0.0 ? -X.y / mag : 0.0;     // conj(W)
        const double cr = c0.x - c1.y, ci = c0.y + c1.x;                                        // C0 + i C1
        sm.x[k] = make_double2(wr * cr - wi * ci, wr * ci + wi * cr);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < WM_P; k += WM_FFT_THREADS) {
        const int q = wm_rev(k);
        if (k < q) { const double2 t = sm.x[k]; sm.x[k] = sm.x[q]; sm.x[q] = t; }
    }
    __syncthreads();
    wm_fft(sm.x, sm.tw, true);
    for (int k = threadIdx.x; k < WM_P; k += WM_FFT_THREADS)
        sm.x[k] = make_double2(sm.x[k].x / WM_P, sm.x[k].y / WM_P);
    __syncthreads();
    // the peaks
    double b0 = -INFINITY, b1 = -INFINITY;
    int o0 = WM_P, o1 = WM_P;
    for (int k = threadIdx.x; k < WM_P; k += WM_FFT_THREADS) {
        wm_best(b0, o0, sm.x[k].x, k);
        wm_best(b1, o1, sm.x[k].y, k);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        wm_best(b0, o0, __shfl_xor_sync(0xffffffffu, b0, o), __shfl_xor_sync(0xffffffffu, o0, o));
        wm_best(b1, o1, __shfl_xor_sync(0xffffffffu, b1, o), __shfl_xor_sync(0xffffffffu, o1, o));
    }
    if ((threadIdx.x & 31) == 0) {
        sm.red[threadIdx.x >> 5] = make_double2(b0, b1);
        sm.idx[0][threadIdx.x >> 5] = o0; sm.idx[1][threadIdx.x >> 5] = o1;
    }
    __syncthreads();
    b0 = b1 = -INFINITY; o0 = o1 = WM_P;
    for (int w = 0; w < WM_FFT_THREADS / 32; w++) {
        wm_best(b0, o0, sm.red[w].x, sm.idx[0][w]);
        wm_best(b1, o1, sm.red[w].y, sm.idx[1][w]);
    }
    __syncthreads();
    // mean, then the population variance, of the other lags
    double2 s = make_double2(0.0, 0.0);
    for (int k = threadIdx.x; k < WM_P; k += WM_FFT_THREADS) {
        if (k != o0) s.x += sm.x[k].x;
        if (k != o1) s.y += sm.x[k].y;
    }
    s = wm_sum(sm, s);
    const double mu0 = s.x / (WM_P - 1), mu1 = s.y / (WM_P - 1);
    double2 d = make_double2(0.0, 0.0);
    for (int k = threadIdx.x; k < WM_P; k += WM_FFT_THREADS) {
        const double e0 = sm.x[k].x - mu0, e1 = sm.x[k].y - mu1;
        if (k != o0) d.x += e0 * e0;
        if (k != o1) d.y += e1 * e1;
    }
    d = wm_sum(sm, d);
    if (threadIdx.x == 0) {
        const double sg0 = sqrt(d.x / (WM_P - 1)), sg1 = sqrt(d.y / (WM_P - 1));
        WatermarkScore r;
        r.z0 = sg0 > 0.0 ? (b0 - mu0) / sg0 : 0.0;
        r.z1 = sg1 > 0.0 ? (b1 - mu1) / sg1 : 0.0;
        r.marked = r.z0 >= 6.5;
        r.payload = r.marked && r.z1 >= 6.5 ? (o0 - o1 + WM_P) % WM_P : -1;
        r.offset = o0;
        out[blockIdx.x] = r;
    }
}

// Device memory of one detection call, freed however the call ends.
struct WmScratch {
    void* p = nullptr;
    ~WmScratch() { if (p) cudaFree(p); }
};

}  // namespace

signed char* build_watermark_chips(unsigned long long key) {
    signed char* chips = nullptr;
    SB_CUDA(cudaMalloc(&chips, 2 * WM_P));
    cudaStream_t st = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
    if (e == cudaSuccess) {
        launch_pdl(wm_chips_kernel, dim3(2 * WM_P / 256), dim3(256), 0, st, key, chips);
        g_launch_count++;
        e = cudaStreamSynchronize(st);
        cudaStreamDestroy(st);
    }
    if (e != cudaSuccess) {
        cudaFree(chips);
        SB_CUDA(e);
    }
    return chips;
}

namespace {
WatermarkSeg marked_seg(const Watermark& wm, long long rate) {
    WatermarkSeg g{};
    g.blk = (int)(rate / 100); g.payload = wm.payload; g.chips = wm.chips;
    g.alpha = std::pow(10.0, (double)wm.strength_db / 20.0);
    return g;
}
}  // namespace

void WatermarkPlan::add(const Watermark& wm, long long off, long long n, int rate) {
    WatermarkSeg g = marked_seg(wm, rate);
    g.x_off = g.y_off = off; g.n = g.m = n;
    const long long K = (n + g.blk - 1) / g.blk;
    max_runs = std::max(max_runs, (K + WM_RUN - 1) / WM_RUN);
    max_n = std::max(max_n, n);
    bytes += 8.0 * (double)n;
    segs.push_back(g);
}

void WatermarkPlan::add_chunk(const WatermarkStream* ws, long long x_off, long long m, bool last) {
    WatermarkSeg g{};
    g.x_off = x_off; g.m = g.n = m; g.y_off = total;
    long long runs = (m + (long long)WM_THREADS * WM_RUN - 1) / ((long long)WM_THREADS * WM_RUN);
    if (ws) {
        g = marked_seg(ws->wm, ws->rate);
        g.x_off = x_off; g.m = m; g.y_off = total;
        g.h = (int)(ws->in - ws->out);
        g.pos0 = ws->out;
        const long long J1 = ws->in + m, end = last ? J1 : J1 / ws->blk * ws->blk;
        g.n = end - ws->out;
        runs = (g.n + g.blk - 1) / g.blk;
        runs = std::max((runs + WM_RUN - 1) / WM_RUN, 1LL);
    }
    max_runs = std::max(max_runs, runs);
    max_n = std::max(max_n, g.n);
    bytes += 4.0 * (double)(m + g.h + g.n);
    total += g.n;
    segs.push_back(g);
}

void launch_watermark(const WatermarkPlan& p, const WatermarkSeg* segs, const float* x, float* y, cudaStream_t st) {
    if (p.segs.empty() || p.max_runs <= 0) return;
    const long long bx = std::min<long long>(p.max_runs, 2048);
    launch_pdl(watermark_kernel, dim3((unsigned)bx, (unsigned)p.segs.size()), dim3(WM_THREADS), 0, st, segs, x, y);
    g_launch_count++;
}

WatermarkStream::~WatermarkStream() {
    if (mem) {
        cudaSetDevice(v->device);
        cudaFree(mem);
    }
}

WatermarkStream* create_watermark_stream(Voice* v, long long rate) {
    Watermark wm;
    {
        std::shared_lock<std::shared_mutex> g(v->cfg_mu);
        if (!v->wm_on) return nullptr;
        wm = v->wm;
    }
    std::unique_ptr<WatermarkStream> s(new WatermarkStream());
    s->v = v; s->wm = wm; s->rate = rate; s->blk = rate / 100;
    SB_CUDA(cudaSetDevice(v->device));
    const size_t hold = ((size_t)s->blk * 4 + 255) & ~(size_t)255;
    SB_CUDA(cudaMalloc(&s->mem, 2 * hold + 2 * 256));
    char* base = static_cast<char*>(s->mem);
    s->hold[0] = reinterpret_cast<float*>(base); s->hold[1] = reinterpret_cast<float*>(base + hold);
    s->s[0] = reinterpret_cast<long long*>(base + 2 * hold); s->s[1] = reinterpret_cast<long long*>(base + 2 * hold + 256);
    return s.release();
}

void watermark_detect(unsigned long long key, int fmt, const void* d_x, const size_t* offs, size_t batch,
                      WatermarkScore* out, cudaStream_t st, long long* F_out) {
    if (fmt != 0 && fmt != 1)
        throw Error(19, "watermark detect: format " + std::to_string(fmt) + " is not 0 (f32) or 1 (i16)");
    if (batch == 0) return;
    std::vector<FoldTile> tiles;
    for (size_t b = 0; b < batch; b++)
        for (long long o = (long long)offs[b]; o < (long long)offs[b + 1]; o += (long long)WM_FOLD * WM_P)
            tiles.push_back(FoldTile{o, std::min<long long>((long long)offs[b + 1] - o, (long long)WM_FOLD * WM_P),
                                     (int)b});
    // the folds, the chip spectra, the tiles and the scores, in one allocation
    const size_t f_bytes = batch * WM_P * 8, c_bytes = 2 * WM_P * 16, t_bytes = tiles.size() * sizeof(FoldTile),
                 s_bytes = batch * sizeof(WatermarkScore);
    WmScratch m;
    SB_CUDA(cudaMalloc(&m.p, f_bytes + c_bytes + t_bytes + s_bytes + 64));
    char* base = static_cast<char*>(m.p);
    long long* F = reinterpret_cast<long long*>(base);
    double2* C = reinterpret_cast<double2*>(base + f_bytes);
    FoldTile* T = reinterpret_cast<FoldTile*>(base + f_bytes + c_bytes);
    WatermarkScore* S = reinterpret_cast<WatermarkScore*>(base + ((f_bytes + c_bytes + t_bytes + 15) & ~(size_t)15));
    SB_CUDA(cudaMemsetAsync(F, 0, f_bytes, st));
    if (!tiles.empty()) {
        SB_CUDA(cudaMemcpyAsync(T, tiles.data(), t_bytes, cudaMemcpyHostToDevice, st));
        if (fmt == 0)
            launch_pdl(wm_fold_kernel<float>, dim3((unsigned)tiles.size()), dim3(WM_FOLD_THREADS), 0, st,
                       static_cast<const float*>(d_x), (const FoldTile*)T, reinterpret_cast<unsigned long long*>(F));
        else
            launch_pdl(wm_fold_kernel<short>, dim3((unsigned)tiles.size()), dim3(WM_FOLD_THREADS), 0, st,
                       static_cast<const short*>(d_x), (const FoldTile*)T, reinterpret_cast<unsigned long long*>(F));
        g_launch_count++;
    }
    static PerDeviceOnce attr;
    attr.run([] {
        SB_CUDA(cudaFuncSetAttribute(wm_spectra_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(WmSmem)));
        SB_CUDA(cudaFuncSetAttribute(wm_detect_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(WmSmem)));
    });
    launch_pdl(wm_spectra_kernel, dim3(2), dim3(WM_FFT_THREADS), sizeof(WmSmem), st, key, C);
    launch_pdl(wm_detect_kernel, dim3((unsigned)batch), dim3(WM_FFT_THREADS), sizeof(WmSmem), st, (const long long*)F,
               (const double2*)C, S);
    g_launch_count += 2;
    SB_CUDA(cudaMemcpyAsync(out, S, s_bytes, cudaMemcpyDeviceToHost, st));
    if (F_out) SB_CUDA(cudaMemcpyAsync(F_out, F, f_bytes, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    SB_CUDA(cudaGetLastError());
}

}  // namespace sb200
