// Formant ratio: the spectral envelope of what the pitch stage hands out, moved to the voice's own envelope times phi
// (DESIGN.md section 4, "Formants").  Frames of N = 1024 at a hop of 256 with a periodic Hann window; each frame's
// envelope is its real cepstrum liftered below about 4 ms of the unshifted voice, and the frame is rescaled bin by bin
// by the envelope read at k p / phi over the envelope at k, then overlap-added with the same window.  The FFTs are
// radix-2 in double in shared memory, so the result is a rounding of the float64 specification
// (include/sonata_b200.h, sb200_speak_batch_ids_formants); a sample's value depends on its utterance alone.
#include "engine.h"
#include <algorithm>
#include <climits>
#include <cmath>

namespace sb200 {

// ------------------------------------------------------------------ host: checks and the plan
bool check_formants(const float* phi, size_t B) {
    if (!phi) return false;
    bool any = false;
    for (size_t b = 0; b < B; b++) {
        if (std::isnan(phi[b])) continue;
        if (!(std::isfinite(phi[b]) && phi[b] >= 0.5f && phi[b] <= 2.f))
            throw Error(19, "utterance " + std::to_string(b) + ": formant ratio " + std::to_string(phi[b]) +
                                " is not a finite value in [0.5, 2] (NaN: none)");
        any = true;
    }
    return any;
}

namespace {
// p_m of the frame centred at c: the pitch ratio p, or with a contour the p of the last piece with Q <= c
double frame_pitch(double p, const ContourPiece* pc, int c_n, long long c) {
    if (c_n == 0) return p;
    int r = 0;
    for (int top = c_n - 1; r < top;) {
        const int mid = (r + top + 1) / 2;
        if (pc[mid].Q <= (double)c) r = mid; else top = mid - 1;
    }
    return pc[r].p;
}
long long frame_centre(long long m, long long n) { return std::min(std::max(m * FM_H + FM_N / 2, 0ll), n - 1); }
}  // namespace

bool formant_asks(long long n, float phi, double p, const ContourPiece* pc, int c_n) {
    if (std::isnan(phi) || n <= 0) return false;
    if (c_n == 0) return p / (double)phi != 1.0;
    for (long long m = -3, M = (n + FM_H - 1) / FM_H; m < M; m++)
        if (frame_pitch(p, pc, c_n, frame_centre(m, n)) / (double)phi != 1.0) return true;
    return false;
}

void FormantPlan::add(int rate, long long off, long long n, float phi, double p, int c_off, int c_n) {
    FormantSeg g{};
    g.off = off; g.n = n;
    g.p = p; g.phi = (double)phi; g.Q0 = rate / 250; g.c_off = c_off; g.c_n = c_n;
    const long long hops = (n + FM_H - 1) / FM_H, runs = (hops + FM_HOPS - 1) / FM_HOPS;
    g.h1 = hops; g.y_off = off;
    max_runs = std::max(max_runs, runs);
    // every CTA analyses its hops and the 3 frames before them: 4 FFTs of N points and about 40 operations per bin
    const double frames = (double)hops + 3.0 * (double)runs;
    flops += frames * (4.0 * 5.0 * FM_N * 10.0 + 40.0 * FM_N);
    bytes += 4.0 * ((double)n + 3.0 * FM_H * (double)runs + (FM_N - FM_H) * (double)runs) + 4.0 * (double)n;
    segs.push_back(g);
}

void FormantPlan::copy(long long off, long long n) {
    if (!copies.empty() && copies.back().first + copies.back().second == off) copies.back().second += n;
    else copies.emplace_back(off, n);
    bytes += 8.0 * (double)n;
}

// ------------------------------------------------------------------ host: streams
// Hop h needs frames h - 3 .. h, so inputs up to (h + 4) H: before its last chunk a stream emits the hops whose 4 frames
// lie inside its G inputs, and those frames neither reach the clamp at n2 - 1 nor read past G, so they are the whole
// signal's.  The last chunk emits the rest up to n2 = G.  The next pass recomputes the 3 frames before its first hop,
// so it carries the inputs from (h1 - 3) H on.
FormantStep formant_stream_step(const ProsodyStream& ps, long long g1, bool last) {
    FormantStep t{};
    t.g1 = g1; t.e0 = ps.fm_out; t.h0 = ps.fm_out / FM_H;
    if (last) {
        t.h1 = (g1 + FM_H - 1) / FM_H; t.e1 = g1; t.from = g1;
    } else {
        t.h1 = std::max(0ll, g1 / FM_H - (FM_N / FM_H - 1)); t.e1 = t.h1 * FM_H;
        t.from = std::max(0ll, (t.h1 - 3) * FM_H);
    }
    if (g1 < ps.fm_in || t.h1 < t.h0 || t.e1 < t.e0 || ps.fm_out % FM_H != 0)
        throw Error(19, "internal: a formant stream would go back");
    if (g1 - t.from > FM_CARRY || ps.fm_in - ps.fm_h > std::max(0ll, (t.h0 - 3) * FM_H))
        throw Error(19, "internal: a formant stream's carry exceeds its buffers");
    return t;
}

void FormantPlan::add_stream(const ProsodyStream& ps, const FormantStep& t) {
    FormantSeg g{};
    const long long nx = ps.fm_h + (t.g1 - ps.fm_in);
    g.off = in_total; in_total += nx; max_in = std::max(max_in, nx);
    g.n = t.g1; g.x0 = ps.fm_in - ps.fm_h; g.h0 = t.h0; g.h1 = t.h1;
    g.y_off = total; total += t.e1 - t.e0;
    g.p = ps.sh.p; g.phi = (double)ps.formant; g.Q0 = ps.rate / 250;
    if (!ps.pieces.empty()) { g.c_n = (int)ps.pieces.size() - 1; g.cp = ps.pieces_d; }
    const long long hops = t.h1 - t.h0, runs = (hops + FM_STREAM_HOPS - 1) / FM_STREAM_HOPS;
    max_runs = std::max(max_runs, runs);
    const double frames = (double)hops + 3.0 * (double)runs;
    flops += frames * (4.0 * 5.0 * FM_N * 10.0 + 40.0 * FM_N);
    bytes += 4.0 * (2.0 * (double)nx + (double)(t.g1 - t.from)) + 4.0 * (frames * FM_H + 3.0 * FM_H * (double)runs) +
             4.0 * (double)(t.e1 - t.e0);
    segs.push_back(g);
}

FormantCarry formant_carry(const ProsodyStream& ps, const FormantStep& t, int chunk, const float* direct) {
    FormantCarry c{};
    c.chunk = chunk; c.h = ps.fm_h; c.n_new = t.g1 - ps.fm_in;
    c.from = t.from - (ps.fm_in - ps.fm_h); c.keep = (int)(t.g1 - t.from);
    c.direct = direct;
    c.hist = ps.fm_hist[ps.cur]; c.next = ps.fm_hist[1 - ps.cur];
    return c;
}

void formant_stream_advance(ProsodyStream& ps, const FormantStep& t) {
    ps.fm_in = t.g1; ps.fm_out = t.e1; ps.fm_h = (int)(t.g1 - t.from);
}

// ------------------------------------------------------------------ the kernel
// Block (run, segment): 512 threads own hops [run * FM_HOPS, +FM_HOPS) of the segment's output and walk frames
// m = h0 - 3 .. h1 - 1 in order.  The overlap-add keeps the last 4 hops in a ring of doubles: after frame m, samples
// [m H, m H + H) have all 4 of their frames and leave, rounded once.
constexpr int FM_THREADS = 512;
struct FmSmem {
    double2 a[FM_N];          // the frame's spectrum, then the rescaled spectrum and its inverse
    double2 b[FM_N];          // the log magnitude, the cepstrum and the envelope
    double2 tw[FM_N / 2];     // e^{-2 pi i k / N}
    double ring[FM_N];        // the overlap-add of samples [m H, m H + N), indexed by sample mod N
    double red[FM_THREADS / 32];
};

__device__ __forceinline__ int fm_rev(int i) { return (int)(__brev((unsigned)i) >> 22); }     // 10-bit reversal
__device__ __forceinline__ double fm_window(const double2* tw, int i) {
    // 0.5 - 0.5 cos(2 pi i / N), with cos(2 pi (i + N/2) / N) = -cos(2 pi i / N)
    return i < FM_N / 2 ? 0.5 - 0.5 * tw[i].x : 0.5 + 0.5 * tw[i - FM_N / 2].x;
}

// In-place radix-2 FFT of x (bit-reversed in, natural order out), e^{-2 pi i / N} forward and the conjugate inverse,
// unscaled; one butterfly per thread per stage.  Ends synchronised.
__device__ void fm_fft(double2* x, const double2* tw, bool inverse) {
    const int t = threadIdx.x;
#pragma unroll 1
    for (int s = 1; s <= 10; s++) {
        const int half = 1 << (s - 1);
        const int pos = t & (half - 1);
        const int i0 = ((t >> (s - 1)) << s) + pos, i1 = i0 + half;
        double2 w = tw[pos << (10 - s)];
        if (inverse) w.y = -w.y;
        const double2 u = x[i0], v = x[i1];
        const double vr = v.x * w.x - v.y * w.y, vi = v.x * w.y + v.y * w.x;
        x[i0] = make_double2(u.x + vr, u.y + vi);
        x[i1] = make_double2(u.x - vr, u.y - vi);
        __syncthreads();
    }
}

__global__ void __launch_bounds__(FM_THREADS)
formant_kernel(const float* __restrict__ in, const FormantSeg* __restrict__ segs, const ContourPiece* __restrict__ pieces,
               float* __restrict__ out, int run) {
    extern __shared__ __align__(16) unsigned char fm_raw[];
    FmSmem& sm = *reinterpret_cast<FmSmem*>(fm_raw);
    const int t = threadIdx.x;
    {
        double s, c;
        sincospi((double)t / (FM_N / 2), &s, &c);
        sm.tw[t] = make_double2(c, -s);
        sm.ring[t] = 0.0; sm.ring[t + FM_THREADS] = 0.0;
    }
    pdl_trigger(); pdl_wait();
    const FormantSeg g = segs[blockIdx.y];
    const long long n = g.n;
    const long long h0 = g.h0 + (long long)blockIdx.x * run;
    if (h0 >= g.h1) return;
    const long long h1 = min(h0 + run, g.h1);
    const long long j_lo = h0 * FM_H, j_hi = min(h1 * FM_H, n);
    const float* y = in + g.off - g.x0;              // y[j]: sample j, for j >= x0
    float* o = out + g.y_off - g.h0 * FM_H;          // o[j]: where sample j leaves
    const ContourPiece* pc = g.c_n ? (g.cp ? g.cp : pieces + g.c_off) : nullptr;
    const double clamp = 1.2 * 2.30258509299404568402;      // 24 dB as a natural-log amplitude
    __syncthreads();
    for (long long m = h0 - 3; m < h1; m++) {
        // the frame's ratios: p_m at its clamped centre, r_m = p_m / phi and the lifter's cutoff Q_m
        const long long cm = min(max(m * FM_H + FM_N / 2, 0ll), n - 1);
        double pm = g.p;
        if (pc) {
            int r = 0;
            for (int top = g.c_n - 1; r < top;) {
                const int mid = (r + top + 1) / 2;
                if (pc[mid].Q <= (double)cm) r = mid; else top = mid - 1;
            }
            pm = pc[r].p;
        }
        const double rm = pm / g.phi;
        const int Qm = (int)floor((double)g.Q0 / pm + 0.5);
        // X = FFT(w frame)
        for (int i = t; i < FM_N; i += FM_THREADS) {
            const long long j = m * FM_H + i;
            const double v = j >= 0 && j < n ? (double)y[j] : 0.0;
            sm.a[fm_rev(i)] = make_double2(v * fm_window(sm.tw, i), 0.0);
        }
        __syncthreads();
        fm_fft(sm.a, sm.tw, false);
        // P = |X|^2 over bins 0 .. N/2, its mean in a fixed order, and Lambda = log(P + eps) / 2 as an even sequence
        const double2 x0 = sm.a[t];
        const double P0 = x0.x * x0.x + x0.y * x0.y;
        const double P1 = t == 0 ? sm.a[FM_N / 2].x * sm.a[FM_N / 2].x + sm.a[FM_N / 2].y * sm.a[FM_N / 2].y : 0.0;
        double sum = P0 + P1;
        for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, d);
        if ((t & 31) == 0) sm.red[t >> 5] = sum;
        __syncthreads();
        double tot = 0.0;
        for (int w = 0; w < FM_THREADS / 32; w++) tot += sm.red[w];
        const double eps = 1e-10 * (tot / (double)(FM_N / 2 + 1)) + 1e-30;
        const double L0 = 0.5 * log(P0 + eps);
        sm.b[fm_rev(t)] = make_double2(L0, 0.0);
        if (t > 0) sm.b[fm_rev(FM_N - t)] = make_double2(L0, 0.0);
        else sm.b[fm_rev(FM_N / 2)] = make_double2(0.5 * log(P1 + eps), 0.0);
        __syncthreads();
        fm_fft(sm.b, sm.tw, true);
        // the cepstrum c = IFFT(Lambda) / N, liftered, and E = Re FFT(c l)
        double cl[2];
        for (int h = 0; h < 2; h++) {
            const int q = t + h * FM_THREADS, qq = min(q, FM_N - q);
            const double l = qq == 0 ? 1.0 : qq < Qm ? 0.5 * (1.0 + cospi((double)qq / (double)Qm)) : 0.0;
            cl[h] = sm.b[q].x * (1.0 / FM_N) * l;
        }
        __syncthreads();
        sm.b[fm_rev(t)] = make_double2(cl[0], 0.0);
        sm.b[fm_rev(t + FM_THREADS)] = make_double2(cl[1], 0.0);
        __syncthreads();
        fm_fft(sm.b, sm.tw, false);
        // g_k = clamp(E(k r_m) - E(k)) and Z = X e^g as a Hermitian spectrum
        double2 z[2];
        for (int h = 0; h < 2; h++) {
            const int k = h == 0 ? t : FM_N / 2;
            if (h == 1 && t != 0) break;
            const double u = (double)k * rm;
            double e;
            if (u >= (double)(FM_N / 2)) {
                e = sm.b[FM_N / 2].x;
            } else {
                const int i = (int)floor(u);
                const double f = u - (double)i, e0 = sm.b[i].x;
                e = e0 + f * (sm.b[i + 1].x - e0);
            }
            const double gk = fmin(fmax(e - sm.b[k].x, -clamp), clamp);
            const double s = exp(gk);
            const double2 xk = sm.a[k];
            z[h] = make_double2(xk.x * s, xk.y * s);
        }
        __syncthreads();
        if (t == 0) {
            sm.a[fm_rev(0)] = make_double2(z[0].x, 0.0);
            sm.a[fm_rev(FM_N / 2)] = make_double2(z[1].x, 0.0);
        } else {
            sm.a[fm_rev(t)] = z[0];
            sm.a[fm_rev(FM_N - t)] = make_double2(z[0].x, -z[0].y);
        }
        __syncthreads();
        fm_fft(sm.a, sm.tw, true);
        // overlap-add w z / N in ascending m, then the hop this frame completes leaves
        for (int i = t; i < FM_N; i += FM_THREADS) {
            const long long j = m * FM_H + i;
            if (j >= j_lo && j < j_hi) sm.ring[j & (FM_N - 1)] += fm_window(sm.tw, i) * (sm.a[i].x * (1.0 / FM_N));
        }
        __syncthreads();
        if (m >= h0 && t < FM_H) {
            const long long j = m * FM_H + t;
            if (j < j_hi) {
                o[j] = (float)(sm.ring[j & (FM_N - 1)] / 1.5);
                sm.ring[j & (FM_N - 1)] = 0.0;
            }
        }
        __syncthreads();
    }
}

void launch_formant(const float* in, const FormantSeg* segs, int nseg, long long max_runs, const ContourPiece* pieces,
                    float* out, cudaStream_t st, int run) {
    if (nseg <= 0 || max_runs <= 0) return;
    if (max_runs > INT_MAX) throw_launch_error("formant: an utterance too long for the grid");
    static PerDeviceOnce once;
    once.run([] {
        cudaFuncSetAttribute(formant_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FmSmem));
    });
    launch_pdl(formant_kernel, dim3((unsigned)max_runs, nseg), dim3(FM_THREADS), sizeof(FmSmem), st, in, segs, pieces,
               out, run);
    g_launch_count++;
}

// ------------------------------------------------------------------ a stream's chunk pass: staging and carry
// Writes each segment's window (the carried samples, then the new ones) and, from the same values, the samples the
// stream's next pass carries into its other buffer.
__global__ void formant_stage_kernel(const float* __restrict__ src, const FrameSeg* __restrict__ fsegs,
                                     const PcmPost* __restrict__ posts, int hop, const FormantSeg* __restrict__ segs,
                                     const FormantCarry* __restrict__ cs, float* __restrict__ win) {
    pdl_trigger(); pdl_wait();
    const FormantCarry c = cs[blockIdx.y];
    float* w = win + segs[blockIdx.y].off;
    const PcmSeg x = c.direct ? PcmSeg{} : pcm_seg(src, fsegs[c.chunk], posts + c.chunk, hop);
    const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, step = (long long)gridDim.x * blockDim.x;
    for (long long i = i0; i < c.h + c.n_new; i += step) {
        const float v = i < c.h ? c.hist[i] : c.direct ? c.direct[i - c.h] : pcm_value(x, i - c.h);
        w[i] = v;
        if (i >= c.from) c.next[i - c.from] = v;
    }
}

void launch_formant_stage(const float* src, const FrameSeg* fsegs, const PcmPost* posts, int hop, const FormantSeg* segs,
                          const FormantCarry* cs, int nseg, long long max_in, float* win, cudaStream_t st) {
    if (nseg <= 0) return;
    const unsigned grid = (unsigned)std::min<long long>(std::max<long long>((max_in + 1023) / 1024, 1), 4096);
    launch_pdl(formant_stage_kernel, dim3(grid, nseg), dim3(256), 0, st, src, fsegs, posts, hop, segs, cs, win);
    g_launch_count++;
}

void launch_formant_stream(const FormantPlan& p, const FormantSeg* segs, const FormantCarry* cs, const float* src,
                           const FrameSeg* fsegs, const PcmPost* posts, int hop, float* win, float* y, cudaStream_t st) {
    const int n = (int)p.segs.size();
    launch_formant_stage(src, fsegs, posts, hop, segs, cs, n, p.max_in, win, st);
    launch_formant(win, segs, n, p.max_runs, nullptr, y, st, FM_STREAM_HOPS);
}

}  // namespace sb200
