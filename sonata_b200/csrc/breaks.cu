// Pauses: a break in milliseconds after any id, inserted on the device as zeros into the delivered samples at the
// voice's rate (DESIGN.md section 4, "Pauses").  The host turns the ids' breaks into a table of merged positions and
// running lengths; the device gives every output sample either a zero (inside a pause) or its input sample times the
// product of the smoothstep fades of the few pauses within about 5 ms of it.  The fades use only +, -, x and / in
// double, each rounded, so the kernel and the float64 specification agree bit for bit.
#include "engine.h"
#include <algorithm>
#include <climits>
#include <cmath>

namespace sb200 {

namespace {
bool break_asked(float v) { return !std::isnan(v) && v != 0.f; }
}  // namespace

bool check_breaks(const float* packed, const size_t* offs, size_t B, bool per_utterance) {
    if (!packed) return false;
    bool any = false;
    for (size_t b = 0; b < B; b++)
        for (size_t i = offs[b]; i < offs[b + 1]; i++) {
            const float v = packed[i];
            if (!break_asked(v)) continue;
            if (!(std::isfinite(v) && v > 0.f && v <= 10000.f))
                throw Error(19, (per_utterance ? "utterance " + std::to_string(b) + ", " : std::string()) + "id " +
                                    std::to_string(i - offs[b]) + ": break " + std::to_string(v) +
                                    " ms is not a finite value in (0, 10000] (NaN or 0: none)");
            any = true;
        }
    return any;
}

long long break_samples(float ms, int rate) {
    if (!break_asked(ms)) return 0;
    return (long long)std::floor((double)ms * (double)rate / 1000.0 + 0.5);
}

std::vector<BreakPiece> break_plan(const long long* ends, const float* ms, size_t n_ids, long long n2, int rate,
                                   const std::string& who) {
    std::vector<BreakPiece> bk;
    long long prev = 0, D = 0;
    for (size_t i = 0; i < n_ids; i++) {
        if (ends[i] < prev || ends[i] > n2)
            throw Error(19, who + "breaks: id " + std::to_string(i) + " ends at " + std::to_string(ends[i]) +
                                ", before the id ahead of it or past the signal's " + std::to_string(n2) + " samples");
        prev = ends[i];
        const long long N = break_samples(ms[i], rate);
        if (!N) continue;
        D += N;
        if (!bk.empty() && bk.back().P == ends[i]) bk.back().D = D;
        else bk.push_back(BreakPiece{ends[i], D});
    }
    if (n2 + D > (long long)INT_MAX)
        throw Error(19, who + "breaks: the delivered length " + std::to_string(n2) + " + " + std::to_string(D) +
                            " samples passes 2^31 - 1");
    return bk;
}

long long break_shift(const std::vector<BreakPiece>& bk, long long pos) {
    // the running length of the last break at or before pos
    const auto it = std::upper_bound(bk.begin(), bk.end(), pos, [](long long p, const BreakPiece& k) { return p < k.P; });
    return it == bk.begin() ? 0 : (it - 1)->D;
}

void BreakPlan::add(long long at_, long long n_in, long long j0, long long o0, long long n_out, int half,
                    const std::vector<BreakPiece>& bk, const BreakPiece* bk_d) {
    BreakSeg g{};
    g.n = n_out; g.o0 = o0; g.j0 = j0; g.half = half; g.m = (int)bk.size(); g.chunk = -1;
    g.bk = bk_d;
    if (!bk_d) {
        p_off.push_back((long long)pieces.size());
        pieces.insert(pieces.end(), bk.begin(), bk.end());
    } else {
        p_off.push_back(-1);
    }
    at.push_back(at_);
    y_off.push_back(total);
    total += n_out;
    max_n = std::max(max_n, n_out);
    bytes += 4.0 * (double)n_in + 4.0 * (double)n_out + (double)sizeof(BreakPiece) * (double)bk.size();
    segs.push_back(g);
}

// ------------------------------------------------------------------ the kernel
constexpr int BK_THREADS = 256;

// The smoothstep S(t) = t t (3 - 2 t), each operation rounded.
__device__ __forceinline__ double break_step(double t) {
    return __dmul_rn(__dmul_rn(t, t), __dsub_rn(3.0, __dmul_rn(2.0, t)));
}

// h_j: 1 times the fade of each break k with P_k - F <= j < P_k + F, in ascending k, rounded to f32 once.
__device__ __forceinline__ float break_fade(const BreakPiece* __restrict__ bk, int m, int F, long long j) {
    int lo = 0, hi = m;                 // the first break with P > j - F
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(&bk[mid].P) > j - F) hi = mid; else lo = mid + 1;
    }
    double h = 1.0;
    const double f = (double)F;
    for (int k = lo; k < m; k++) {
        const long long P = __ldg(&bk[k].P);
        if (P > j + F) break;
        const double t = j < P ? __ddiv_rn(__dsub_rn((double)(P - j), 0.5), f)
                               : __ddiv_rn(__dadd_rn((double)(j - P), 0.5), f);
        h = __dmul_rn(h, break_step(t));
    }
    return __double2float_rn(h);
}

__global__ void __launch_bounds__(BK_THREADS)
break_kernel(const BreakSeg* __restrict__ segs, const float* __restrict__ src, const FrameSeg* __restrict__ fsegs,
             const PcmPost* __restrict__ posts, int hop) {
    pdl_trigger(); pdl_wait();
    const BreakSeg g = segs[blockIdx.y];
    PcmSeg ps{};
    if (!g.x) ps = pcm_seg(src, fsegs[g.chunk], posts + g.chunk, hop);
    for (long long i = (long long)blockIdx.x * BK_THREADS + threadIdx.x; i < g.n; i += (long long)gridDim.x * BK_THREADS) {
        const long long q = g.o0 + i;
        // c: the breaks whose zeros all lie before output q (P_k + D_k <= q)
        int lo = 0, hi = g.m;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (__ldg(&g.bk[mid].P) + __ldg(&g.bk[mid].D) <= q) lo = mid + 1; else hi = mid;
        }
        const long long Dc = lo ? __ldg(&g.bk[lo - 1].D) : 0;
        if (lo < g.m && __ldg(&g.bk[lo].P) + Dc <= q) {
            g.y[i] = 0.f;
            continue;
        }
        const long long j = q - Dc;
        const float x = g.x ? g.x[j - g.j0] : pcm_value(ps, j - g.j0);
        g.y[i] = g.m ? __fmul_rn(x, break_fade(g.bk, g.m, g.half, j)) : x;
    }
}

void launch_breaks(const BreakSeg* segs, int nseg, long long max_n, const float* src, const FrameSeg* fsegs,
                   const PcmPost* posts, int hop, cudaStream_t st) {
    if (nseg <= 0 || max_n <= 0) return;
    const long long bx = std::min<long long>((max_n + BK_THREADS - 1) / BK_THREADS, 2048);
    launch_pdl(break_kernel, dim3((unsigned)bx, nseg), dim3(BK_THREADS), 0, st, segs, src, fsegs, posts, hop);
    g_launch_count++;
}

}  // namespace sb200
