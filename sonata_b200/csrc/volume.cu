// Volume contours: a level in dB per id, applied on the device as a gain curve over the delivered samples at the
// voice's rate (DESIGN.md section 4, "Volume contours").  The host merges the ids into pieces of one gain each; the
// device gives every sample the gain of its piece, with a smoothstep ramp of about 10 ms centred on each boundary.  The
// curve uses only +, -, x and / in double, each rounded, so the kernel and the float64 specification agree bit for bit.
#include "engine.h"
#include <algorithm>
#include <cmath>

namespace sb200 {

namespace {
bool volume_asked(float v) { return !std::isnan(v) && v != 0.f; }
}  // namespace

bool check_volume_contour(const float* packed, const size_t* offs, size_t B, bool per_utterance) {
    if (!packed) return false;
    bool any = false;
    for (size_t b = 0; b < B; b++)
        for (size_t i = offs[b]; i < offs[b + 1]; i++) {
            const float v = packed[i];
            if (!volume_asked(v)) continue;
            if (!(v == -INFINITY || (std::isfinite(v) && v >= -60.f && v <= 20.f)))
                throw Error(19, (per_utterance ? "utterance " + std::to_string(b) + ", " : std::string()) + "id " +
                                    std::to_string(i - offs[b]) + ": volume level " + std::to_string(v) +
                                    " dB is not a finite value in [-60, 20] or -inf (NaN or 0: none)");
            any = true;
        }
    return any;
}

float volume_gain_of(float level) {
    if (std::isnan(level)) return 1.f;
    return level == -INFINITY ? 0.f : (float)std::pow(10.0, (double)level / 20.0);
}

std::vector<VolumePiece> volume_pieces(const long long* ends, const float* levels, size_t n_ids, long long n2) {
    std::vector<VolumePiece> pc;
    float level = 0.f;
    long long prev = 0;
    for (size_t i = 0; i < n_ids; i++) {
        if (ends[i] < prev || ends[i] > n2)
            throw Error(19, "volume contour: id " + std::to_string(i) + " ends at " + std::to_string(ends[i]) +
                                ", before the id ahead of it or past the signal's " + std::to_string(n2) + " samples");
        const float v = std::isnan(levels[i]) ? 0.f : levels[i];
        if (ends[i] > prev && (pc.empty() || v != level)) {
            pc.push_back(VolumePiece{prev, volume_gain_of(v)});
            level = v;
        }
        prev = ends[i];
    }
    if (n_ids && prev != n2)
        throw Error(19, "volume contour: the last id ends at " + std::to_string(prev) + ", not at " + std::to_string(n2));
    if (std::all_of(pc.begin(), pc.end(), [](const VolumePiece& p) { return p.g == 1.f; })) pc.clear();
    return pc;
}

void VolumePlan::add(long long at_, long long n, long long j0, int half, const std::vector<VolumePiece>& pc,
                     const VolumePiece* pc_d) {
    VolumeSeg g{};
    g.n = n; g.j0 = j0; g.half = half; g.m = (int)pc.size(); g.chunk = -1;
    g.pc = pc_d;
    if (!pc_d) {
        p_off.push_back((long long)pieces.size());
        pieces.insert(pieces.end(), pc.begin(), pc.end());
    } else {
        p_off.push_back(-1);
    }
    at.push_back(at_);
    max_n = std::max(max_n, n);
    bytes += 8.0 * (double)n + (double)sizeof(VolumePiece) * (double)pc.size();
    segs.push_back(g);
}

// ------------------------------------------------------------------ the kernel
constexpr int VM_THREADS = 256;

// G_j: the gain of the piece before the first boundary whose ramp covers j (the piece of j when none does), plus each
// covering boundary's step times its smoothstep, in ascending order, rounded to f32 once.
__device__ __forceinline__ float volume_gain(const VolumePiece* __restrict__ pc, int m, int half, long long j) {
    int lo = 1, hi = m;                 // the first boundary r >= 1 with B_r > j - half (ramp: B_r - half <= j < B_r + half)
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(&pc[mid].B) > j - half) hi = mid; else lo = mid + 1;
    }
    const float ga = __ldg(&pc[lo - 1].g);
    if (lo == m || __ldg(&pc[lo].B) > j + half) return ga;
    const double L = (double)(2 * half);
    double acc = (double)ga;
    float prev = ga;
    for (int r = lo; r < m; r++) {
        const long long B = __ldg(&pc[r].B);
        if (B > j + half) break;
        const float g = __ldg(&pc[r].g);
        const double t = __ddiv_rn(__dadd_rn((double)(j - B + half), 0.5), L);
        const double s = __dmul_rn(__dmul_rn(t, t), __dsub_rn(3.0, __dmul_rn(2.0, t)));
        acc = __dadd_rn(acc, __dmul_rn(__dsub_rn((double)g, (double)prev), s));
        prev = g;
    }
    return __double2float_rn(acc);
}

__global__ void __launch_bounds__(VM_THREADS)
volume_kernel(const VolumeSeg* __restrict__ segs, const float* __restrict__ src, const FrameSeg* __restrict__ fsegs,
              const PcmPost* __restrict__ posts, int hop) {
    pdl_trigger(); pdl_wait();
    const VolumeSeg g = segs[blockIdx.y];
    PcmSeg ps{};
    if (!g.x) ps = pcm_seg(src, fsegs[g.chunk], posts + g.chunk, hop);
    for (long long i = (long long)blockIdx.x * VM_THREADS + threadIdx.x; i < g.n; i += (long long)gridDim.x * VM_THREADS) {
        const float x = g.x ? g.x[i] : pcm_value(ps, i);
        g.y[i] = __fmul_rn(x, volume_gain(g.pc, g.m, g.half, g.j0 + i));
    }
}

void launch_volume(const VolumeSeg* segs, int nseg, long long max_n, const float* src, const FrameSeg* fsegs,
                   const PcmPost* posts, int hop, cudaStream_t st) {
    if (nseg <= 0 || max_n <= 0) return;
    const long long bx = std::min<long long>((max_n + VM_THREADS - 1) / VM_THREADS, 2048);
    launch_pdl(volume_kernel, dim3((unsigned)bx, nseg), dim3(VM_THREADS), 0, st, segs, src, fsegs, posts, hop);
    g_launch_count++;
}

}  // namespace sb200
