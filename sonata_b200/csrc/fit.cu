// Target durations: fit an utterance, or spans of it, to a caller-chosen length in the same pass, between the duration
// predictor and the alignment (DESIGN.md section 4, "Target durations").  Each span's ids get one f32 factor u on their
// predicted durations, c_i(u) = ceil(w_i u), and u* is the largest f32 in [0.5, 2] whose frames fit the span's budget.
// Every c_i is nondecreasing in u, so the frames are too, and a bisection over the 2^24 + 1 bit patterns of [0.5, 2]
// finds u* in at most 25 integer warp sums.  Integer sums make u* independent of the order of the ids and of the batch.
#include "engine.h"
#include <cmath>

namespace sb200 {

namespace {

__device__ __forceinline__ long long warp_sum(long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// The span's frames at factor u: its predicted ids' ceil(w u) and its fixed counts.
__device__ __forceinline__ long long span_frames(const FitSpan& s, const float* w, const int* dur_frames, float u,
                                                 long long fixed, int lane) {
    long long t = 0;
    for (int i = lane; i < s.len; i += 32) {
        const int row = s.row0 + i;
        if (!dur_frames || dur_frames[row] < 0) t += dur_count(w[row] * u);
    }
    return warp_sum(t) + fixed;
}

// One warp per span, 8 spans per block.
__global__ void __launch_bounds__(256) fit_kernel(const FitSpan* __restrict__ spans, int nspans,
                                                  const float* __restrict__ z, float m0, float logs0,
                                                  const float* __restrict__ length_scales,
                                                  const float* __restrict__ dur_scale,
                                                  const int* __restrict__ dur_frames, float* w,
                                                  float* __restrict__ factor, float* __restrict__ u_out,
                                                  long long* __restrict__ frames_out) {
    pdl_trigger(); pdl_wait();
    const int k = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (k >= nspans) return;
    const FitSpan s = spans[k];
    long long fixed = 0;
    bool pred = false;
    const float einv = z ? expf(-logs0) : 0.f;
    const float length_scale = z ? length_scales[s.seg] : 0.f;
    for (int i = lane; i < s.len; i += 32) {
        const int row = s.row0 + i;
        const int f = dur_frames ? dur_frames[row] : -1;
        if (f >= 0) { fixed += f; continue; }
        pred = true;
        if (z) w[row] = dur_weight(dur_logw(z, row, m0, einv), length_scale, dur_scale, row);
    }
    fixed = warp_sum(fixed);
    pred = __any_sync(0xffffffffu, pred);
    __syncwarp();       // every lane's w writes are visible to the warp
    float u = 1.f;
    long long frames;
    if (!pred) {
        frames = fixed;
    } else {
        unsigned lo = __float_as_uint(0.5f), hi = __float_as_uint(2.0f);
        frames = span_frames(s, w, dur_frames, 0.5f, fixed, lane);
        if (frames <= s.budget) {       // lo fits; find the last bit pattern that does
            while (lo < hi) {
                const unsigned mid = lo + (hi - lo + 1) / 2;
                const long long t = span_frames(s, w, dur_frames, __uint_as_float(mid), fixed, lane);
                if (t <= s.budget) { lo = mid; frames = t; } else hi = mid - 1;
            }
        }
        u = __uint_as_float(lo);
        for (int i = lane; i < s.len; i += 32) factor[s.row0 + i] = u;
    }
    if (lane == 0) { u_out[k] = u; frames_out[k] = frames; }
}

bool asked(float ms) { return !std::isnan(ms); }

}  // namespace

void launch_fit(const FitSpan* spans, int nspans, const float* z, float m0, float logs0, const float* length_scales,
                const float* dur_scale, const int* dur_frames, float* w, float* factor, float* u_out,
                long long* frames_out, cudaStream_t st) {
    if (nspans <= 0) return;
    launch_pdl(fit_kernel, dim3((nspans + 7) / 8), dim3(256), 0, st, spans, nspans, z, m0, logs0, length_scales,
               dur_scale, dur_frames, w, factor, u_out, frames_out);
    g_launch_count++;
}

bool check_targets(const long long* first, const long long* end, const float* ms, const size_t* fit_offs,
                   const size_t* offs, size_t B, const float* tempo, bool per_utterance) {
    if (!fit_offs) return false;
    if (fit_offs[0] != 0) throw Error(19, "target durations: the span offsets do not start at 0");
    for (size_t b = 0; b < B; b++)
        if (fit_offs[b + 1] < fit_offs[b]) throw Error(19, "target durations: the span offsets decrease");
    if (fit_offs[B] && (!first || !end || !ms)) throw Error(19, "target durations: null span arrays");
    bool any = false;
    for (size_t b = 0; b < B; b++) {
        const std::string who = per_utterance ? "utterance " + std::to_string(b) + ", " : std::string();
        const long long n = (long long)(offs[b + 1] - offs[b]);
        long long prev = 0;
        bool here = false;
        for (size_t k = fit_offs[b]; k < fit_offs[b + 1]; k++) {
            const std::string span = who + "span " + std::to_string(k - fit_offs[b]) + ": ";
            if (!(first[k] >= 0 && first[k] < end[k] && end[k] <= n))
                throw Error(19, span + "ids [" + std::to_string(first[k]) + ", " + std::to_string(end[k]) +
                                    ") are not a non-empty range of the " + std::to_string(n) + " ids");
            if (first[k] < prev)
                throw Error(19, span + "ids [" + std::to_string(first[k]) + ", " + std::to_string(end[k]) +
                                    ") overlap or precede the span before it, which ends at id " +
                                    std::to_string(prev));
            prev = end[k];
            if (!asked(ms[k])) continue;
            if (!(std::isfinite(ms[k]) && ms[k] > 0.f && ms[k] <= 600000.f))
                throw Error(19, span + "target duration " + std::to_string(ms[k]) +
                                    " ms is not a finite value in (0, 600000] (NaN: none)");
            here = true;
        }
        if (here && tempo && !std::isnan(tempo[b]) && tempo[b] != 1.f)
            throw Error(19, (per_utterance ? "utterance " + std::to_string(b) : std::string("stream")) +
                                ": a target duration and a tempo ratio together (give one or the other)");
        any |= here;
    }
    return any;
}

long long target_samples(float ms, int rate) {
    return (long long)std::floor((double)ms * (double)rate / 1000.0 + 0.5);
}

FitPlan fit_plan(const Job& j) {
    FitPlan p;
    if (j.targets.empty()) return p;
    const int rate = j.v->sample_rate;
    const long long hop = j.v->a.hop();
    for (size_t b = 0; b < j.B; b++)
        for (size_t k = j.target_offs[b]; k < j.target_offs[b + 1]; k++) {
            const FitTarget& t = j.targets[k];
            if (!asked(t.ms)) continue;
            long long P = 0;
            if (!j.breaks.empty())
                for (long long i = t.first; i < t.end; i++) P += break_samples(j.breaks[j.offs[b] + i], rate);
            const long long room = target_samples(t.ms, rate) - P;
            const long long budget = room >= 0 ? room / hop : -((-room + hop - 1) / hop);
            p.spans.push_back(FitSpan{j.xsegs[b].off + (int)t.first, (int)(t.end - t.first), (int)b, budget});
            p.pause.push_back(P);
            p.index.push_back(k);
        }
    return p;
}

void set_job_targets(Job& j, const long long* first, const long long* end, const float* ms, const size_t* fit_offs) {
    if (!check_targets(first, end, ms, fit_offs, j.offs.data(), j.B, j.tempo.empty() ? nullptr : j.tempo.data())) {
        j.targets.clear(); j.target_offs.clear();
        return;
    }
    j.targets.resize(fit_offs[j.B]);
    for (size_t k = 0; k < fit_offs[j.B]; k++) j.targets[k] = FitTarget{first[k], end[k], ms[k]};
    j.target_offs.assign(fit_offs, fit_offs + j.B + 1);
}

}  // namespace sb200
