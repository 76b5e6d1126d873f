// Host side of loudness normalisation: the K-weighting filter of ITU-R BS.1770-4 designed for any rate the way
// libebur128 designs it (in double), the state recurrence of its two-biquad cascade raised to the gating step, and the
// check of per-utterance targets; and the live meters of streams.  The kernels are loudness_kernel and
// loudness_stream_kernel (kernels_misc.cu).
#include "engine.h"
#include <algorithm>
#include <cmath>
#include <memory>

namespace sb200 {

namespace {
// A 4x4 product c = a * b, row-major.
void mat4_mul(const double* a, const double* b, double* c) {
    for (int r = 0; r < 4; r++)
        for (int q = 0; q < 4; q++) {
            double s = 0.0;
            for (int t = 0; t < 4; t++) s += a[4 * r + t] * b[4 * t + q];
            c[4 * r + q] = s;
        }
}
}  // namespace

bool loudness_rate_supported(long long rate) { return rate >= 8000 && rate <= 384000; }

void loudness_design(long long rate, LoudSeg& s) {
    if (!loudness_rate_supported(rate))
        throw Error(19, "loudness: no K-weighting filter for a rate of " + std::to_string(rate) + " Hz (8000 .. 384000)");
    const double pi = 3.14159265358979323846, fs = (double)rate;
    // high shelf (BS.1770-4 Table 1 at 48 kHz)
    {
        const double f0 = 1681.974450955533, G = 3.999843853973347, Q = 0.7071752369554196;
        const double K = std::tan(pi * f0 / fs), Vh = std::pow(10.0, G / 20.0), Vb = std::pow(Vh, 0.4996667741545416);
        const double a0 = 1.0 + K / Q + K * K;
        s.k[0] = (Vh + Vb * K / Q + K * K) / a0;
        s.k[1] = 2.0 * (K * K - Vh) / a0;
        s.k[2] = (Vh - Vb * K / Q + K * K) / a0;
        s.k[3] = 2.0 * (K * K - 1.0) / a0;
        s.k[4] = (1.0 - K / Q + K * K) / a0;
    }
    // high-pass (Table 2)
    {
        const double f0 = 38.13547087602444, Q = 0.5003270373238773;
        const double K = std::tan(pi * f0 / fs), a0 = 1.0 + K / Q + K * K;
        s.k[5] = 1.0; s.k[6] = -2.0; s.k[7] = 1.0;
        s.k[8] = 2.0 * (K * K - 1.0) / a0;
        s.k[9] = (1.0 - K / Q + K * K) / a0;
    }
    s.S = (int)((rate + 5) / 10);
    // With zero input, the states {s1, s2, t1, t2} of the two transposed-direct-form-II biquads evolve as s' = A s:
    // y1 = s1, s1' = s2 - a1 y1, s2' = -a2 y1, y = b0 y1 + t1, t1' = b1 y1 + t2 - a1 y, t2' = b2 y1 - a2 y.
    const double* k = s.k;
    const double A[16] = {-k[3], 1.0, 0.0, 0.0,
                          -k[4], 0.0, 0.0, 0.0,
                          k[6] - k[8] * k[5], 0.0, -k[8], 1.0,
                          k[7] - k[9] * k[5], 0.0, -k[9], 0.0};
    // A^S by squaring
    double R[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}, P[16], T[16];
    std::copy(A, A + 16, P);
    for (long long e = s.S; e > 0; e >>= 1) {
        if (e & 1) { mat4_mul(R, P, T); std::copy(T, T + 16, R); }
        mat4_mul(P, P, T); std::copy(T, T + 16, P);
    }
    std::copy(R, R + 16, s.AS);
}

bool check_loudness_targets(const float* t, size_t B) {
    if (!t) return false;
    bool any = false;
    for (size_t b = 0; b < B; b++) {
        if (std::isnan(t[b])) continue;
        if (!(std::isfinite(t[b]) && t[b] >= -70.f && t[b] <= 0.f))
            throw Error(19, "utterance " + std::to_string(b) + ": loudness target " + std::to_string(t[b]) +
                                " LUFS is not a finite value in [-70, 0] (NaN: none)");
        any = true;
    }
    return any;
}

LoudnessStream* create_loudness_stream(Voice* v, int device, long long rate, float target, float max_gain_db) {
    if (!(std::isfinite(target) && target >= -70.f && target <= 0.f))
        throw Error(19, "live loudness target " + std::to_string(target) + " LUFS is not a finite value in [-70, 0]");
    if (!(std::isfinite(max_gain_db) && max_gain_db >= 0.f && max_gain_db <= 40.f))
        throw Error(19, "live loudness maximum gain " + std::to_string(max_gain_db) +
                            " dB is not a finite value in [0, 40]");
    std::unique_ptr<LoudnessStream> s(new LoudnessStream());
    loudness_design(rate, s->d);
    s->v = v; s->device = device; s->rate = rate;
    s->target = target; s->max_gain_db = max_gain_db;
    // two carries of 4 doubles and S floats each, then q
    const size_t carry = 4 + ((size_t)s->d.S + 1) / 2;
    SB_CUDA(cudaSetDevice(device));
    SB_CUDA(cudaMalloc(&s->mem, sizeof(double) * (2 * carry + (size_t)LS_MAX_STEPS)));
    double* base = static_cast<double*>(s->mem);
    SB_CUDA(cudaMemset(base, 0, sizeof(double) * 2 * carry));
    s->carry[0] = base; s->carry[1] = base + carry;
    s->q = base + 2 * carry;
    return s.release();
}

LoudnessStream::~LoudnessStream() {
    if (!mem) return;
    cudaSetDevice(device);
    cudaFree(mem);
}

long long loudness_stream_steps(const LoudnessStream& s, long long n, const std::string& who) {
    const long long steps = (s.samples + n) / s.d.S;
    if (steps > LS_MAX_STEPS)
        throw Error(19, who + "the loudness stream would pass its capacity of " + std::to_string(LS_MAX_STEPS) +
                            " steps of 100 ms (" + std::to_string(s.samples + n) + " samples at " +
                            std::to_string(s.rate) + " Hz)");
    return steps - s.steps;
}

LoudStreamSeg loudness_stream_seg(const LoudnessStream& s, float* y, long long n, float gain) {
    LoudStreamSeg g{};
    g.y = y; g.n = n;
    g.cin = s.carry[s.cur]; g.cout = s.carry[1 - s.cur];
    g.q = s.q;
    g.m0 = s.steps; g.p = (int)(s.samples - s.steps * s.d.S); g.S = s.d.S;
    g.a_prev = s.a_prev; g.a_cur = s.a;
    g.target = s.target; g.max_gain_db = s.max_gain_db; g.gain = gain;
    std::copy(s.d.k, s.d.k + 10, g.k);
    std::copy(s.d.AS, s.d.AS + 16, g.AS);
    return g;
}

void loudness_stream_advance(LoudnessStream& s, long long n, const double* lufs, const float* gains,
                             unsigned long long clipped) {
    const long long nc = (s.samples + n) / s.d.S - s.steps;
    if (nc >= 2) s.a_prev = gains[nc - 2];
    else if (nc == 1) s.a_prev = s.a;
    if (nc >= 1) { s.a = gains[nc - 1]; s.lufs = lufs[nc - 1]; }
    s.samples += n;
    s.steps += nc;
    s.clipped += (long long)clipped;
    s.cur ^= 1;
}

}  // namespace sb200
