// Host side of output-rate conversion: the anti-aliasing filter of scipy.signal.resample_poly's default (designed in
// double, rounded to f32), the reduced up / down ratio of a rate pair, and each voice's cache of phase-major tap tables
// on its device.  The kernel is resample_kernel (kernels_misc.cu).
#include "engine.h"
#include <cmath>
#include <numeric>

namespace sb200 {

namespace {
constexpr long long kRates[] = {8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000};
constexpr int kMaxFactor = 640;       // largest max(up, down) of a supported rate pair for 16 kHz and 22.05 kHz voices

// Modified Bessel function of the first kind, order 0: sum_k ((x/2)^k / k!)^2, to double precision for |x| <= 5.
double bessel_i0(double x) {
    const double q = 0.25 * x * x;
    double s = 1.0, t = 1.0;
    for (int k = 1; k < 200; k++) {
        t *= q / ((double)k * (double)k);
        s += t;
        if (t < s * 1e-18) break;
    }
    return s;
}
}  // namespace

bool output_rate_supported(long long rate) {
    for (long long r : kRates)
        if (r == rate) return true;
    return false;
}

ResampleFilter resample_ratio(int in_rate, long long out_rate, const std::string& who) {
    if (!output_rate_supported(out_rate))
        throw Error(19, who + "output rate " + std::to_string(out_rate) +
                            " Hz is not supported (8000, 11025, 16000, 22050, 24000, 32000, 44100 or 48000, or 0 for the "
                            "voice's rate)");
    if (in_rate <= 0 || in_rate == out_rate) throw Error(19, who + "no resampling ratio for equal rates");
    const long long g = std::gcd((long long)in_rate, out_rate);
    const long long up = out_rate / g, down = in_rate / g;
    if (std::max(up, down) > kMaxFactor)
        throw Error(19, who + "resampling " + std::to_string(in_rate) + " Hz to " + std::to_string(out_rate) +
                            " Hz needs a ratio of " + std::to_string(up) + "/" + std::to_string(down) +
                            ", beyond the supported " + std::to_string(kMaxFactor));
    ResampleFilter f;
    f.up = (int)up; f.down = (int)down;
    f.H = 10 * (int)std::max(up, down);
    f.K = (2 * f.H + 1 + f.up - 1) / f.up;
    return f;
}

// scipy.signal.resample_poly: h = firwin(2H + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up.  firwin's lowpass is
// cutoff * sinc(cutoff * m), m = n - H, times the symmetric Kaiser window, scaled to unit sum at DC.
std::vector<float> resample_taps(int up, int down) {
    const int m = std::max(up, down), H = 10 * m, L = 2 * H + 1;
    const double fc = 1.0 / m, beta = 5.0, i0b = bessel_i0(beta), pi = 3.14159265358979323846;
    std::vector<double> h(L);
    double sum = 0.0;
    for (int n = 0; n < L; n++) {
        const double x = fc * (double)(n - H);
        const double sinc = x == 0.0 ? 1.0 : std::sin(pi * x) / (pi * x);
        const double r = (double)(n - H) / (double)H;
        const double w = bessel_i0(beta * std::sqrt(std::max(0.0, 1.0 - r * r))) / i0b;
        h[n] = fc * sinc * w;
        sum += h[n];
    }
    std::vector<float> out(L);
    for (int n = 0; n < L; n++) out[n] = (float)(h[n] / sum * (double)up);
    return out;
}

std::vector<float> resample_phase_major(const std::vector<float>& h, int up, int K) {
    std::vector<float> t((size_t)up * K, 0.f);
    for (int p = 0; p < up; p++)
        for (int k = 0; k < K && p + (size_t)k * up < h.size(); k++) t[(size_t)p * K + k] = h[p + (size_t)k * up];
    return t;
}

const ResampleFilter& voice_resampler(Voice& v, long long out_rate, const std::string& who) {
    std::lock_guard<std::mutex> g(v.rs_mu);
    auto it = v.rs_filters.find(out_rate);
    if (it != v.rs_filters.end()) return it->second;
    ResampleFilter f = resample_ratio(v.sample_rate, out_rate, who);
    const std::vector<float> t = resample_phase_major(resample_taps(f.up, f.down), f.up, f.K);
    SB_CUDA(cudaSetDevice(v.device));
    void* d = nullptr;
    SB_CUDA(cudaMalloc(&d, t.size() * sizeof(float)));
    v.dev_allocs.push_back(d);
    SB_CUDA(cudaMemcpy(d, t.data(), t.size() * sizeof(float), cudaMemcpyHostToDevice));
    f.taps = static_cast<float*>(d);
    return v.rs_filters.emplace(out_rate, f).first->second;
}

long long resample_emit_end(const ResampleFilter& f, long long n, bool ended) {
    if (ended) return (n * f.up + f.down - 1) / f.down;
    const long long room = n * f.up - f.H;       // output j has all its inputs once j * down + H < n * up
    return room <= 0 ? 0 : (room + f.down - 1) / f.down;
}

Resampler* create_resampler(Voice* v, long long out_rate) {
    if (v->device < 0 || !v->emb)
        throw Error(19, "Failed to run model inference. Error: voice was loaded config-only (device -1); libsonata_b200 has no CPU path");
    std::unique_ptr<Resampler> r(new Resampler());
    r->v = v;
    r->f = voice_resampler(*v, out_rate, "");
    SB_CUDA(cudaSetDevice(v->device));
    for (float*& p : r->hist) SB_CUDA(cudaMalloc(&p, sizeof(float) * (size_t)r->f.K));
    return r.release();
}

Resampler::~Resampler() {
    if (!v) return;
    cudaSetDevice(v->device);
    for (float* p : hist) if (p) cudaFree(p);
}

}  // namespace sb200
