// extern "C" surface of libsonata_b200 (declared in include/sonata_b200.h).
// Error handling mirrors ffi_support::call_with_result used by libsonata (capi/src/lib.rs:187-336):
// no exception crosses the ABI; failures become {code, heap message}.
#include "../../include/sonata_b200.h"
#include "engine.h"
#include "tc_common.cuh"
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <deque>

using namespace sb200;

// Handles.  A job returns its context to the voice's pool when it dies and a latent belongs to a voice, so both share
// ownership of the voice: freeing the voice handle first (garbage-collected callers free in any order) is safe.
struct sb200_voice { std::shared_ptr<Voice> v; };
struct sb200_job {
    Job* j; std::shared_ptr<Voice> keep;
    ~sb200_job() { delete j; }
};
struct sb200_latent {
    Latent* l; std::shared_ptr<Voice> keep;
    ~sb200_latent() { delete l; }
};
struct sb200_prosody_stream {
    ProsodyStream* p; std::shared_ptr<Voice> keep;
    ~sb200_prosody_stream() { delete p; }
};
struct sb200_resampler {
    Resampler* r; std::shared_ptr<Voice> keep;
    ~sb200_resampler() { delete r; }
};
struct sb200_loudness_stream {
    LoudnessStream* s; std::shared_ptr<Voice> keep;
    ~sb200_loudness_stream() { delete s; }
};
struct sb200_watermark_stream {
    WatermarkStream* w; std::shared_ptr<Voice> keep;
    ~sb200_watermark_stream() { delete w; }
};

namespace {

// ---- pinned result blocks, shared by the sb200_audio entries of one batch and recycled ----
struct PinnedBlock { std::atomic<int> refs{0}; float* base = nullptr; size_t bytes = 0; };
std::mutex g_pin_mu;
std::deque<PinnedBlock*> g_pin_free;
std::unordered_map<const float*, PinnedBlock*> g_owner;   // audio.data -> block

// Smallest pooled block that fits (a larger one is fine: an exact-size policy made a caller that alternates between
// big and small batches pay cudaMallocHost + cudaFreeHost, ~1 ms, on every small call).
PinnedBlock* pin_acquire(size_t bytes) {
    {
        std::lock_guard<std::mutex> g(g_pin_mu);
        auto best = g_pin_free.end();
        for (auto it = g_pin_free.begin(); it != g_pin_free.end(); ++it)
            if ((*it)->bytes >= bytes && (best == g_pin_free.end() || (*it)->bytes < (*best)->bytes)) best = it;
        if (best != g_pin_free.end()) {
            PinnedBlock* b = *best;
            g_pin_free.erase(best);
            return b;
        }
    }
    PinnedBlock* b = new PinnedBlock();
    b->bytes = bytes + bytes / 8 + 4096;
    void* p = nullptr;
    if (cudaMallocHost(&p, b->bytes) != cudaSuccess) { delete b; throw Error(19, "cudaMallocHost failed for the result buffer"); }
    b->base = (float*)p;
    return b;
}
void pin_release(PinnedBlock* b) {
    PinnedBlock* victim = nullptr;
    {
        std::lock_guard<std::mutex> g(g_pin_mu);
        g_pin_free.push_back(b);
        if (g_pin_free.size() > 8) { victim = g_pin_free.front(); g_pin_free.pop_front(); }     // oldest goes
    }
    if (victim) { cudaFreeHost(victim->base); delete victim; }
}

char* dup_cstr(const std::string& s) {
    char* p = (char*)malloc(s.size() + 1);
    if (p) memcpy(p, s.c_str(), s.size() + 1);
    return p;
}

// A copy of `w` in a buffer from malloc, which the caller frees.
template <typename T> T* malloc_copy(const std::vector<T>& w) {
    T* p = static_cast<T*>(malloc(w.size() * sizeof(T) + 4));
    memcpy(p, w.data(), w.size() * sizeof(T));
    return p;
}
// Chunk k's samples w[k] in a buffer of its own from malloc (sb200_i16_free), its length in lens[k].
template <typename T, typename P> void copy_out(const std::vector<std::vector<T>>& w, P* outs, size_t* lens) {
    for (size_t k = 0; k < w.size(); k++) {
        outs[k] = malloc_copy(w[k]);
        lens[k] = w[k].size();
    }
}

template <typename F>
int32_t guarded(sb200_error* err, F&& f) {
    if (err) { err->code = 0; err->message = nullptr; }
    try {
        f();
        return 0;
    } catch (const Error& e) {
        if (err) { err->code = e.code; err->message = dup_cstr(e.what()); }
        return e.code;
    } catch (const std::exception& e) {
        if (err) { err->code = 19; err->message = dup_cstr(e.what()); }
        return 19;
    } catch (...) {
        if (err) { err->code = -1; err->message = dup_cstr("panic"); }
        return -1;
    }
}

void fetch_audio(Job& j, sb200_audio* outs, float wall_ms) {
    if (!j.ran || j.encode_only) throw Error(19, "job has not produced audio");
    Voice& v = *j.v;
    SB_CUDA(cudaSetDevice(v.device));
    PinnedBlock* blk = pin_acquire((size_t)j.out_total * 4 + 16);
    cudaError_t e = cudaMemcpyAsync(blk->base, j.d_wav, (size_t)j.out_total * 4, cudaMemcpyDeviceToHost, j.ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(j.ctx->stream);
    if (e != cudaSuccess) { pin_release(blk); throw Error(19, std::string("CUDA error: ") + cudaGetErrorString(e)); }
    blk->refs = (int)j.B;
    std::lock_guard<std::mutex> g(g_pin_mu);
    for (size_t b = 0; b < j.B; b++) {
        outs[b].data = blk->base + j.osegs[b].out_off;
        outs[b].len = (size_t)j.osegs[b].len * j.out_hop;
        outs[b].sample_rate = (uint32_t)j.osr[b];
        outs[b].inference_ms = wall_ms * (j.out_total ? (float)outs[b].len / (float)j.out_total : 0.f);
        g_owner[outs[b].data] = blk;
    }
}

double now_ms() {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// Device buffers of one debug hook call, freed however the call ends (an SB_CUDA that throws included).
struct DeviceBuffers {
    std::vector<void*> ptrs;
    DeviceBuffers() = default;
    DeviceBuffers(const DeviceBuffers&) = delete;
    DeviceBuffers& operator=(const DeviceBuffers&) = delete;
    ~DeviceBuffers() { for (void* p : ptrs) cudaFree(p); }
    template <typename T> T* alloc(size_t n) {
        void* p = nullptr;
        SB_CUDA(cudaMalloc(&p, n * sizeof(T)));
        ptrs.push_back(p);
        return static_cast<T*>(p);
    }
    // n elements: the m of host array h, then zeros
    template <typename T> T* upload(const T* h, size_t m, size_t n) {
        T* d = alloc<T>(n);
        if (n > m) SB_CUDA(cudaMemset(d, 0, n * sizeof(T)));
        SB_CUDA(cudaMemcpy(d, h, m * sizeof(T), cudaMemcpyHostToDevice));
        return d;
    }
};

// The output stage of a debug hook's plan o run on stream 0 over the n samples at x, one segment at hop 1 read plainly,
// with its buffers carved from arenas of the call's own, freed however the call ends.  taps (when given): the filter
// the plan's resample segments read, put on the device here.  The stage has finished when the constructor returns.
struct HookStage {
    struct Arenas {
        Arena dev, pin{true};
        ~Arenas() { dev.release(); pin.release(); }
    } a;
    OutputBufs b;
    Wave out;
    HookStage(OutputPlan& o, const float* x, size_t n, const std::vector<float>& taps = {}) {
        Staged<FrameSeg> seg; Staged<PcmPost> post; float* dt = nullptr;
        plan(a.dev, a.pin, [&](Arena& dev, Arena& pin) {
            seg.carve(dev, pin, 1); post.carve(dev, pin, 1);
            dt = taps.empty() ? nullptr : dev.get<float>(taps.size());
            b.carve(dev, pin, o, (long long)n, nullptr);
        });
        if (dt) {
            SB_CUDA(cudaMemcpy(dt, taps.data(), taps.size() * 4, cudaMemcpyHostToDevice));
            for (ResampleSeg& r : o.rp.segs) r.taps = dt;
        }
        seg.h[0] = FrameSeg{0, (int)n, 0, 0, 0}; post.h[0] = PcmPost();
        seg.upload(0); post.upload(0);
        SB_CUDA(cudaMemset(b.in + n, 0, 4 * sizeof(float)));
        if (n) SB_CUDA(cudaMemcpy(b.in, x, n * 4, cudaMemcpyHostToDevice));
        b.upload(o, 1, seg.h, post.h, 0);
        Profile none;
        out = run_output_stage(none, o, b, Wave{b.in, seg.d, post.d, 1}, 0);
        SB_CUDA(cudaDeviceSynchronize());
        SB_CUDA(cudaGetLastError());
    }
};

// The branches of a 64-channel ResBlock2 stage of kernel sizes ks[b] and dilations dils[2b], dils[2b + 1]; each conv's
// ConvW from `make` (weights and images, or only the shape).  False on a malformed description.
template <typename Make> bool debug_stage(int32_t nbr, const int32_t* ks, const int32_t* dils, std::vector<ResBW>& res, Make&& make) {
    if (nbr <= 0 || !ks || !dils) return false;
    res.assign(nbr, ResBW{});
    for (int b = 0; b < nbr; b++) {
        if (ks[b] <= 0 || ks[b] > SB_MAX_TAPS || dils[2 * b] <= 0 || dils[2 * b + 1] <= 0) return false;
        res[b].k = ks[b];
        res[b].dils = {dils[2 * b], dils[2 * b + 1]};
        for (int cv = 0; cv < 2; cv++) res[b].c1.push_back(make(b, cv));
    }
    return true;
}

}  // namespace

extern "C" {

const char* sb200_version(void) { return "sonata_b200 0.1.0 (sm_90a)"; }
void sb200_string_free(char* s) { free(s); }
void sb200_ids_free(int64_t* ids) { free(ids); }
void sb200_buffer_free(float* p) { free(p); }
int32_t sb200_device_count(void) { int n = 0; return cudaGetDeviceCount(&n) == cudaSuccess ? n : 0; }

void sb200_audio_free(sb200_audio* a) {
    if (!a || !a->data) return;
    PinnedBlock* blk = nullptr;
    {
        std::lock_guard<std::mutex> g(g_pin_mu);
        auto it = g_owner.find(a->data);
        if (it != g_owner.end()) { blk = it->second; g_owner.erase(it); }
    }
    if (blk) { if (--blk->refs == 0) pin_release(blk); }
    else free(a->data);
    a->data = nullptr; a->len = 0;
}

int32_t sb200_voice_load(const char* config_path, int32_t device, sb200_voice** out, sb200_error* err) {
    return guarded(err, [&] {
        if (!config_path || !out) throw Error(19, "null argument");
        Voice* v = load_voice(config_path, device);
        *out = new sb200_voice{std::shared_ptr<Voice>(v)};
    });
}
void sb200_voice_free(sb200_voice* v) { delete v; }

int32_t sb200_audio_output_info(const sb200_voice* v, sb200_audio_info* out, sb200_error* err) {
    return guarded(err, [&] {
        out->sample_rate = (uint32_t)v->v->sample_rate; out->num_channels = 1; out->sample_width = 2;
    });
}

static void cfg_out(const SynthConfig& c, sb200_synth_config* o) {
    o->speaker = c.speaker; o->has_speaker = c.has_speaker ? 1 : 0;
    o->noise_scale = c.noise_scale; o->length_scale = c.length_scale; o->noise_w = c.noise_w;
}
static std::vector<SynthConfig> cfgs_in(const sb200_synth_config* c, size_t n) {
    std::vector<SynthConfig> out(n);
    for (size_t b = 0; b < n; b++) {
        out[b].speaker = c[b].speaker; out[b].has_speaker = c[b].has_speaker != 0;
        out[b].noise_scale = c[b].noise_scale; out[b].length_scale = c[b].length_scale; out[b].noise_w = c[b].noise_w;
    }
    return out;
}
int32_t sb200_get_default_synthesis_config(const sb200_voice* v, sb200_synth_config* out, sb200_error* err) {
    return guarded(err, [&] {   // always Some(0), piper/src/lib.rs:444-451
        SynthConfig c = v->v->factory_cfg; c.speaker = 0; c.has_speaker = true; cfg_out(c, out);
    });
}
int32_t sb200_get_fallback_synthesis_config(const sb200_voice* v, sb200_synth_config* out, sb200_error* err) {
    return guarded(err, [&] { std::shared_lock<std::shared_mutex> g(v->v->cfg_mu); cfg_out(v->v->cfg, out); });
}
int32_t sb200_set_fallback_synthesis_config(sb200_voice* v, const sb200_synth_config* c, sb200_error* err) {
    return guarded(err, [&] {   // _do_set_default_synth_config, piper/src/lib.rs:215-231
        std::unique_lock<std::shared_mutex> g(v->v->cfg_mu);
        v->v->cfg.length_scale = c->length_scale; v->v->cfg.noise_scale = c->noise_scale; v->v->cfg.noise_w = c->noise_w;
        if (c->has_speaker) {
            check_config(*v->v, cfgs_in(c, 1)[0], "");
            v->v->cfg.speaker = c->speaker; v->v->cfg.has_speaker = true;
        }
    });
}
int32_t sb200_get_language(const sb200_voice* v, char** out, sb200_error* err) {
    return guarded(err, [&] { *out = dup_cstr(v->v->language_code.empty() ? v->v->espeak_voice : v->v->language_code); });
}
int32_t sb200_get_quality(const sb200_voice* v, char** out, sb200_error* err) {
    return guarded(err, [&] { *out = dup_cstr(v->v->quality.empty() ? "unknown" : v->v->quality); });
}
int32_t sb200_supports_streaming_output(const sb200_voice* v) { return v->v->streaming ? 1 : 0; }
int32_t sb200_num_speakers(const sb200_voice* v) { return v->v->num_speakers; }
int64_t sb200_speaker_name_to_id(const sb200_voice* v, const char* name) {
    auto it = v->v->speaker_id_map.find(name ? name : "");
    return it == v->v->speaker_id_map.end() ? -1 : it->second;
}

int32_t sb200_phonemes_to_input_ids(const sb200_voice* v, const char* ph, int64_t** ids, size_t* n, sb200_error* err) {
    return guarded(err, [&] {
        std::vector<long long> r = v->v->phonemes_to_ids(ph);
        *ids = (int64_t*)malloc(r.size() * sizeof(int64_t));
        for (size_t i = 0; i < r.size(); i++) (*ids)[i] = r[i];
        *n = r.size();
    });
}

int32_t sb200_phonemes_to_input_ids_map(const sb200_voice* v, const char* ph, int64_t** ids, int64_t** src_char,
                                        size_t* n, sb200_error* err) {
    return guarded(err, [&] {
        std::vector<long long> src;
        std::vector<long long> r = v->v->phonemes_to_ids(ph, &src);
        *ids = (int64_t*)malloc(r.size() * sizeof(int64_t));
        *src_char = (int64_t*)malloc(r.size() * sizeof(int64_t));
        for (size_t i = 0; i < r.size(); i++) { (*ids)[i] = r[i]; (*src_char)[i] = src[i]; }
        *n = r.size();
    });
}

// Measured loudness and applied gains of a job's last run into lufs / gain (either may be null).
static void job_loudness(const Job& j, double* lufs, float* gain) {
    if (!j.ran || j.loud_ran.empty()) throw Error(19, "the job's last run measured no loudness (no utterance had a target)");
    if (lufs) std::copy(j.loud_lufs.begin(), j.loud_lufs.end(), lufs);
    if (gain) std::copy(j.loud_gain.begin(), j.loud_gain.end(), gain);
}

// Each utterance's stretched length, delivered length and frame count of a job's last run (each may be null).
static void job_prosody(const Job& j, int64_t* n1, int64_t* n2, int32_t* frames) {
    if (!j.ran || j.pros_ran.empty())
        throw Error(19, "the job's last run had no prosody stage (no utterance asked for a pitch or a tempo)");
    for (size_t b = 0; b < j.B; b++) {
        if (n1) n1[b] = j.pros_ran[b].n1;
        if (n2) n2[b] = j.pros_ran[b].n2;
        if (frames) frames[b] = j.pros_ran[b].F;
    }
}

// u* and L(u*) of every span of a job's last run's targets (each may be null).
static void job_targets(const Job& j, float* factor, int64_t* len) {
    if (!j.ran || j.fit_u.empty()) throw Error(19, "the job's last run had no target durations");
    if (factor) std::copy(j.fit_u.begin(), j.fit_u.end(), factor);
    if (len) std::copy(j.fit_len.begin(), j.fit_len.end(), len);
}

int32_t sb200_speak_batch_ids_fit(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                  const sb200_synth_config* cfgs, const float* scale_packed,
                                  const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                  const uint32_t* output_rates, const float* target_lufs, const float* pitch,
                                  const float* tempo, const float* pitch_packed, const float* formants,
                                  const int64_t* blend_speakers, const float* blend_weights,
                                  const size_t* blend_offsets, const float* volume_db_packed,
                                  const float* breaks_ms_packed, const int64_t* fit_first, const int64_t* fit_end,
                                  const float* fit_ms, const size_t* fit_offsets, sb200_audio* outs,
                                  int32_t* id_frames_out, int64_t* bounds_out, double* lufs_out, float* gain_out,
                                  float* fit_factor_out, int64_t* fit_len_out, sb200_error* err) {
    return guarded(err, [&] {
        const double t0 = now_ms();
        static_assert(sizeof(long long) == sizeof(int64_t), "");
        static_assert(sizeof(unsigned long long) == sizeof(uint64_t), "");
        if (output_rates)       // before the job: the rates are checked against the voice's config alone
            for (size_t b = 0; b < batch; b++)
                if (output_rates[b] != 0 && output_rates[b] != (uint32_t)v->v->sample_rate)
                    resample_ratio(v->v->sample_rate, output_rates[b], "utterance " + std::to_string(b) + ": ");
        const bool loud = check_loudness_targets(target_lufs, batch);
        check_prosody(pitch, tempo, batch);
        check_pitch_contour(pitch_packed, offsets, batch, pitch);
        check_formants(formants, batch);
        canonical_blends(*v->v, reinterpret_cast<const long long*>(blend_speakers), blend_weights, blend_offsets, batch,
                         "utterance");
        check_volume_contour(volume_db_packed, offsets, batch);
        check_breaks(breaks_ms_packed, offsets, batch);
        const long long* ff = reinterpret_cast<const long long*>(fit_first);
        const long long* fe = reinterpret_cast<const long long*>(fit_end);
        const bool fit = check_targets(ff, fe, fit_ms, fit_offsets, offsets, batch, tempo);
        std::unique_ptr<Job> j(create_job(v->v.get(), reinterpret_cast<const long long*>(ids), offsets, batch, nullptr,
                                          nullptr, nullptr, false));
        if (cfgs) set_job_configs(*j, cfgs_in(cfgs, batch).data());
        set_job_durations(*j, scale_packed, frames_packed);
        set_job_seeds(*j, reinterpret_cast<const unsigned long long*>(seeds), seeded);
        set_job_output_rates(*j, output_rates);
        set_job_loudness(*j, target_lufs);
        set_job_prosody(*j, pitch, tempo);
        set_job_pitch_contour(*j, pitch_packed);
        set_job_formants(*j, formants);
        set_job_blends(*j, reinterpret_cast<const long long*>(blend_speakers), blend_weights, blend_offsets);
        set_job_volume_contour(*j, volume_db_packed);
        set_job_breaks(*j, breaks_ms_packed);
        set_job_targets(*j, ff, fe, fit_ms, fit_offsets);
        j->run(nullptr, 0);
        fetch_audio(*j, outs, 0.f);
        if (id_frames_out) {
            const std::vector<int>& f = job_id_frames(*j);
            std::copy(f.begin(), f.end(), id_frames_out);
        }
        if (bounds_out) {
            const std::vector<long long> e = job_prosody_bounds(*j);
            std::copy(e.begin(), e.end(), bounds_out);
        }
        if (loud) job_loudness(*j, lufs_out, gain_out);
        if (fit) job_targets(*j, fit_factor_out, fit_len_out);
        const float wall = (float)(now_ms() - t0);
        for (size_t b = 0; b < batch; b++)
            outs[b].inference_ms = wall * (j->out_total ? (float)outs[b].len / (float)j->out_total : 0.f);
    });
}
int32_t sb200_speak_batch_ids_breaks(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                     const sb200_synth_config* cfgs, const float* scale_packed,
                                     const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                     const uint32_t* output_rates, const float* target_lufs, const float* pitch,
                                     const float* tempo, const float* pitch_packed, const float* formants,
                                     const int64_t* blend_speakers, const float* blend_weights,
                                     const size_t* blend_offsets, const float* volume_db_packed,
                                     const float* breaks_ms_packed, sb200_audio* outs, int32_t* id_frames_out,
                                     int64_t* bounds_out, double* lufs_out, float* gain_out, sb200_error* err) {
    return sb200_speak_batch_ids_fit(v, ids, offsets, batch, cfgs, scale_packed, frames_packed, seeds, seeded,
                                     output_rates, target_lufs, pitch, tempo, pitch_packed, formants, blend_speakers,
                                     blend_weights, blend_offsets, volume_db_packed, breaks_ms_packed, nullptr, nullptr,
                                     nullptr, nullptr, outs, id_frames_out, bounds_out, lufs_out, gain_out, nullptr,
                                     nullptr, err);
}
int32_t sb200_speak_batch_ids_volume(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                     const sb200_synth_config* cfgs, const float* scale_packed,
                                     const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                     const uint32_t* output_rates, const float* target_lufs, const float* pitch,
                                     const float* tempo, const float* pitch_packed, const float* formants,
                                     const int64_t* blend_speakers, const float* blend_weights,
                                     const size_t* blend_offsets, const float* volume_db_packed, sb200_audio* outs,
                                     int32_t* id_frames_out, int64_t* bounds_out, double* lufs_out, float* gain_out,
                                     sb200_error* err) {
    return sb200_speak_batch_ids_breaks(v, ids, offsets, batch, cfgs, scale_packed, frames_packed, seeds, seeded,
                                        output_rates, target_lufs, pitch, tempo, pitch_packed, formants, blend_speakers,
                                        blend_weights, blend_offsets, volume_db_packed, nullptr, outs, id_frames_out,
                                        bounds_out, lufs_out, gain_out, err);
}
int32_t sb200_speak_batch_ids_blends(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                     const sb200_synth_config* cfgs, const float* scale_packed,
                                     const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                     const uint32_t* output_rates, const float* target_lufs, const float* pitch,
                                     const float* tempo, const float* pitch_packed, const float* formants,
                                     const int64_t* blend_speakers, const float* blend_weights,
                                     const size_t* blend_offsets, sb200_audio* outs, int32_t* id_frames_out,
                                     int64_t* bounds_out, double* lufs_out, float* gain_out, sb200_error* err) {
    return sb200_speak_batch_ids_volume(v, ids, offsets, batch, cfgs, scale_packed, frames_packed, seeds, seeded,
                                        output_rates, target_lufs, pitch, tempo, pitch_packed, formants, blend_speakers,
                                        blend_weights, blend_offsets, nullptr, outs, id_frames_out, bounds_out, lufs_out,
                                        gain_out, err);
}
int32_t sb200_speak_batch_ids_formants(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                       const sb200_synth_config* cfgs, const float* scale_packed,
                                       const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                       const uint32_t* output_rates, const float* target_lufs, const float* pitch,
                                       const float* tempo, const float* pitch_packed, const float* formants,
                                       sb200_audio* outs, int32_t* id_frames_out, int64_t* bounds_out,
                                       double* lufs_out, float* gain_out, sb200_error* err) {
    return sb200_speak_batch_ids_blends(v, ids, offsets, batch, cfgs, scale_packed, frames_packed, seeds, seeded,
                                        output_rates, target_lufs, pitch, tempo, pitch_packed, formants, nullptr, nullptr,
                                        nullptr, outs, id_frames_out, bounds_out, lufs_out, gain_out, err);
}
int32_t sb200_speak_batch_ids_contour(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                      const sb200_synth_config* cfgs, const float* scale_packed,
                                      const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                      const uint32_t* output_rates, const float* target_lufs, const float* pitch,
                                      const float* tempo, const float* pitch_packed, sb200_audio* outs,
                                      int32_t* id_frames_out, int64_t* bounds_out, double* lufs_out, float* gain_out,
                                      sb200_error* err) {
    return sb200_speak_batch_ids_formants(v, ids, offsets, batch, cfgs, scale_packed, frames_packed, seeds, seeded,
                                          output_rates, target_lufs, pitch, tempo, pitch_packed, nullptr, outs,
                                          id_frames_out, bounds_out, lufs_out, gain_out, err);
}
int32_t sb200_speak_batch_ids_prosody(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                      const sb200_synth_config* cfgs, const float* scale_packed,
                                      const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                      const uint32_t* output_rates, const float* target_lufs, const float* pitch,
                                      const float* tempo, sb200_audio* outs, int32_t* id_frames_out, double* lufs_out,
                                      float* gain_out, sb200_error* err) {
    return sb200_speak_batch_ids_contour(v, ids, offsets, batch, cfgs, scale_packed, frames_packed, seeds, seeded,
                                         output_rates, target_lufs, pitch, tempo, nullptr, outs, id_frames_out, nullptr,
                                         lufs_out, gain_out, err);
}
int32_t sb200_speak_batch_ids_loudness(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                       const sb200_synth_config* cfgs, const float* scale_packed,
                                       const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                       const uint32_t* output_rates, const float* target_lufs, sb200_audio* outs,
                                       int32_t* id_frames_out, double* lufs_out, float* gain_out, sb200_error* err) {
    return sb200_speak_batch_ids_prosody(v, ids, offsets, batch, cfgs, scale_packed, frames_packed, seeds, seeded,
                                         output_rates, target_lufs, nullptr, nullptr, outs, id_frames_out, lufs_out,
                                         gain_out, err);
}
int32_t sb200_speak_batch_ids_rates(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                    const sb200_synth_config* cfgs, const float* scale_packed,
                                    const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                    const uint32_t* output_rates, sb200_audio* outs, int32_t* id_frames_out,
                                    sb200_error* err) {
    return sb200_speak_batch_ids_loudness(v, ids, offsets, batch, cfgs, scale_packed, frames_packed, seeds, seeded,
                                          output_rates, nullptr, outs, id_frames_out, nullptr, nullptr, err);
}
int32_t sb200_speak_batch_ids_seeded(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                     const sb200_synth_config* cfgs, const float* scale_packed,
                                     const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                     sb200_audio* outs, int32_t* id_frames_out, sb200_error* err) {
    return sb200_speak_batch_ids_rates(v, ids, offsets, batch, cfgs, scale_packed, frames_packed, seeds, seeded, nullptr,
                                       outs, id_frames_out, err);
}
int32_t sb200_speak_batch_ids_durations(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                        const sb200_synth_config* cfgs, const float* scale_packed,
                                        const int32_t* frames_packed, sb200_audio* outs, int32_t* id_frames_out,
                                        sb200_error* err) {
    return sb200_speak_batch_ids_seeded(v, ids, offsets, batch, cfgs, scale_packed, frames_packed, nullptr, nullptr, outs,
                                        id_frames_out, err);
}
int32_t sb200_speak_batch_ids_configs(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                      const sb200_synth_config* cfgs, sb200_audio* outs, sb200_error* err) {
    return sb200_speak_batch_ids_durations(v, ids, offsets, batch, cfgs, nullptr, nullptr, outs, nullptr, err);
}
int32_t sb200_speak_batch_ids(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                              sb200_audio* outs, sb200_error* err) {
    return sb200_speak_batch_ids_configs(v, ids, offsets, batch, nullptr, outs, err);
}
int32_t sb200_speak_ids(sb200_voice* v, const int64_t* ids, size_t n, sb200_audio* out, sb200_error* err) {
    const size_t offs[2] = {0, n};
    return sb200_speak_batch_ids(v, ids, offs, 1, out, err);
}
int32_t sb200_speak_batch(sb200_voice* v, const char* const* ph, size_t batch, sb200_audio* outs, sb200_error* err) {
    std::vector<int64_t> ids; std::vector<size_t> offs{0};
    int32_t rc = guarded(err, [&] {
        for (size_t b = 0; b < batch; b++) {
            std::vector<long long> r = v->v->phonemes_to_ids(ph[b]);
            ids.insert(ids.end(), r.begin(), r.end());
            offs.push_back(ids.size());
        }
    });
    if (rc) return rc;
    return sb200_speak_batch_ids(v, ids.data(), offs.data(), batch, outs, err);
}
int32_t sb200_speak_one_sentence(sb200_voice* v, const char* ph, sb200_audio* out, sb200_error* err) {
    return sb200_speak_batch(v, &ph, 1, out, err);
}

// ---- job API ----
int32_t sb200_job_create(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                         const float* const* eps_w, const float* const* eps_z, const size_t* eps_z_frames,
                         sb200_job** out, sb200_error* err) {
    return guarded(err, [&] {
        Job* j = create_job(v->v.get(), reinterpret_cast<const long long*>(ids), offsets, batch, eps_w, eps_z, eps_z_frames, false);
        *out = new sb200_job{j, v->v};
    });
}
int32_t sb200_job_set_debug(sb200_job* job, int32_t on) { job->j->debug = on != 0; return 0; }
int32_t sb200_job_set_configs(sb200_job* job, const sb200_synth_config* cfgs, sb200_error* err) {
    return guarded(err, [&] {
        Job& j = *job->j;
        set_job_configs(j, cfgs ? cfgs_in(cfgs, j.B).data() : nullptr);
    });
}
int32_t sb200_job_set_durations(sb200_job* job, const float* scale_packed, const int32_t* frames_packed, sb200_error* err) {
    return guarded(err, [&] { set_job_durations(*job->j, scale_packed, frames_packed); });
}
int32_t sb200_job_set_seeds(sb200_job* job, const uint64_t* seeds, const int32_t* seeded, sb200_error* err) {
    return guarded(err, [&] { set_job_seeds(*job->j, reinterpret_cast<const unsigned long long*>(seeds), seeded); });
}
int32_t sb200_job_set_output_rates(sb200_job* job, const uint32_t* rates, sb200_error* err) {
    return guarded(err, [&] { set_job_output_rates(*job->j, rates); });
}
int32_t sb200_job_set_loudness(sb200_job* job, const float* target_lufs, sb200_error* err) {
    return guarded(err, [&] { set_job_loudness(*job->j, target_lufs); });
}
int32_t sb200_job_loudness(const sb200_job* job, double* lufs, float* gain, sb200_error* err) {
    return guarded(err, [&] { job_loudness(*job->j, lufs, gain); });
}
int32_t sb200_job_set_prosody(sb200_job* job, const float* pitch, const float* tempo, sb200_error* err) {
    return guarded(err, [&] { set_job_prosody(*job->j, pitch, tempo); });
}
int32_t sb200_job_prosody(const sb200_job* job, int64_t* n1, int64_t* n2, int32_t* frames, sb200_error* err) {
    return guarded(err, [&] { job_prosody(*job->j, n1, n2, frames); });
}
int32_t sb200_job_set_pitch_contour(sb200_job* job, const float* pitch_packed, sb200_error* err) {
    return guarded(err, [&] { set_job_pitch_contour(*job->j, pitch_packed); });
}
int32_t sb200_job_set_formants(sb200_job* job, const float* formants, sb200_error* err) {
    return guarded(err, [&] { set_job_formants(*job->j, formants); });
}
int32_t sb200_job_set_volume_contour(sb200_job* job, const float* volume_db_packed, sb200_error* err) {
    return guarded(err, [&] { set_job_volume_contour(*job->j, volume_db_packed); });
}
int32_t sb200_job_set_breaks(sb200_job* job, const float* breaks_ms_packed, sb200_error* err) {
    return guarded(err, [&] { set_job_breaks(*job->j, breaks_ms_packed); });
}
int32_t sb200_job_set_targets(sb200_job* job, const int64_t* fit_first, const int64_t* fit_end, const float* fit_ms,
                              const size_t* fit_offsets, sb200_error* err) {
    return guarded(err, [&] {
        set_job_targets(*job->j, reinterpret_cast<const long long*>(fit_first),
                        reinterpret_cast<const long long*>(fit_end), fit_ms, fit_offsets);
    });
}
int32_t sb200_job_targets(const sb200_job* job, float* fit_factor, int64_t* fit_len, size_t capacity, sb200_error* err) {
    return guarded(err, [&] {
        const Job& j = *job->j;
        if (j.ran && capacity < j.fit_u.size())
            throw Error(19, "target durations: the destination holds " + std::to_string(capacity) + " spans, the job has " +
                                std::to_string(j.fit_u.size()));
        job_targets(j, fit_factor, fit_len);
    });
}
int32_t sb200_job_set_speaker_blends(sb200_job* job, const int64_t* speakers, const float* weights, const size_t* offsets,
                                     sb200_error* err) {
    return guarded(err, [&] {
        set_job_blends(*job->j, reinterpret_cast<const long long*>(speakers), weights, offsets);
    });
}
int32_t sb200_job_prosody_bounds(sb200_job* job, int64_t* out_packed, size_t capacity, sb200_error* err) {
    return guarded(err, [&] {
        Job& j = *job->j;
        if (!out_packed || capacity < j.ids.size())
            throw Error(19, "prosody bounds: the destination holds " + std::to_string(capacity) + " entries, the job has " +
                                std::to_string(j.ids.size()) + " ids");
        const std::vector<long long> e = job_prosody_bounds(j);
        std::copy(e.begin(), e.end(), out_packed);
    });
}
int32_t sb200_job_id_frames(sb200_job* job, int32_t* out_packed, size_t capacity, sb200_error* err) {
    return guarded(err, [&] {
        Job& j = *job->j;
        if (!out_packed) throw Error(19, "null destination");
        const std::vector<int>& f = job_id_frames(j);
        if (capacity < f.size())
            throw Error(19, "capacity " + std::to_string(capacity) + " is smaller than the job's " + std::to_string(f.size()) + " ids");
        std::copy(f.begin(), f.end(), out_packed);
    });
}
int32_t sb200_job_run(sb200_job* job, float* d_out, size_t cap, float* device_ms, sb200_error* err) {
    return guarded(err, [&] { job->j->run(d_out, cap); if (device_ms) *device_ms = job->j->last_ms; });
}
int32_t sb200_job_fetch(sb200_job* job, sb200_audio* outs, sb200_error* err) {
    return guarded(err, [&] { fetch_audio(*job->j, outs, job->j->last_ms); });
}
int32_t sb200_job_fetch_i16(sb200_job* job, int16_t** outs, size_t* lens, sb200_error* err) {
    return guarded(err, [&] {
        Job& j = *job->j;
        SB_CUDA(cudaSetDevice(j.v->device));
        PinnedBlock* blk = pin_acquire((size_t)j.out_total * 2 + 16);
        int16_t* h = reinterpret_cast<int16_t*>(blk->base);
        try { job_i16_to_host(j, 1.f, h); } catch (...) { pin_release(blk); throw; }
        for (size_t b = 0; b < j.B; b++) {
            const size_t n = (size_t)j.osegs[b].len * j.out_hop;
            outs[b] = (int16_t*)malloc(n * 2 + 2);
            memcpy(outs[b], h + j.osegs[b].out_off, n * 2);
            lens[b] = n;
        }
        pin_release(blk);
    });
}
void sb200_i16_free(int16_t* p) { free(p); }
int32_t sb200_job_fetch_g711(sb200_job* job, int32_t law, const float* gains, uint8_t** outs, size_t* lens,
                             sb200_error* err) {
    return guarded(err, [&] {
        Job& j = *job->j;
        g711_format(law, "");
        if (!j.ran || j.encode_only) throw Error(19, "job has not produced audio");
        if (!outs || !lens) throw Error(19, "null argument");
        SB_CUDA(cudaSetDevice(j.v->device));
        PinnedBlock* blk = pin_acquire((size_t)j.out_total + 16);
        uint8_t* h = reinterpret_cast<uint8_t*>(blk->base);
        try { job_g711_to_host(j, law, gains, h); } catch (...) { pin_release(blk); throw; }
        for (size_t b = 0; b < j.B; b++) {
            const size_t n = (size_t)j.osegs[b].len * j.out_hop;
            outs[b] = (uint8_t*)malloc(n + 1);
            memcpy(outs[b], h + j.osegs[b].out_off, n);
            lens[b] = n;
        }
        pin_release(blk);
    });
}
void sb200_bytes_free(uint8_t* p) { free(p); }
int32_t sb200_job_fetch_flac(sb200_job* job, const float* gains, uint8_t** outs, size_t* lens, sb200_error* err) {
    return guarded(err, [&] {
        Job& j = *job->j;
        if (!j.ran || j.encode_only) throw Error(19, "job has not produced audio");
        if (!outs || !lens) throw Error(19, "null argument");
        job_flac_to_host(j, gains, outs, lens);
    });
}
int32_t sb200_flac_encode(int32_t device, const int16_t* x, size_t n, uint32_t sample_rate, uint8_t** out, size_t* len,
                          sb200_error* err) {
    return guarded(err, [&] {
        if (!flac_rate_supported(sample_rate))
            throw Error(19, "FLAC: sample rate " + std::to_string(sample_rate) + " Hz is not one of the output rates");
        if (!out || !len || (!x && n > 0)) throw Error(19, "null argument");
        SB_CUDA(cudaSetDevice(device));
        DeviceBuffers d;
        const short* dx = n ? d.upload(reinterpret_cast<const short*>(x), n, n) : nullptr;
        flac_encode(dx, {FlacStream{0, (long long)n, (long long)sample_rate}}, 0, out, len);
    });
}

int32_t sb200_voice_set_watermark(sb200_voice* v, const sb200_watermark* wm, sb200_error* err) {
    return guarded(err, [&] {
        Voice& V = *v->v;
        if (!wm) {
            std::unique_lock<std::shared_mutex> g(V.cfg_mu);
            V.wm_on = false;
            return;
        }
        check_watermark(wm->payload, wm->strength_db);
        bool known;
        {
            std::shared_lock<std::shared_mutex> g(V.cfg_mu);
            known = V.wm_chips.count(wm->key) != 0;
        }
        // a new key's tables are built before the lock is taken, so running jobs of the voice do not wait for them
        signed char* built = nullptr;
        if (!known) {
            SB_CUDA(cudaSetDevice(V.device));
            built = build_watermark_chips(wm->key);
        }
        std::unique_lock<std::shared_mutex> g(V.cfg_mu);
        const signed char*& chips = V.wm_chips[wm->key];
        if (!chips && built) {
            V.dev_allocs.push_back(built);
            chips = built;
        } else if (built) {
            cudaFree(built);       // another thread set the same key meanwhile
        }
        V.wm = Watermark{wm->key, wm->payload, wm->strength_db, chips};
        V.wm_on = true;
    });
}
int32_t sb200_voice_watermark(const sb200_voice* v, sb200_watermark* out, int32_t* on, sb200_error* err) {
    return guarded(err, [&] {
        if (!on) throw Error(19, "null argument");
        const Voice& V = *v->v;
        std::shared_lock<std::shared_mutex> g(V.cfg_mu);
        *on = V.wm_on ? 1 : 0;
        if (V.wm_on && out) *out = sb200_watermark{V.wm.key, V.wm.payload, V.wm.strength_db};
    });
}
int32_t sb200_watermark_detect(int32_t device, uint64_t key, int32_t fmt, const void* packed, const size_t* offsets,
                               size_t batch, sb200_watermark_result* out, sb200_error* err) {
    return guarded(err, [&] {
        if (fmt != 0 && fmt != 1)
            throw Error(19, "watermark detect: format " + std::to_string(fmt) + " is not 0 (f32) or 1 (i16)");
        if (batch && (!offsets || !out)) throw Error(19, "null argument");
        if (batch == 0) return;
        for (size_t b = 0; b < batch; b++)
            if (offsets[b + 1] < offsets[b])
                throw Error(19, "watermark detect: clip " + std::to_string(b) + " ends before it starts");
        const size_t n = offsets[batch] - offsets[0];
        if (n && !packed) throw Error(19, "null argument");
        SB_CUDA(cudaSetDevice(device));
        DeviceBuffers d;
        const size_t es = fmt == 0 ? 4 : 2;
        char* dx = d.alloc<char>(n * es + 16);
        if (n) SB_CUDA(cudaMemcpy(dx, static_cast<const char*>(packed) + offsets[0] * es, n * es, cudaMemcpyHostToDevice));
        std::vector<size_t> offs(offsets, offsets + batch + 1);
        for (size_t& o : offs) o -= offsets[0];
        std::vector<WatermarkScore> s(batch);
        watermark_detect(key, fmt, dx, offs.data(), batch, s.data(), 0);
        for (size_t b = 0; b < batch; b++) out[b] = sb200_watermark_result{s[b].marked, s[b].payload, s[b].offset, s[b].z0, s[b].z1};
    });
}

int32_t sb200_job_copy_out(sb200_job* job, void* dst, size_t cap, int32_t format, size_t* written, sb200_error* err) {
    return guarded(err, [&] {
        Job& j = *job->j;
        if (format < PCM_F32 || format > PCM_ALAW)
            throw Error(19, "format " + std::to_string(format) + " is not 0 (f32), 1 (i16), 2 (mu-law) or 3 (A-law)");
        if (!j.ran || j.encode_only) throw Error(19, "job has not produced audio");
        if (!dst) throw Error(19, "null destination");
        Voice& v = *j.v;
        SB_CUDA(cudaSetDevice(v.device));
        cudaStream_t st = j.ctx->stream;
        const size_t n = (size_t)j.out_total;
        const size_t bytes = n * pcm_bytes(format);
        if (bytes > cap) throw Error(19, "destination buffer is too small for the synthesis result");
        if (format == PCM_I16) {
            job_i16_to_host(j, 1.f, static_cast<int16_t*>(dst));
        } else if (format != PCM_F32) {
            job_g711_to_host(j, format == PCM_MULAW ? G711_MULAW : G711_ALAW, nullptr, static_cast<uint8_t*>(dst));
        } else {
            SB_CUDA(cudaMemcpyAsync(dst, j.d_wav, bytes, cudaMemcpyDeviceToHost, st));
            SB_CUDA(cudaStreamSynchronize(st));
        }
        if (written) *written = bytes;
    });
}
int32_t sb200_host_register(void* ptr, size_t bytes, sb200_error* err) {
    return guarded(err, [&] {
        const cudaError_t e = cudaHostRegister(ptr, bytes, cudaHostRegisterPortable);
        if (e != cudaSuccess) { cudaGetLastError(); throw Error(19, std::string("cudaHostRegister failed: ") + cudaGetErrorString(e)); }
    });
}
int32_t sb200_host_unregister(void* ptr) {
    const cudaError_t e = cudaHostUnregister(ptr);
    if (e != cudaSuccess) cudaGetLastError();
    return e == cudaSuccess ? 0 : 19;
}
size_t sb200_job_batch(const sb200_job* job) { return job->j->B; }
int32_t sb200_job_lengths(const sb200_job* job, int64_t* frames, int64_t* samples, int64_t* out_offsets) {
    const Job& j = *job->j;
    if (!j.ran) return 19;
    for (size_t b = 0; b < j.B; b++) {
        if (frames) frames[b] = j.y_len[b];
        if (samples) samples[b] = (int64_t)j.osegs[b].len * j.out_hop;
        if (out_offsets) out_offsets[b] = j.osegs[b].out_off;
    }
    return 0;
}
void sb200_job_free(sb200_job* job) { delete job; }

// ---- streaming halves ----
int32_t sb200_encode_ids(sb200_voice* v, const int64_t* ids, size_t n, sb200_latent** out, sb200_error* err) {
    return guarded(err, [&] { *out = new sb200_latent{encode_latent(v->v.get(), reinterpret_cast<const long long*>(ids), n), v->v}; });
}
int64_t sb200_latent_frames(const sb200_latent* z) { return z->l->frames; }
int32_t sb200_decode_chunk(sb200_voice* v, const sb200_latent* z, int64_t lo, int64_t hi, sb200_audio* out, sb200_error* err) {
    return guarded(err, [&] {
        ChunkPass p;
        p.chunks = {ChunkSpec{z->l, lo, hi}};
        p.single = true;
        ChunkResult r;
        decode_chunks(v->v.get(), p, r);
        out->data = malloc_copy(r.f32[0]);
        out->len = r.f32[0].size(); out->inference_ms = r.ms; out->sample_rate = (uint32_t)v->v->sample_rate;
    });
}
void sb200_latent_free(sb200_latent* z) { delete z; }

int32_t sb200_encode_batch_ids_targets(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                       const sb200_synth_config* cfgs, const float* scale_packed,
                                       const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                       const int64_t* blend_speakers, const float* blend_weights,
                                       const size_t* blend_offsets, const float* breaks_ms_packed,
                                       const int64_t* fit_first, const int64_t* fit_end, const float* fit_ms,
                                       const size_t* fit_offsets, float* fit_factor_out, int64_t* fit_len_out,
                                       sb200_latent** outs, sb200_error* err) {
    return guarded(err, [&] {
        const std::vector<SynthConfig> c = cfgs ? cfgs_in(cfgs, batch) : std::vector<SynthConfig>();
        check_breaks(breaks_ms_packed, offsets, batch);
        std::vector<Latent*> ls = encode_latents(v->v.get(), reinterpret_cast<const long long*>(ids), offsets, batch,
                                                 cfgs ? c.data() : nullptr, scale_packed, frames_packed,
                                                 reinterpret_cast<const unsigned long long*>(seeds), seeded,
                                                 reinterpret_cast<const long long*>(blend_speakers), blend_weights,
                                                 blend_offsets, breaks_ms_packed,
                                                 reinterpret_cast<const long long*>(fit_first),
                                                 reinterpret_cast<const long long*>(fit_end), fit_ms, fit_offsets,
                                                 fit_factor_out, reinterpret_cast<long long*>(fit_len_out));
        for (size_t b = 0; b < batch; b++) outs[b] = new sb200_latent{ls[b], v->v};
    });
}
int32_t sb200_encode_batch_ids_blends(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                      const sb200_synth_config* cfgs, const float* scale_packed,
                                      const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                      const int64_t* blend_speakers, const float* blend_weights,
                                      const size_t* blend_offsets, sb200_latent** outs, sb200_error* err) {
    return sb200_encode_batch_ids_targets(v, ids, offsets, batch, cfgs, scale_packed, frames_packed, seeds, seeded,
                                          blend_speakers, blend_weights, blend_offsets, nullptr, nullptr, nullptr,
                                          nullptr, nullptr, nullptr, nullptr, outs, err);
}
int32_t sb200_encode_batch_ids_seeded(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                      const sb200_synth_config* cfgs, const float* scale_packed,
                                      const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                      sb200_latent** outs, sb200_error* err) {
    return sb200_encode_batch_ids_blends(v, ids, offsets, batch, cfgs, scale_packed, frames_packed, seeds, seeded, nullptr,
                                         nullptr, nullptr, outs, err);
}
int32_t sb200_encode_batch_ids_durations(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                         const sb200_synth_config* cfgs, const float* scale_packed,
                                         const int32_t* frames_packed, sb200_latent** outs, sb200_error* err) {
    return sb200_encode_batch_ids_seeded(v, ids, offsets, batch, cfgs, scale_packed, frames_packed, nullptr, nullptr, outs,
                                         err);
}
int32_t sb200_encode_batch_ids_configs(sb200_voice* v, const int64_t* ids, const size_t* offsets, size_t batch,
                                       const sb200_synth_config* cfgs, sb200_latent** outs, sb200_error* err) {
    return sb200_encode_batch_ids_durations(v, ids, offsets, batch, cfgs, nullptr, nullptr, outs, err);
}
int64_t sb200_latent_id_frames(const sb200_latent* z, int32_t* out, size_t capacity) {
    const std::vector<int>& f = z->l->id_frames;
    if (out && capacity >= f.size()) std::copy(f.begin(), f.end(), out);
    return (int64_t)f.size();
}

namespace {
// A pass over chunks zs[k] frames [lo[k], hi[k]), k < n, with trims (null: none) and gains (null: 1).
ChunkPass chunk_pass(const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi, size_t n,
                     const int64_t* trim_lo_frames = nullptr, const int64_t* trim_hi_frames = nullptr,
                     const float* gain = nullptr) {
    ChunkPass p;
    p.chunks.resize(n);
    for (size_t k = 0; k < n; k++) {
        if (!zs[k]) throw Error(19, "chunk " + std::to_string(k) + ": null latent");
        ChunkSpec& c = p.chunks[k];
        c.z = zs[k]->l; c.lo = lo[k]; c.hi = hi[k];
        if (trim_lo_frames) c.trim_lo = trim_lo_frames[k];
        if (trim_hi_frames) c.trim_hi = trim_hi_frames[k];
        if (gain) c.gain = gain[k];
    }
    return p;
}
}  // namespace

int32_t sb200_decode_chunks(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi, size_t n,
                            sb200_audio* outs, sb200_error* err) {
    return guarded(err, [&] {
        ChunkResult r;
        decode_chunks(v->v.get(), chunk_pass(zs, lo, hi, n), r);
        size_t total = 0;
        for (auto& w : r.f32) total += w.size();
        for (size_t k = 0; k < n; k++) {
            outs[k].data = malloc_copy(r.f32[k]);
            outs[k].len = r.f32[k].size(); outs[k].sample_rate = (uint32_t)v->v->sample_rate;
            outs[k].inference_ms = r.ms * (total ? (float)r.f32[k].size() / (float)total : 0.f);
        }
    });
}

int32_t sb200_decode_chunks_i16(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi,
                                const int64_t* trim_lo_frames, const int64_t* trim_hi_frames, size_t n, int32_t fade,
                                const float* gain, int16_t** outs, size_t* lens, sb200_error* err) {
    return guarded(err, [&] {
        ChunkPass p = chunk_pass(zs, lo, hi, n, trim_lo_frames, trim_hi_frames, gain);
        p.fade = fade; p.format = 1;
        ChunkResult r;
        decode_chunks(v->v.get(), p, r);
        copy_out(r.i16, outs, lens);
    });
}

int32_t sb200_decode_chunks_g711(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi,
                                 const int64_t* trim_lo_frames, const int64_t* trim_hi_frames, size_t n, int32_t fade,
                                 const float* gain, int32_t law, uint8_t** outs, size_t* lens, sb200_error* err) {
    return guarded(err, [&] {
        const int fmt = g711_format(law, "");
        ChunkPass p = chunk_pass(zs, lo, hi, n, trim_lo_frames, trim_hi_frames, gain);
        p.fade = fade; p.format = fmt;
        ChunkResult r;
        decode_chunks(v->v.get(), p, r);
        copy_out(r.g711, outs, lens);
    });
}

int32_t sb200_resampler_create(sb200_voice* v, uint32_t out_rate, sb200_resampler** out, sb200_error* err) {
    return guarded(err, [&] {
        if (!v || !out) throw Error(19, "null argument");
        *out = new sb200_resampler{create_resampler(v->v.get(), out_rate), v->v};
    });
}
void sb200_resampler_free(sb200_resampler* r) { delete r; }

int32_t sb200_prosody_stream_create(sb200_voice* v, float pitch, float tempo, sb200_prosody_stream** out,
                                    sb200_error* err) {
    return guarded(err, [&] {
        if (!v || !out) throw Error(19, "null argument");
        Voice* w = v->v.get();
        if (w->device < 0 || !w->emb)
            throw Error(19, "Failed to run model inference. Error: voice was loaded config-only (device -1); libsonata_b200 has no CPU path");
        *out = new sb200_prosody_stream{create_prosody_stream(w, w->device, w->sample_rate, pitch, tempo), v->v};
    });
}
int32_t sb200_prosody_stream_create_contour(sb200_voice* v, const sb200_latent* z, const float* pitch_per_id,
                                            size_t n_ids, float tempo, sb200_prosody_stream** out, sb200_error* err) {
    return guarded(err, [&] {
        if (!v || !z || !out || (n_ids > 0 && !pitch_per_id)) throw Error(19, "null argument");
        Voice* w = v->v.get();
        if (w->device < 0 || !w->emb)
            throw Error(19, "Failed to run model inference. Error: voice was loaded config-only (device -1); libsonata_b200 has no CPU path");
        if (z->l->v != w) throw Error(19, "the latent was not encoded by this voice");
        const std::vector<int>& f = z->l->id_frames;
        if (n_ids != f.size())
            throw Error(19, "pitch contour: " + std::to_string(n_ids) + " ratios for a latent of " +
                                std::to_string(f.size()) + " ids");
        // the stream's input: the latent's frames at the hop, each id ending at its cumulative frames
        const long long hop = w->a.hop();
        std::vector<long long> ends(n_ids);
        long long c = 0;
        for (size_t i = 0; i < n_ids; i++) ends[i] = (c += f[i]) * hop;
        *out = new sb200_prosody_stream{create_prosody_stream_contour(w, w->device, w->sample_rate, z->l->frames * hop,
                                                                      ends.data(), pitch_per_id, n_ids, tempo),
                                        v->v};
    });
}
int32_t sb200_prosody_stream_create_formant(sb200_voice* v, const sb200_latent* z, float pitch,
                                            const float* pitch_per_id, size_t n_ids, float tempo, float formant,
                                            sb200_prosody_stream** out, sb200_error* err) {
    return sb200_prosody_stream_create_volume(v, z, pitch, pitch_per_id, n_ids, tempo, formant, nullptr, out, err);
}
int32_t sb200_prosody_stream_create_volume(sb200_voice* v, const sb200_latent* z, float pitch,
                                           const float* pitch_per_id, size_t n_ids, float tempo, float formant,
                                           const float* volume_db_per_id, sb200_prosody_stream** out,
                                           sb200_error* err) {
    return sb200_prosody_stream_create_breaks(v, z, pitch, pitch_per_id, n_ids, tempo, formant, volume_db_per_id,
                                              nullptr, out, err);
}
int32_t sb200_prosody_stream_create_breaks(sb200_voice* v, const sb200_latent* z, float pitch,
                                           const float* pitch_per_id, size_t n_ids, float tempo, float formant,
                                           const float* volume_db_per_id, const float* breaks_ms_per_id,
                                           sb200_prosody_stream** out, sb200_error* err) {
    return guarded(err, [&] {
        const bool per_id = pitch_per_id || volume_db_per_id || breaks_ms_per_id;
        if (!v || !out || (per_id && !z)) throw Error(19, "null argument");
        Voice* w = v->v.get();
        if (w->device < 0 || !w->emb)
            throw Error(19, "Failed to run model inference. Error: voice was loaded config-only (device -1); libsonata_b200 has no CPU path");
        std::vector<long long> ends;
        long long n = -1;
        if (per_id) {
            if (z->l->v != w) throw Error(19, "the latent was not encoded by this voice");
            const std::vector<int>& f = z->l->id_frames;
            if (n_ids != f.size())
                throw Error(19, std::string(pitch_per_id ? "pitch contour: " : volume_db_per_id ? "volume contour: "
                                                                                                : "breaks: ") +
                                    std::to_string(n_ids) +
                                    (pitch_per_id ? " ratios" : volume_db_per_id ? " levels" : " breaks") +
                                    " for a latent of " + std::to_string(f.size()) + " ids");
            const long long hop = w->a.hop();
            ends.resize(n_ids);
            long long c = 0;
            for (size_t i = 0; i < n_ids; i++) ends[i] = (c += f[i]) * hop;
            n = z->l->frames * hop;
        }
        *out = new sb200_prosody_stream{create_prosody_stream_breaks(w, w->device, w->sample_rate, n, ends.data(),
                                                                     pitch_per_id, n_ids, pitch, tempo, formant,
                                                                     volume_db_per_id, breaks_ms_per_id),
                                        v->v};
    });
}
int32_t sb200_prosody_stream_bounds(const sb200_prosody_stream* s, int64_t* out, size_t capacity, sb200_error* err) {
    return guarded(err, [&] {
        if (!s) throw Error(19, "null argument");
        const std::vector<long long>& b = s->p->bounds;
        if (s->p->n_total < 0 && s->p->brk.empty())
            throw Error(19, "prosody stream bounds: the stream was made without a pitch contour or breaks");
        if (capacity < b.size() || (!out && !b.empty()))
            throw Error(19, "prosody stream bounds: room for " + std::to_string(capacity) + " of " +
                                std::to_string(b.size()) + " ids");
        std::copy(b.begin(), b.end(), out);
    });
}
void sb200_prosody_stream_free(sb200_prosody_stream* s) { delete s; }
int32_t sb200_prosody_stream_profile(const sb200_prosody_stream* s, float* stretch_ms, float* pitch_ms) {
    if (!s) return 19;
    if (stretch_ms) *stretch_ms = s->p->last_ms[0];
    if (pitch_ms) *pitch_ms = s->p->last_ms[1];
    return 0;
}
int32_t sb200_prosody_stream_profile_formant(const sb200_prosody_stream* s, float* formant_ms) {
    if (!s) return 19;
    if (formant_ms) *formant_ms = s->p->last_fm_ms;
    return 0;
}
int32_t sb200_prosody_stream_profile_volume(const sb200_prosody_stream* s, float* volume_ms) {
    if (!s) return 19;
    if (volume_ms) *volume_ms = s->p->last_vol_ms;
    return 0;
}
int32_t sb200_prosody_stream_profile_breaks(const sb200_prosody_stream* s, float* break_ms) {
    if (!s) return 19;
    if (break_ms) *break_ms = s->p->last_brk_ms;
    return 0;
}

int32_t sb200_decode_chunks_resampled(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi,
                                      const int64_t* trim_lo_frames, const int64_t* trim_hi_frames, size_t n,
                                      int32_t fade, const float* gain, sb200_resampler* const* resamplers,
                                      const int32_t* last, int32_t format, void** outs, size_t* lens, sb200_error* err) {
    return sb200_decode_chunks_warped(v, zs, lo, hi, trim_lo_frames, trim_hi_frames, n, fade, gain, resamplers, nullptr,
                                      last, format, outs, lens, err);
}

int32_t sb200_decode_chunks_warped(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi,
                                   const int64_t* trim_lo_frames, const int64_t* trim_hi_frames, size_t n, int32_t fade,
                                   const float* gain, sb200_resampler* const* resamplers,
                                   sb200_prosody_stream* const* warps, const int32_t* last, int32_t format, void** outs,
                                   size_t* lens, sb200_error* err) {
    return sb200_decode_chunks_metered(v, zs, lo, hi, trim_lo_frames, trim_hi_frames, n, fade, gain, resamplers, warps,
                                       nullptr, last, format, outs, lens, err);
}

int32_t sb200_decode_chunks_metered(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi,
                                    const int64_t* trim_lo_frames, const int64_t* trim_hi_frames, size_t n, int32_t fade,
                                    const float* gain, sb200_resampler* const* resamplers,
                                    sb200_prosody_stream* const* warps, sb200_loudness_stream* const* meters,
                                    const int32_t* last, int32_t format, void** outs, size_t* lens, sb200_error* err) {
    return sb200_decode_chunks_marked(v, zs, lo, hi, trim_lo_frames, trim_hi_frames, n, fade, gain, resamplers, warps,
                                      meters, nullptr, last, format, outs, lens, err);
}

int32_t sb200_decode_chunks_marked(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi,
                                   const int64_t* trim_lo_frames, const int64_t* trim_hi_frames, size_t n, int32_t fade,
                                   const float* gain, sb200_resampler* const* resamplers,
                                   sb200_prosody_stream* const* warps, sb200_loudness_stream* const* meters,
                                   sb200_watermark_stream* const* marks, const int32_t* last, int32_t format, void** outs,
                                   size_t* lens, sb200_error* err) {
    return guarded(err, [&] {
        ChunkPass p = chunk_pass(zs, lo, hi, n, trim_lo_frames, trim_hi_frames, gain);
        if (n > 0 && (!resamplers || !outs || !lens)) throw Error(19, "null argument");
        for (size_t k = 0; k < n; k++) {
            p.chunks[k].rs = resamplers[k] ? resamplers[k]->r : nullptr;
            p.chunks[k].ps = warps && warps[k] ? warps[k]->p : nullptr;
            p.chunks[k].ls = meters && meters[k] ? meters[k]->s : nullptr;
            p.chunks[k].ws = marks && marks[k] ? marks[k]->w : nullptr;
            if (last) p.chunks[k].last = last[k];
        }
        p.fade = fade; p.resample = true; p.format = format;
        ChunkResult r;
        decode_chunks(v->v.get(), p, r);
        if (format == PCM_I16) copy_out(r.i16, outs, lens);
        else if (format == PCM_F32) copy_out(r.f32, outs, lens);
        else copy_out(r.g711, outs, lens);
    });
}

int32_t sb200_loudness_stream_create(sb200_voice* v, uint32_t out_rate, float target_lufs, float max_gain_db,
                                     sb200_loudness_stream** out, sb200_error* err) {
    return guarded(err, [&] {
        if (!v || !out) throw Error(19, "null argument");
        Voice* w = v->v.get();
        if (w->device < 0 || !w->emb)
            throw Error(19, "Failed to run model inference. Error: voice was loaded config-only (device -1); libsonata_b200 has no CPU path");
        long long rate = w->sample_rate;
        if (out_rate && out_rate != (uint32_t)w->sample_rate) {
            resample_ratio(w->sample_rate, out_rate, "loudness stream: ");
            rate = out_rate;
        }
        *out = new sb200_loudness_stream{create_loudness_stream(w, w->device, rate, target_lufs, max_gain_db), v->v};
    });
}
void sb200_loudness_stream_free(sb200_loudness_stream* s) { delete s; }

int32_t sb200_watermark_stream_create(sb200_voice* v, uint32_t out_rate, sb200_watermark_stream** out,
                                      sb200_error* err) {
    return guarded(err, [&] {
        if (!v || !out) throw Error(19, "null argument");
        *out = nullptr;
        Voice* w = v->v.get();
        long long rate = w->sample_rate;
        if (out_rate && out_rate != (uint32_t)w->sample_rate) {
            resample_ratio(w->sample_rate, out_rate, "watermark stream: ");
            rate = out_rate;
        }
        if (WatermarkStream* s = create_watermark_stream(w, rate)) *out = new sb200_watermark_stream{s, v->v};
    });
}
void sb200_watermark_stream_free(sb200_watermark_stream* s) { delete s; }
int32_t sb200_watermark_stream_profile(const sb200_watermark_stream* s, float* ms) {
    if (!s || !ms) return 19;
    *ms = s->w->last_ms;
    return 0;
}
int32_t sb200_loudness_stream_state(const sb200_loudness_stream* s, double* lufs, float* gain, int64_t* samples,
                                    int64_t* clipped, float* ms, sb200_error* err) {
    return guarded(err, [&] {
        if (!s) throw Error(19, "null argument");
        const LoudnessStream& m = *s->s;
        if (lufs) *lufs = m.lufs;
        if (gain) *gain = m.a;
        if (samples) *samples = m.samples;
        if (clipped) *clipped = m.clipped;
        if (ms) *ms = m.last_ms;
    });
}

// ---- introspection ----
int32_t sb200_job_debug_fetch(sb200_job* job, const char* name, size_t b, float** data, size_t* rows, size_t* cols, sb200_error* err) {
    return guarded(err, [&] {
        Job& j = *job->j;
        auto it = j.dbg.find(name);
        if (!j.ran || it == j.dbg.end()) throw Error(19, std::string("no debug buffer named `") + name + "` (was debug enabled before run?)");
        const int U = j.dbg_level[name];
        const int C = it->second.second;
        size_t r0, nr;
        if (U <= 0) { r0 = (size_t)j.xsegs[b].off; nr = (size_t)j.xsegs[b].len; }
        else { r0 = (size_t)j.frames.fsegs[b].off * U; nr = (size_t)j.frames.fsegs[b].len * U; }
        *data = (float*)malloc(nr * C * 4 + 4);
        SB_CUDA(cudaSetDevice(j.v->device));
        if (U < 0) {        // transposed [C][RX]: the utterance's columns of every row -> [C][len]
            SB_CUDA(cudaMemcpy2D(*data, nr * 4, it->second.first + r0, (size_t)j.RX * 4, nr * 4, (size_t)C, cudaMemcpyDeviceToHost));
            *rows = (size_t)C; *cols = nr;
            return;
        }
        SB_CUDA(cudaMemcpy(*data, it->second.first + r0 * C, nr * C * 4, cudaMemcpyDeviceToHost));
        *rows = nr; *cols = (size_t)C;
    });
}
int32_t sb200_job_debug_durations(sb200_job* job, size_t b, int32_t** cum, size_t* n, sb200_error* err) {
    return guarded(err, [&] {
        Job& j = *job->j;
        if (!j.ran) throw Error(19, "job not run");
        const size_t len = (size_t)j.xsegs[b].len;
        *cum = (int32_t*)malloc(len * 4 + 4);
        SB_CUDA(cudaSetDevice(j.v->device));
        SB_CUDA(cudaMemcpy(*cum, j.d_cum + j.xsegs[b].off, len * 4, cudaMemcpyDeviceToHost));
        *n = len;
    });
}
int32_t sb200_debug_decode_chunks(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi,
                                  size_t n, sb200_chunk_capture** caps, size_t* n_caps, sb200_error* err) {
    return guarded(err, [&] {
        if (!caps || !n_caps) throw Error(19, "null argument");
        *caps = nullptr; *n_caps = 0;
        ChunkPass p = chunk_pass(zs, lo, hi, n);
        p.debug = true;
        ChunkResult r;
        decode_chunks(v->v.get(), p, r);
        if (n == 0) return;
        // per chunk: the stages in order, then the waveform; records first, their data after them in the same block
        const size_t per = r.captures.size() + 1, count = n * per;
        size_t floats = 0;
        for (size_t k = 0; k < n; k++) {
            for (const ChunkCapture& c : r.captures) floats += c.rows[k].size();
            floats += r.f32[k].size();
        }
        char* block = static_cast<char*>(malloc(count * sizeof(sb200_chunk_capture) + floats * 4 + 4));
        if (!block) throw Error(19, "out of host memory");
        sb200_chunk_capture* rec = reinterpret_cast<sb200_chunk_capture*>(block);
        float* data = reinterpret_cast<float*>(block + count * sizeof(sb200_chunk_capture));
        const auto put = [&](const std::string& name, size_t k, const std::vector<float>& x, size_t cols) {
            memset(rec, 0, sizeof(*rec));
            strncpy(rec->name, name.c_str(), sizeof(rec->name) - 1);
            rec->chunk = k; rec->rows = x.size() / cols; rec->cols = cols; rec->data = data;
            std::copy(x.begin(), x.end(), data);
            data += x.size(); rec++;
        };
        for (size_t k = 0; k < n; k++) {
            for (const ChunkCapture& c : r.captures) put(c.name, k, c.rows[k], (size_t)c.cols);
            put("wav", k, r.f32[k], 1);
        }
        *caps = reinterpret_cast<sb200_chunk_capture*>(block);
        *n_caps = count;
    });
}
int32_t sb200_job_profile(const sb200_job* job, sb200_region_stat* out, int32_t cap) {
    const Job& j = *job->j;
    int32_t n = 0;
    for (const Region& r : j.regions) {
        if (n >= cap) break;
        memset(&out[n], 0, sizeof(out[n]));
        strncpy(out[n].name, r.name.c_str(), sizeof(out[n].name) - 1);
        out[n].ms = r.ms; out[n].flops = r.flops; out[n].bytes = r.bytes; out[n].launches = r.launches;
        n++;
    }
    return n;
}
static int32_t debug_plan(int32_t backend, int64_t rows, int32_t cin, int32_t cout, int32_t k, int32_t dil, int32_t act,
                          int32_t has_res, int32_t accumulate, int32_t* out16, int32_t* staging_bytes) {
    // Planning only: nothing is allocated or launched, so this also runs where there is no GPU (host-logic tests); tensor
    // maps are assumed available, as on any sm_90+ driver.  Buffers are described by stand-in addresses (the planners look
    // at alignment only).  Layer conventions as in sb200_debug_conv / the engine's ResBlock and flow layers.
    if (!out16 || cin <= 0 || cout <= 0 || k <= 0 || k > SB_MAX_TAPS || dil <= 0 || rows <= 0) return 19;
    static float anchor[64];
    float* const stand_in = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(anchor) + 127) & ~(uintptr_t)127);
    ConvW w = conv_layout(cin, cout, centred_taps(k, dil), false);
    w.w = w.bias = w.wtf = stand_in;
    w.tc_nt = tc_tile_for(cout);
    w.wtc = w.tc_nt ? stand_in : nullptr;
    const int R = (int)((rows + 255) / 256 * 256);
    ConvCall c;
    c.in_slope = 0.1f; c.act = act; c.res = has_res ? stand_in : nullptr; c.ldres = cout;
    c.y0 = c.y1 = stand_in; c.ldy0 = c.ldy1 = act == ACT_GATE ? cout / 2 : cout; c.acc0 = c.acc1 = accumulate;
    const ConvArgs p = conv_args(w, stand_in, cin, RowMap{nullptr, R, 1, R}, c);
    const bool ok = backend == 2 ? conv_tf_plan_info(p, out16) : conv_tc_plan_info(p, out16, staging_bytes);
    return ok ? 0 : 19;
}
int32_t sb200_debug_plan(int32_t backend, int64_t rows, int32_t cin, int32_t cout, int32_t k, int32_t dil, int32_t act,
                         int32_t has_res, int32_t accumulate, int32_t* out16) {
    return debug_plan(backend, rows, cin, cout, k, dil, act, has_res, accumulate, out16, nullptr);
}
int32_t sb200_debug_plan_staging(int64_t rows, int32_t cin, int32_t cout, int32_t k, int32_t dil, int32_t act,
                                 int32_t has_res, int32_t accumulate, int32_t* staging_bytes) {
    int32_t out16[16];
    if (!staging_bytes) return 19;
    return debug_plan(1, rows, cin, cout, k, dil, act, has_res, accumulate, out16, staging_bytes);
}

int32_t sb200_debug_conv_grid_cap(int32_t cap) {
    const int32_t old = g_conv_tc_grid_cap;
    g_conv_tc_grid_cap = cap > 0 ? cap : 0;
    return old;
}

int32_t sb200_debug_conv_ex(int32_t device, int32_t backend, const float* x, int32_t rows, int32_t cin, const float* w,
                            const float* bias, int32_t cout, int32_t k, int32_t dil, float in_slope, int32_t act,
                            const float* res, float scale, const int32_t* seg_end, int32_t gran, int32_t seg_mul,
                            float* y0, int32_t acc0, int32_t split, float* y1, int32_t acc1, sb200_error* err) {
    return guarded(err, [&] {
        if (rows <= 0 || gran <= 0 || seg_mul <= 0 || !seg_end) throw Error(19, "debug conv: bad row map");
        if (split < 0 || split > cout) split = cout;
        if (split < cout && (act == ACT_GATE || !y1)) throw Error(19, "debug conv: a split output needs y1 and no gate");
        SB_CUDA(cudaSetDevice(device));
        Voice tmp; tmp.device = device;
        ConvW cw = debug_make_conv(tmp, w, bias, cout, cin, k, dil);
        const int R = (rows + 255) / 256 * 256;
        const int ycols = act == ACT_GATE ? cout / 2 : cout;
        const int ld0 = std::min(split, ycols), ld1 = cout - split;    // y0 [rows][ld0], y1 [rows][ld1]
        const int ngran = (R + gran - 1) / gran;
        std::vector<int> ends(ngran, 0);                                // granules past the caller's table: all gap rows
        for (int g = 0; g < ngran && g * gran < rows; g++) ends[g] = seg_end[g];
        DeviceBuffers d;
        float* dx = d.upload(x, (size_t)rows * cin, (size_t)R * cin);
        float* dy0 = ld0 > 0 ? d.upload(y0, (size_t)rows * ld0, (size_t)R * ld0) : nullptr;
        float* dy1 = ld1 > 0 ? d.upload(y1, (size_t)rows * ld1, (size_t)R * ld1) : nullptr;
        const float* dres = res ? d.upload(res, (size_t)rows * cout, (size_t)R * cout) : nullptr;
        const int* dend = d.upload(ends.data(), (size_t)ngran, (size_t)ngran);
        ConvCall c;
        c.in_slope = in_slope; c.act = act; c.scale = scale; c.res = dres; c.ldres = cout;
        c.y0 = dy0 ? dy0 : dy1; c.ldy0 = dy0 ? ld0 : ld1; c.acc0 = acc0; c.split = split;
        c.y1 = dy1 ? dy1 : dy0; c.ldy1 = dy1 ? ld1 : ld0; c.acc1 = acc1;
        if (res && getenv("SB200_DEBUG_RES_IS_X") && cin == cout) { c.res = dx; c.ldres = cin; }   // ResBlock aliasing (timing only)
        const ConvArgs p = conv_args(cw, dx, cin, RowMap{dend, gran, seg_mul, R}, c);
        if (backend == 2) {
            if (!try_launch_conv_tf(p, 0)) throw Error(19, "conv shape not supported by the tf32 chunk-flush backend");
        } else if (backend == 1) {
            if (!try_launch_conv_tc(p, 0)) throw Error(19, "conv shape not supported by the wgmma backend");
        } else launch_conv_simt(p, 0);
        SB_CUDA(cudaDeviceSynchronize());
        if (dy0) SB_CUDA(cudaMemcpy(y0, dy0, (size_t)rows * ld0 * 4, cudaMemcpyDeviceToHost));
        if (dy1) SB_CUDA(cudaMemcpy(y1, dy1, (size_t)rows * ld1 * 4, cudaMemcpyDeviceToHost));
    });
}

int32_t sb200_debug_resblock2_plan(int64_t rows, int32_t nbr, const int32_t* ks, const int32_t* dils, int32_t* out8) {
    if (!out8 || rows <= 0 || rows > (1 << 30)) return 19;
    static float anchor[64];
    float* const stand_in = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(anchor) + 127) & ~(uintptr_t)127);
    std::vector<ResBW> res;
    const bool ok = debug_stage(nbr, ks, dils, res, [&](int b, int cv) {
        ConvW w = conv_layout(64, 64, centred_taps(ks[b], dils[2 * b + cv]), false);
        w.w = w.bias = w.wtc = stand_in;
        w.tc_nt = tc_tile_for(64);
        return w;
    });
    return ok && resblock2_tc_plan(res, (int)rows, out8) ? 0 : 19;
}

int32_t sb200_debug_resblock2_stage(int32_t device, const float* x, int32_t rows, int32_t nbr, const int32_t* ks,
                                    const int32_t* dils, const float* w, const float* bias, const int32_t* seg_end,
                                    int32_t gran, int32_t seg_mul, float* y, sb200_error* err) {
    return guarded(err, [&] {
        if (rows <= 0 || gran <= 0 || seg_mul <= 0 || !seg_end || !x || !w || !bias || !y)
            throw Error(19, "debug resblock2 stage: bad arguments");
        SB_CUDA(cudaSetDevice(device));
        Voice tmp; tmp.device = device;
        std::vector<ResBW> res;
        size_t woff = 0;
        const bool ok = debug_stage(nbr, ks, dils, res, [&](int b, int cv) {
            const float* wb = w + woff;
            woff += (size_t)64 * 64 * ks[b];
            return debug_make_conv(tmp, wb, bias + (size_t)(2 * b + cv) * 64, 64, 64, ks[b], dils[2 * b + cv]);
        });
        if (!ok || !resblock2_tc_plan(res, rows, nullptr)) throw Error(19, "debug resblock2 stage: shape not supported");
        const int R = (rows + 255) / 256 * 256;
        const int ngran = (R + gran - 1) / gran;
        std::vector<int> ends(ngran, 0);
        for (int g = 0; g < ngran && g * gran < rows; g++) ends[g] = seg_end[g];
        DeviceBuffers d;
        const float* dx = d.upload(x, (size_t)rows * 64, (size_t)R * 64);
        float* dy = d.alloc<float>((size_t)R * 64);
        const int* dend = d.upload(ends.data(), (size_t)ngran, (size_t)ngran);
        launch_resblock2_tc(res, dx, dy, RowMap{dend, gran, seg_mul, R}, 0);
        SB_CUDA(cudaDeviceSynchronize());
        SB_CUDA(cudaMemcpy(y, dy, (size_t)rows * 64 * 4, cudaMemcpyDeviceToHost));
    });
}

int32_t sb200_debug_conv(int32_t device, int32_t backend, const float* x, int32_t rows, int32_t cin, const float* w,
                         const float* bias, int32_t cout, int32_t k, int32_t dil, float in_slope, int32_t act,
                         const float* res, float scale, int32_t accumulate, float* y, int32_t valid_rows,
                         sb200_error* err) {
    // one segment [0, valid_rows): a single granule spanning the whole (256-row padded) launch
    const int32_t R = (rows + 255) / 256 * 256;
    return sb200_debug_conv_ex(device, backend, x, rows, cin, w, bias, cout, k, dil, in_slope, act, res, scale, &valid_rows,
                               R, 1, y, accumulate, cout, nullptr, accumulate, err);
}

int32_t sb200_debug_spline(int32_t device, const float* h29, int32_t ldh, float* z, int32_t rows, int32_t tcol,
                           int32_t valid_rows, sb200_error* err) {
    return guarded(err, [&] {
        if (rows <= 0 || ldh < 29 || (tcol != 0 && tcol != 1) || valid_rows < 0 || valid_rows > rows)
            throw Error(19, "debug spline: bad arguments");
        SB_CUDA(cudaSetDevice(device));
        const int R = (rows + 255) / 256 * 256;                          // one granule spanning the padded launch
        DeviceBuffers d;
        const float* dh = d.upload(h29, (size_t)rows * ldh, (size_t)R * ldh);
        float* dz = d.upload(z, (size_t)rows * 2, (size_t)R * 2);
        const int* dend = d.upload(&valid_rows, 1, 1);
        launch_spline(dh, ldh, dz, tcol, 10, 1.f, RowMap{dend, R, 1, R}, 0);
        SB_CUDA(cudaDeviceSynchronize());
        SB_CUDA(cudaMemcpy(z, dz, (size_t)rows * 2 * 4, cudaMemcpyDeviceToHost));
    });
}

int32_t sb200_debug_durations(int32_t device, const float* z, int32_t rows, const int32_t* seg_off, const int32_t* seg_len,
                              int32_t nseg, float m0, float logs0, float length_scale, float* logw, int32_t* cum,
                              int32_t* y_len, sb200_error* err) {
    return guarded(err, [&] {
        if (rows <= 0 || nseg <= 0 || !seg_off || !seg_len) throw Error(19, "debug durations: bad arguments");
        std::vector<SegInfo> segs(nseg);
        for (int b = 0; b < nseg; b++) {
            if (seg_off[b] < 0 || seg_len[b] < 0 || (long long)seg_off[b] + seg_len[b] > rows)
                throw Error(19, "debug durations: segment outside the rows");
            segs[b] = SegInfo{seg_off[b], seg_len[b]};
        }
        SB_CUDA(cudaSetDevice(device));
        const std::vector<float> scales(nseg, length_scale);
        DeviceBuffers d;
        const float* dscale = d.upload(scales.data(), (size_t)nseg, (size_t)nseg);
        const float* dz = d.upload(z, (size_t)rows * 2, (size_t)rows * 2);
        float* dlogw = d.upload(logw, (size_t)rows, (size_t)rows);
        int* dcum = d.upload(cum, (size_t)rows, (size_t)rows);
        int* dylen = d.alloc<int>((size_t)nseg);
        const SegInfo* dseg = d.upload(segs.data(), (size_t)nseg, (size_t)nseg);
        launch_durations(dz, m0, logs0, dscale, dseg, nseg, dlogw, dcum, dylen, 0);
        SB_CUDA(cudaDeviceSynchronize());
        SB_CUDA(cudaMemcpy(logw, dlogw, (size_t)rows * 4, cudaMemcpyDeviceToHost));
        SB_CUDA(cudaMemcpy(cum, dcum, (size_t)rows * 4, cudaMemcpyDeviceToHost));
        SB_CUDA(cudaMemcpy(y_len, dylen, (size_t)nseg * 4, cudaMemcpyDeviceToHost));
    });
}

int32_t sb200_debug_fit(int32_t device, const float* w, size_t n, const int32_t* frames, const int64_t* first,
                        const int64_t* end, const int64_t* budget, size_t n_spans, float* factor, float* u_out,
                        int64_t* frames_out, sb200_error* err) {
    return guarded(err, [&] {
        if (n == 0 || n > (size_t)INT_MAX || !w || (n_spans && (!first || !end || !budget)))
            throw Error(19, "debug fit: bad arguments");
        std::vector<FitSpan> spans(n_spans);
        for (size_t k = 0; k < n_spans; k++) {
            if (!(first[k] >= 0 && first[k] < end[k] && end[k] <= (int64_t)n))
                throw Error(19, "debug fit: span " + std::to_string(k) + " is not a non-empty range of the ids");
            spans[k] = FitSpan{(int)first[k], (int)(end[k] - first[k]), 0, (long long)budget[k]};
        }
        SB_CUDA(cudaSetDevice(device));
        std::vector<float> ones(n, 1.f);
        DeviceBuffers d;
        float* dw = d.upload(w, n, n);
        const int* df = frames ? d.upload(frames, n, n) : nullptr;
        float* dfac = d.upload(ones.data(), n, n);
        float* du = d.alloc<float>(std::max<size_t>(n_spans, 1));
        long long* dfr = d.alloc<long long>(std::max<size_t>(n_spans, 1));
        const FitSpan* ds = n_spans ? d.upload(spans.data(), n_spans, n_spans) : nullptr;
        launch_fit(ds, (int)n_spans, nullptr, 0.f, 0.f, nullptr, nullptr, df, dw, dfac, du, dfr, 0);
        SB_CUDA(cudaDeviceSynchronize());
        if (factor) SB_CUDA(cudaMemcpy(factor, dfac, n * 4, cudaMemcpyDeviceToHost));
        if (n_spans && u_out) SB_CUDA(cudaMemcpy(u_out, du, n_spans * 4, cudaMemcpyDeviceToHost));
        if (n_spans && frames_out) SB_CUDA(cudaMemcpy(frames_out, dfr, n_spans * 8, cudaMemcpyDeviceToHost));
    });
}

int32_t sb200_debug_resample_filter(int32_t in_rate, int32_t out_rate, float* taps, size_t cap, int32_t* up,
                                    int32_t* down) {
    try {
        const ResampleFilter f = resample_ratio(in_rate, out_rate, "");
        if (up) *up = f.up;
        if (down) *down = f.down;
        if (taps && cap >= (size_t)(2 * f.H + 1)) {
            const std::vector<float> h = resample_taps(f.up, f.down);
            std::copy(h.begin(), h.end(), taps);
        }
        return 0;
    } catch (const Error& e) {
        return e.code;
    }
}

int32_t sb200_debug_resample_emit(int32_t in_rate, int32_t out_rate, const int64_t* chunk_lens, size_t n,
                                  int64_t* emitted) {
    try {
        if (!chunk_lens || !emitted) return 19;
        const ResampleFilter f = resample_ratio(in_rate, out_rate, "");
        long long consumed = 0, done = 0;
        for (size_t k = 0; k < n; k++) {
            if (chunk_lens[k] < 0) return 19;
            consumed += chunk_lens[k];
            const long long end = resample_emit_end(f, consumed, k + 1 == n);
            emitted[k] = end - done;
            done = end;
        }
        return 0;
    } catch (const Error& e) {
        return e.code;
    }
}

int32_t sb200_debug_resample(int32_t device, const float* x, size_t n, int32_t in_rate, int32_t out_rate, float* y,
                             sb200_error* err) {
    return guarded(err, [&] {
        if (!x || !y || n == 0 || n > (size_t)INT32_MAX) throw Error(19, "debug resample: bad arguments");
        const ResampleFilter f = resample_ratio(in_rate, out_rate, "");
        const std::vector<float> t = resample_phase_major(resample_taps(f.up, f.down), f.up, f.K);
        SB_CUDA(cudaSetDevice(device));
        OutputPlan o;
        o.rp.add(&f, (long long)n);
        HookStage h(o, x, n, t);
        SB_CUDA(cudaMemcpy(y, h.out.buf, (size_t)o.rp.total * 4, cudaMemcpyDeviceToHost));
    });
}

int32_t sb200_debug_loudness_filter(int32_t rate, double* coeffs) {
    try {
        if (!coeffs) return 19;
        LoudSeg s{};
        loudness_design(rate, s);
        std::copy(s.k, s.k + 10, coeffs);
        return 0;
    } catch (const Error& e) {
        return e.code;
    }
}

int32_t sb200_debug_loudness(int32_t device, const float* x, size_t n, int32_t rate, double* lufs, sb200_error* err) {
    return guarded(err, [&] {
        if (!x || !lufs || n == 0) throw Error(19, "debug loudness: bad arguments");
        LoudSeg s{};
        loudness_design(rate, s);
        s.off = 0; s.n = (long long)n; s.c0 = 0; s.target = NAN;
        OutputPlan o;
        o.lp.segs.push_back(s);
        o.lp.chunks = ((long long)n + s.S - 1) / s.S;
        SB_CUDA(cudaSetDevice(device));
        HookStage h(o, x, n);
        *lufs = h.b.lufs.h[0];
    });
}

int32_t sb200_debug_loudness_stream(int32_t device, const float* x, const size_t* chunk_lens, size_t n_chunks,
                                    int32_t rate, float target_lufs, float max_gain_db, float* y, double* lufs_steps,
                                    float* gain_steps, int64_t* clipped, sb200_error* err) {
    return guarded(err, [&] {
        if ((n_chunks && (!chunk_lens || !y)) || !lufs_steps || !gain_steps || !clipped)
            throw Error(19, "debug loudness stream: bad arguments");
        size_t total = 0;
        for (size_t c = 0; c < n_chunks; c++) total += chunk_lens[c];
        if (total && !x) throw Error(19, "debug loudness stream: bad arguments");
        SB_CUDA(cudaSetDevice(device));
        std::unique_ptr<LoudnessStream> m(create_loudness_stream(nullptr, device, rate, target_lufs, max_gain_db));
        loudness_stream_steps(*m, (long long)total, "debug loudness stream: ");
        // chunk by chunk, each in its own pass, as passes feed a meter
        size_t off = 0;
        for (size_t c = 0; c < n_chunks; c++) {
            ChunkSpec spec;
            spec.ls = m.get();
            OutputPlan o = plan_chunk_output({spec}, {(long long)chunk_lens[c]}, false);
            HookStage h(o, x + off, chunk_lens[c]);
            if (chunk_lens[c]) SB_CUDA(cudaMemcpy(y + off, h.b.in, chunk_lens[c] * 4, cudaMemcpyDeviceToHost));
            std::copy(h.b.mlufs.h, h.b.mlufs.h + o.mp.steps[0], lufs_steps + m->steps);
            std::copy(h.b.mgains.h, h.b.mgains.h + o.mp.steps[0], gain_steps + m->steps);
            advance_streams(o, h.b, Profile());
            off += chunk_lens[c];
        }
        *clipped = m->clipped;
    });
}

int32_t sb200_debug_prosody_plan(int32_t rate, int64_t n, float pitch, float tempo, int64_t* shape6, int64_t* positions,
                                 size_t cap) {
    try {
        if (!shape6 || n < 0) return 19;
        check_prosody(&pitch, &tempo, 1);
        const ProsodyShape s = prosody_shape(rate, n, pitch, tempo);
        const int64_t out[6] = {s.Hs, s.N, s.D, s.n1, s.n2, s.F};
        std::copy(out, out + 6, shape6);
        for (int k = 0; positions && k < s.F && (size_t)k < cap; k++) positions[k] = prosody_analysis(s.Hs, s.alpha, k);
        return 0;
    } catch (const Error& e) {
        return e.code;
    }
}

namespace {
// A prosody hook's results: the output, every frame's offset and the stretched signal (the scratch when the pitch stage
// follows, else the output itself).
void debug_prosody_out(const HookStage& h, const ProsodySeg& g, float* y, int32_t* offsets, float* stretched) {
    SB_CUDA(cudaMemcpy(y, h.b.py, (size_t)g.n2 * 4, cudaMemcpyDeviceToHost));
    if (offsets && g.F) SB_CUDA(cudaMemcpy(offsets, h.b.offsets, (size_t)g.F * 4, cudaMemcpyDeviceToHost));
    if (stretched && g.stretch)
        SB_CUDA(cudaMemcpy(stretched, g.pitch ? h.b.ps : h.b.py, (size_t)g.n1 * 4, cudaMemcpyDeviceToHost));
}
}  // namespace

int32_t sb200_debug_prosody(int32_t device, const float* x, size_t n, int32_t rate, float pitch, float tempo, float* y,
                            size_t cap, int32_t* offsets, size_t offsets_cap, float* stretched, size_t stretched_cap,
                            sb200_error* err) {
    return guarded(err, [&] {
        if (!x || !y || n == 0 || n > (size_t)INT32_MAX) throw Error(19, "debug prosody: bad arguments");
        check_prosody(&pitch, &tempo, 1);
        OutputPlan p;
        p.pp.add(prosody_shape(rate, (long long)n, pitch, tempo), 0, (long long)n);
        const ProsodySeg& g = p.pp.segs[0];
        if ((size_t)g.n2 > cap || (offsets && (size_t)g.F > offsets_cap) ||
            (stretched && g.stretch && (size_t)g.n1 > stretched_cap))
            throw Error(19, "debug prosody: a destination is too small for the result");
        SB_CUDA(cudaSetDevice(device));
        HookStage h(p, x, n);
        debug_prosody_out(h, g, y, offsets, stretched);
    });
}

int32_t sb200_debug_prosody_contour_plan(int32_t rate, int64_t n, const int64_t* ends, const float* ratios, size_t n_ids,
                                         float tempo, int64_t* shape6, int64_t* positions, size_t cap, int64_t* bounds) {
    try {
        if (!shape6 || !ends || !ratios || n_ids == 0 || n <= 0) return 19;
        const size_t offs[2] = {0, n_ids};
        check_pitch_contour(ratios, offs, 1, nullptr);
        check_prosody(nullptr, &tempo, 1);
        std::vector<ContourPiece> pc;
        const ProsodyShape s = prosody_contour_plan(rate, n, reinterpret_cast<const long long*>(ends), ratios, n_ids, NAN,
                                                    tempo, pc, reinterpret_cast<long long*>(bounds));
        const int64_t out[6] = {s.Hs, s.N, s.D, s.n1, s.n2, s.F};
        std::copy(out, out + 6, shape6);
        // the positions as the offset chain computes them, with the piece carried from frame to frame
        for (int k = 0; positions && k < s.F && (size_t)k < cap; k++) {
            if (pc.empty()) { positions[k] = prosody_analysis(s.Hs, s.alpha, k); continue; }
            size_t r = 0;
            while (r + 2 < pc.size() && (double)((long long)k * s.Hs) >= pc[r + 1].S) r++;
            positions[k] = (long long)std::floor(pc[r].B + ((double)((long long)k * s.Hs) - pc[r].S) / pc[r].alpha + 0.5);
        }
        return 0;
    } catch (const Error& e) {
        return e.code;
    }
}

int32_t sb200_debug_prosody_contour(int32_t device, const float* x, size_t n, int32_t rate, const int64_t* ends,
                                    const float* ratios, size_t n_ids, float tempo, float* y, size_t cap,
                                    int32_t* offsets, size_t offsets_cap, float* stretched, size_t stretched_cap,
                                    sb200_error* err) {
    return guarded(err, [&] {
        if (!x || !y || !ends || !ratios || n_ids == 0 || n == 0 || n > (size_t)INT32_MAX)
            throw Error(19, "debug prosody contour: bad arguments");
        const size_t offs[2] = {0, n_ids};
        check_pitch_contour(ratios, offs, 1, nullptr);
        check_prosody(nullptr, &tempo, 1);
        std::vector<ContourPiece> pc;
        OutputPlan p;
        p.pp.add(prosody_contour_plan(rate, (long long)n, reinterpret_cast<const long long*>(ends), ratios, n_ids, NAN,
                                      tempo, pc, nullptr),
                 0, (long long)n, &pc);
        const ProsodySeg& g = p.pp.segs[0];
        if ((size_t)g.n2 > cap || (offsets && (size_t)g.F > offsets_cap) ||
            (stretched && g.stretch && (size_t)g.n1 > stretched_cap))
            throw Error(19, "debug prosody contour: a destination is too small for the result");
        SB_CUDA(cudaSetDevice(device));
        HookStage h(p, x, n);
        debug_prosody_out(h, g, y, offsets, stretched);
    });
}

int32_t sb200_debug_formant(int32_t device, const float* x, size_t n, int32_t rate, float pitch, float tempo,
                            const int64_t* ends, const float* ratios, size_t n_ids, float phi, float* pre, float* y,
                            size_t cap, int64_t* n2_out, sb200_error* err) {
    return guarded(err, [&] {
        if (!x || !pre || !y || n == 0 || n > (size_t)INT32_MAX || (n_ids && (!ends || !ratios)))
            throw Error(19, "debug formant: bad arguments");
        check_prosody(&pitch, &tempo, 1);
        check_formants(&phi, 1);
        const size_t offs[2] = {0, n_ids};
        if (n_ids) check_pitch_contour(ratios, offs, 1, &pitch);
        std::vector<ContourPiece> pc;
        ProsodyPlan p;
        p.add(n_ids ? prosody_contour_plan(rate, (long long)n, reinterpret_cast<const long long*>(ends), ratios, n_ids,
                                           NAN, tempo, pc, nullptr)
                    : prosody_shape(rate, (long long)n, pitch, tempo),
              0, (long long)n, &pc);
        const ProsodySeg& g = p.segs[0];
        OutputPlan o;
        if (g.stretch || g.pitch) o.pp = p;
        if (formant_asks(g.n2, phi, g.p, p.pieces.data() + g.c_off, g.c_n)) {
            o.fp.add(rate, 0, g.n2, phi, g.p, g.c_off, g.c_n);
            o.fp.total = g.n2;
        }
        if ((size_t)g.n2 > cap) throw Error(19, "debug formant: a destination is too small for the result");
        SB_CUDA(cudaSetDevice(device));
        HookStage h(o, x, n);
        // the pitch stage's output and the formant stage's
        const float* before = o.pp.segs.empty() ? h.b.in : h.b.py;
        SB_CUDA(cudaMemcpy(pre, before, (size_t)g.n2 * 4, cudaMemcpyDeviceToHost));
        SB_CUDA(cudaMemcpy(y, o.fp.segs.empty() ? before : h.b.fy, (size_t)g.n2 * 4, cudaMemcpyDeviceToHost));
        if (n2_out) *n2_out = g.n2;
    });
}

int32_t sb200_debug_volume(int32_t device, const float* x, size_t n, const int64_t* ends, const float* levels,
                           size_t n_ids, int32_t rate, float* y, sb200_error* err) {
    return guarded(err, [&] {
        if ((n && (!x || !y)) || (n_ids && (!ends || !levels)) || rate < 200)
            throw Error(19, "debug volume: bad arguments");
        const size_t offs[2] = {0, n_ids};
        check_volume_contour(levels, offs, 1, false);
        const std::vector<VolumePiece> pc =
            volume_pieces(reinterpret_cast<const long long*>(ends), levels, n_ids, (long long)n);
        OutputPlan o;
        if (!pc.empty()) o.vp.add(0, (long long)n, 0, volume_half(rate), pc);
        SB_CUDA(cudaSetDevice(device));
        HookStage h(o, x, n);
        if (n) SB_CUDA(cudaMemcpy(y, h.b.in, n * 4, cudaMemcpyDeviceToHost));
    });
}

int32_t sb200_debug_watermark(const float* x, size_t n, int32_t rate, const sb200_watermark* wm, float* y,
                              sb200_error* err) {
    return guarded(err, [&] {
        if ((n && (!x || !y)) || !wm || rate < 8000 || rate > 48000) throw Error(19, "debug watermark: bad arguments");
        check_watermark(wm->payload, wm->strength_db);
        DeviceBuffers d;
        signed char* chips = build_watermark_chips(wm->key);
        d.ptrs.push_back(chips);
        OutputPlan o;
        o.wp.add(Watermark{wm->key, wm->payload, wm->strength_db, chips}, 0, (long long)n, rate);
        o.wp.total = (long long)n;
        HookStage h(o, x, n);
        if (n) SB_CUDA(cudaMemcpy(y, h.out.buf, n * 4, cudaMemcpyDeviceToHost));
    });
}

int32_t sb200_debug_breaks(int32_t device, const float* x, size_t n, const int64_t* ends, const float* ms, size_t n_ids,
                           int32_t rate, float* y, size_t cap, int64_t* n_out, sb200_error* err) {
    return guarded(err, [&] {
        if ((n && !x) || (n_ids && (!ends || !ms)) || !n_out || rate < 200)
            throw Error(19, "debug breaks: bad arguments");
        const size_t offs[2] = {0, n_ids};
        check_breaks(ms, offs, 1, false);
        const std::vector<BreakPiece> bk =
            break_plan(reinterpret_cast<const long long*>(ends), ms, n_ids, (long long)n, rate, "");
        const long long total = (long long)n + (bk.empty() ? 0 : bk.back().D);
        *n_out = total;
        if ((size_t)total > cap || (total && !y))
            throw Error(19, "debug breaks: the destination holds " + std::to_string(cap) + " samples, the result has " +
                                std::to_string(total));
        OutputPlan o;
        if (!bk.empty()) o.bp.add(0, (long long)n, 0, 0, total, volume_half(rate), bk);
        SB_CUDA(cudaSetDevice(device));
        HookStage h(o, x, n);
        if (total) SB_CUDA(cudaMemcpy(y, h.out.buf, (size_t)total * 4, cudaMemcpyDeviceToHost));
    });
}

int32_t sb200_debug_prosody_stream_plan(int32_t rate, float pitch, float tempo, const int64_t* chunk_lens, size_t n_chunks,
                                        int64_t* emitted) {
    try {
        if (n_chunks > 0 && (!chunk_lens || !emitted)) return 19;
        const std::vector<long long> e =
            prosody_stream_plan(rate, pitch, tempo, reinterpret_cast<const long long*>(chunk_lens), n_chunks);
        std::copy(e.begin(), e.end(), emitted);
        return 0;
    } catch (const Error& e) {
        return e.code;
    }
}

int32_t sb200_debug_prosody_contour_stream_plan(int32_t rate, int64_t n, const int64_t* ends, const float* ratios,
                                                size_t n_ids, float tempo, const int64_t* chunk_lens, size_t n_chunks,
                                                int64_t* counts) {
    try {
        if ((n_chunks > 0 && (!chunk_lens || !counts)) || (n_ids > 0 && (!ends || !ratios))) return 19;
        ProsodyStream ps;
        prosody_stream_init_contour(ps, rate, n, reinterpret_cast<const long long*>(ends), ratios, n_ids, tempo);
        const std::vector<long long> c =
            prosody_stream_counts(ps, reinterpret_cast<const long long*>(chunk_lens), n_chunks);
        std::copy(c.begin(), c.end(), counts);
        return 0;
    } catch (const Error& e) {
        return e.code;
    }
}

namespace {
// Pushes x through the fresh stream ps chunk by chunk as one-segment passes: `whole` is the whole signal's shape and
// `counts` what the stream emits per chunk (prosody_stream_counts' first column every `stride` entries), checked
// against the destinations before any device work.  A formant stream's stage runs after its pitch stage, or on the
// chunk itself without one.
void debug_push_stream(ProsodyStream& ps, const ProsodyShape& whole, const std::vector<long long>& counts, size_t stride,
                       const float* x, const int64_t* chunk_lens, size_t n_chunks, float* y, size_t cap, int64_t* lens,
                       int32_t* offsets, size_t offsets_cap) {
    long long out_total = 0;
    for (size_t k = 0; k < n_chunks; k++) out_total += counts[stride * k];
    if ((size_t)out_total > cap) throw Error(19, "debug prosody stream: the destination is too small for the result");
    if (offsets && ps.sh.stretch && (size_t)whole.F > offsets_cap)
        throw Error(19, "debug prosody stream: the offsets destination is too small");
    long long in_at = 0, out_at = 0;
    for (size_t k = 0; k < n_chunks; k++) {
        ChunkSpec c;
        c.ps = &ps; c.last = k + 1 == n_chunks;
        OutputPlan o = plan_chunk_output({c}, {(long long)chunk_lens[k]}, false);
        HookStage h(o, x + in_at, (size_t)chunk_lens[k]);
        const long long m = o.n_res[0];
        const ProsodyStep& t = o.steps[0];
        SB_CUDA(cudaMemcpy(y + out_at, o.fp.segs.empty() ? h.b.py : h.b.fy, (size_t)m * 4, cudaMemcpyDeviceToHost));
        if (offsets && t.k1 > t.k0)
            SB_CUDA(cudaMemcpy(offsets + t.k0, h.b.offsets + 2, (size_t)(t.k1 - t.k0) * 4, cudaMemcpyDeviceToHost));
        lens[k] = m;
        out_at += m; in_at += chunk_lens[k];
        advance_streams(o, h.b, Profile());
    }
}
}  // namespace

int32_t sb200_debug_prosody_contour_stream(int32_t device, const float* x, const int64_t* chunk_lens, size_t n_chunks,
                                           int32_t rate, const int64_t* ends, const float* ratios, size_t n_ids,
                                           float tempo, float* y, size_t cap, int64_t* lens, int32_t* offsets,
                                           size_t offsets_cap, sb200_error* err) {
    return guarded(err, [&] {
        if (!x || !chunk_lens || !y || !lens || n_chunks == 0 || !ends || !ratios || n_ids == 0)
            throw Error(19, "debug prosody contour stream: bad arguments");
        long long total = 0;
        for (size_t k = 0; k < n_chunks; k++) {
            if (chunk_lens[k] < 0) throw Error(19, "debug prosody contour stream: negative chunk length");
            total += chunk_lens[k];
        }
        const long long* e = reinterpret_cast<const long long*>(ends);
        ProsodyStream host;
        prosody_stream_init_contour(host, rate, total, e, ratios, n_ids, tempo);
        const std::vector<long long> counts =
            prosody_stream_counts(host, reinterpret_cast<const long long*>(chunk_lens), n_chunks);
        std::vector<ContourPiece> pc;
        const ProsodyShape whole = prosody_contour_plan(rate, total, e, ratios, n_ids, NAN, tempo, pc, nullptr);
        SB_CUDA(cudaSetDevice(device));
        std::unique_ptr<ProsodyStream> ps(create_prosody_stream_contour(nullptr, device, rate, total, e, ratios, n_ids,
                                                                        tempo));
        debug_push_stream(*ps, whole, counts, 5, x, chunk_lens, n_chunks, y, cap, lens, offsets, offsets_cap);
    });
}

int32_t sb200_debug_prosody_stream(int32_t device, const float* x, const int64_t* chunk_lens, size_t n_chunks,
                                   int32_t rate, float pitch, float tempo, float* y, size_t cap, int64_t* lens,
                                   int32_t* offsets, size_t offsets_cap, sb200_error* err) {
    return guarded(err, [&] {
        if (!x || !chunk_lens || !y || !lens || n_chunks == 0) throw Error(19, "debug prosody stream: bad arguments");
        long long total = 0;
        for (size_t k = 0; k < n_chunks; k++) {
            if (chunk_lens[k] < 0) throw Error(19, "debug prosody stream: negative chunk length");
            total += chunk_lens[k];
        }
        ProsodyStream host;
        prosody_stream_init(host, rate, pitch, tempo);
        const std::vector<long long> counts =
            prosody_stream_counts(host, reinterpret_cast<const long long*>(chunk_lens), n_chunks);
        const ProsodyShape whole = prosody_shape(rate, total, pitch, tempo);
        SB_CUDA(cudaSetDevice(device));
        std::unique_ptr<ProsodyStream> ps(create_prosody_stream(nullptr, device, rate, pitch, tempo));
        debug_push_stream(*ps, whole, counts, 5, x, chunk_lens, n_chunks, y, cap, lens, offsets, offsets_cap);
    });
}

namespace {
// A fresh formant stream on the host (no device memory) for the debug hooks, and the whole signal's shape of n inputs.
ProsodyShape debug_formant_stream(ProsodyStream& ps, int32_t rate, long long n, float pitch, float tempo,
                                  const int64_t* ends, const float* ratios, size_t n_ids, float formant) {
    const long long* e = reinterpret_cast<const long long*>(ends);
    prosody_stream_init_formant(ps, rate, n, e, n_ids ? ratios : nullptr, n_ids, pitch, tempo, formant);
    if (!n_ids) return prosody_shape(rate, n, pitch, tempo);
    std::vector<ContourPiece> pc;
    return prosody_contour_plan(rate, n, e, ratios, n_ids, NAN, tempo, pc, nullptr);
}
}  // namespace

int32_t sb200_debug_formant_stream_plan(int32_t rate, float pitch, float tempo, const int64_t* ends, const float* ratios,
                                        size_t n_ids, float formant, const int64_t* chunk_lens, size_t n_chunks,
                                        int64_t* emitted, sb200_error* err) {
    return guarded(err, [&] {
        if ((n_chunks > 0 && (!chunk_lens || !emitted)) || (n_ids > 0 && (!ends || !ratios)))
            throw Error(19, "debug formant stream plan: bad arguments");
        long long total = 0;
        for (size_t k = 0; k < n_chunks; k++) total += std::max<long long>(chunk_lens[k], 0);
        ProsodyStream ps;
        debug_formant_stream(ps, rate, total, pitch, tempo, ends, ratios, n_ids, formant);
        const std::vector<long long> e =
            formant_stream_counts(ps, reinterpret_cast<const long long*>(chunk_lens), n_chunks);
        std::copy(e.begin(), e.end(), emitted);
    });
}

int32_t sb200_debug_formant_stream(int32_t device, const float* x, const int64_t* chunk_lens, size_t n_chunks,
                                   int32_t rate, float pitch, float tempo, const int64_t* ends, const float* ratios,
                                   size_t n_ids, float formant, float* y, size_t cap, int64_t* lens, sb200_error* err) {
    return guarded(err, [&] {
        if (!x || !chunk_lens || !y || !lens || n_chunks == 0 || (n_ids > 0 && (!ends || !ratios)))
            throw Error(19, "debug formant stream: bad arguments");
        long long total = 0;
        for (size_t k = 0; k < n_chunks; k++) {
            if (chunk_lens[k] < 0) throw Error(19, "debug formant stream: negative chunk length");
            total += chunk_lens[k];
        }
        ProsodyStream host;
        const ProsodyShape whole = debug_formant_stream(host, rate, total, pitch, tempo, ends, ratios, n_ids, formant);
        const std::vector<long long> counts =
            formant_stream_counts(host, reinterpret_cast<const long long*>(chunk_lens), n_chunks);
        SB_CUDA(cudaSetDevice(device));
        std::unique_ptr<ProsodyStream> ps(create_prosody_stream_formant(
            nullptr, device, rate, n_ids ? total : -1, reinterpret_cast<const long long*>(ends),
            n_ids ? ratios : nullptr, n_ids, pitch, tempo, formant));
        debug_push_stream(*ps, whole, counts, 1, x, chunk_lens, n_chunks, y, cap, lens, nullptr, 0);
    });
}

int32_t sb200_debug_g711(int32_t device, int32_t law, const int16_t* x, size_t n, uint8_t* out, sb200_error* err) {
    return guarded(err, [&] {
        const int fmt = g711_format(law, "");
        if ((!x || !out) && n > 0) throw Error(19, "debug g711: null buffer");
        if (device < 0) {
            for (size_t i = 0; i < n; i++) out[i] = fmt == PCM_MULAW ? g711_ulaw(x[i]) : g711_alaw(x[i]);
            return;
        }
        if (n == 0) return;
        SB_CUDA(cudaSetDevice(device));
        DeviceBuffers d;
        const short* dx = d.upload(reinterpret_cast<const short*>(x), n, n);
        uint8_t* dy = d.alloc<uint8_t>(n);
        launch_g711(dx, (long long)n, fmt, dy, 0);
        SB_CUDA(cudaDeviceSynchronize());
        SB_CUDA(cudaMemcpy(out, dy, n, cudaMemcpyDeviceToHost));
    });
}

int32_t sb200_debug_speaker_blend(sb200_voice* v, const int64_t* speakers, const float* weights, size_t n, float* g,
                                  size_t g_cap, float* bias, size_t bias_cap, sb200_error* err) {
    return guarded(err, [&] {
        Voice& V = *v->v;
        const SpeakerBlend b = canonical_blend(V, reinterpret_cast<const long long*>(speakers), weights, n, "");
        if (g_cap < (size_t)V.gin || bias_cap < (size_t)V.cond_rows)
            throw Error(19, "debug speaker blend: a destination is too small for the result");
        std::vector<float> gh, bh;
        debug_speaker_blend(V, b, gh, bh);
        std::copy(gh.begin(), gh.end(), g);
        std::copy(bh.begin(), bh.end(), bias);
    });
}

uint64_t sb200_launch_count(void) { return g_launch_count; }
int32_t sb200_set_backend(sb200_voice* v, int32_t backend) { int32_t p = v->v->backend; v->v->backend = backend; return p; }

}  // extern "C"
