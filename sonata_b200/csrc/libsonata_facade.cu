// libsonata C-ABI facade (drop-in boundary #2, SURVEY §8b): the eleven `libsonata*` symbols of
// crates/frontends/capi/libsonata.h:78-109 with identical struct layouts, implemented over the H100
// engine instead of sonata-synth + onnxruntime (reference implementation: capi/src/lib.rs:187-438).
//
// Differences, all at the edges of the hot path and all loud:
//   * `text` is taken as PHONEMES, one sentence per line: the espeak-ng front-end (SURVEY §2 row 8) is
//     outside this repository.  A Rust host keeps calling espeak and passes its output here.
//   * rate / pitch go through Sonic in the reference (CPU post-processing, §2 row 7): neutral values
//     (rate 10 -> 1.0x, pitch 50 -> 1.0x) are accepted, anything else yields a SYNTH_EVENT_ERROR with
//     OPERATION_ERROR.  volume (linear gain) and appended silence are honoured.
//   * the CUDA ordinal comes from $SONATA_B200_DEVICE (default 0).
// Event payloads are i16 LE PCM, peak-normalised per chunk exactly like AudioSamples::as_wave_bytes
// (audio/ops/src/samples.rs:51-78); realtime mode uses the reference chunk schedule (72, 3) with
// crossfade(42) (piper/src/lib.rs:765-913) and the chunk-size growth rule of synth/src/lib.rs:348-356.
// The whole post-path -- overlap trim, crossfade, volume gain, peak normalisation, 16-bit conversion -- runs on the
// DEVICE (kernels_misc.cu i16 kernels, bit-identical to the host arithmetic of the reference): a callback receives
// bytes that crossed PCIe once, as i16, through page-locked staging.
// The voice is reference-counted like the reference's Arc (capi/src/lib.rs:314,375): a non-blocking speak keeps it
// alive after libsonataUnloadSonataVoice.
#include "engine.h"
#include <cmath>
#include <cstring>
#include <memory>
#include <thread>

using namespace sb200;

extern "C" {

// ---- ABI types: same field order / widths as capi/libsonata.h:32-76 ----
typedef struct SonataVoice { std::shared_ptr<Voice> v; } SonataVoice;
typedef struct PiperSynthConfig { uint32_t speaker; float length_scale; float noise_scale; float noise_w; } PiperSynthConfig;
typedef struct ExternError { int32_t code; char* message; } ExternError;
typedef struct SynthesisEvent { int32_t event_type; ExternError* error_ptr; int64_t len; uint8_t* data; } SynthesisEvent;
typedef struct AudioInfo { uint32_t sample_rate; uint32_t num_channels; uint32_t sample_width; } AudioInfo;
typedef uint8_t (*SpeechSynthesisCallback)(SynthesisEvent);
typedef struct SynthesisParams {
    int32_t mode; uint8_t rate; uint8_t volume; uint8_t pitch; uint32_t appended_silence_ms;
    SpeechSynthesisCallback callback; uint8_t nonblocking;
} SynthesisParams;

}  // extern "C"

namespace {

enum { INVALID_SYNTHESIS_MODE = 16, FAILED_TO_LOAD_RESOURCE = 17, PHONEMIZATION_ERROR = 18, OPERATION_ERROR = 19,
       INVALID_UTF8_SEQUENCE = 20, UNKNOWN_ERROR = 21 };
enum { SYNTH_EVENT_SPEECH = 0, SYNTH_EVENT_FINISHED = 1, SYNTH_EVENT_ERROR = 2 };
enum { SYNTH_MODE_LAZY = 0, SYNTH_MODE_PARALLEL = 1, SYNTH_MODE_REALTIME = 2 };

char* dupstr(const std::string& s) { char* p = (char*)malloc(s.size() + 1); memcpy(p, s.c_str(), s.size() + 1); return p; }
void set_ok(ExternError* e) { if (e) { e->code = 0; e->message = nullptr; } }
void set_err(ExternError* e, int code, const std::string& m) { if (e) { e->code = code; e->message = dupstr(m); } }

template <typename F>
void guarded(ExternError* out, F&& f) {
    set_ok(out);
    try { f(); }
    catch (const Error& e) { set_err(out, e.code, e.what()); }
    catch (const std::exception& e) { set_err(out, UNKNOWN_ERROR, e.what()); }
    catch (...) { set_err(out, -1, "panic"); }
}

std::vector<std::string> split_sentences(const char* text) {
    if (!text) throw Error(INVALID_UTF8_SEQUENCE, "Invalid utf-8 input.");
    std::vector<std::string> out;
    std::string cur;
    for (const char* p = text;; p++) {
        if (*p == '\n' || *p == 0) {
            if (cur.find_first_not_of(" \t\r") != std::string::npos) out.push_back(cur);
            cur.clear();
            if (*p == 0) break;
        } else cur += *p;
    }
    return out;
}

// event carrying i16 PCM (+ appended silence as zero samples: zeros do not move the peak normalisation)
SynthesisEvent speech_event(const std::vector<int16_t>& pcm, size_t silence_samples) {
    const size_t n = pcm.size() + silence_samples;
    SynthesisEvent ev{SYNTH_EVENT_SPEECH, nullptr, (int64_t)(2 * n), (uint8_t*)malloc(2 * n + 2)};
    if (!pcm.empty()) memcpy(ev.data, pcm.data(), 2 * pcm.size());
    if (silence_samples) memset(ev.data + 2 * pcm.size(), 0, 2 * silence_samples);
    return ev;
}
SynthesisEvent error_event(int code, const std::string& m) {
    ExternError* e = (ExternError*)malloc(sizeof(ExternError));
    e->code = code; e->message = dupstr(m);
    return SynthesisEvent{SYNTH_EVENT_ERROR, e, 0, (uint8_t*)malloc(1)};
}
SynthesisEvent finished_event() { return SynthesisEvent{SYNTH_EVENT_FINISHED, nullptr, 0, (uint8_t*)malloc(1)}; }

// AudioOutputConfig::apply_to_raw_samples restricted to what is not Sonic (see header comment)
void check_output_config(const SynthesisParams& p) {
    const float rate = (p.rate / 100.0f) * (5.5f - 0.5f) + 0.5f, pitch = (p.pitch / 100.0f) * (1.5f - 0.5f) + 0.5f;
    if (fabsf(rate - 1.0f) > 1e-6f || fabsf(pitch - 1.0f) > 1e-6f)
        throw Error(OPERATION_ERROR, "Sonic Error: rate / pitch modification is CPU post-processing outside libsonata_b200 "
                                     "(use rate=10, pitch=50, and length_scale for speed)");
}
float gain_of(const SynthesisParams& p) { return p.volume / 100.0f; }
size_t silence_of(const SynthesisParams& p, int sample_rate) { return (size_t)p.appended_silence_ms * sample_rate / 1000; }

// one batched pass over the sentences; per-sentence peak-normalised PCM converted on the device
std::vector<std::vector<int16_t>> speak_sentences_pcm(Voice* v, const std::vector<std::string>& ph, float gain) {
    std::vector<long long> ids; std::vector<size_t> offs{0};
    for (auto& s : ph) { auto r = v->phonemes_to_ids(s.c_str()); ids.insert(ids.end(), r.begin(), r.end()); offs.push_back(ids.size()); }
    std::unique_ptr<Job> j(create_job(v, ids.data(), offs.data(), ph.size(), nullptr, nullptr, nullptr, false));
    j->run(nullptr, 0);
    std::vector<std::vector<int16_t>> out;
    job_pcm16(*j, gain, out);
    return out;
}

// returns false when the callback asked to stop
bool emit(const SynthesisParams& p, const std::vector<int16_t>& pcm, size_t silence) {
    return p.callback(speech_event(pcm, silence)) == 0;
}

void do_synthesize(Voice* v, const std::string& text, const SynthesisParams& p) {
    check_output_config(p);
    const std::vector<std::string> ph = split_sentences(text.c_str());
    const int sr = v->sample_rate;
    const float gain = gain_of(p);
    const size_t sil = silence_of(p, sr);
    if (p.mode == SYNTH_MODE_LAZY) {
        for (auto& s : ph) { auto w = speak_sentences_pcm(v, {s}, gain); if (!emit(p, w[0], sil)) return; }
    } else if (p.mode == SYNTH_MODE_PARALLEL) {
        if (!ph.empty()) { auto ws = speak_sentences_pcm(v, ph, gain); for (auto& w : ws) if (!emit(p, w, sil)) return; }
    } else if (p.mode == SYNTH_MODE_REALTIME) {
        long long chunk = 72; const long long pad = 3; long long produced = 0;
        for (auto& s : ph) {
            if (produced != 0) chunk = chunk * 1 * produced;                       // synth/src/lib.rs:348-356
            auto ids = v->phonemes_to_ids(s.c_str());
            std::unique_ptr<Latent> z(encode_latent(v, ids.data(), ids.size()));
            const long long frames = z->frames;
            long long n = 0;
            ChunkPass cp;                                                           // one chunk, leaving as i16
            cp.format = 1; cp.single = true;
            ChunkResult r;
            if (frames <= 2 * chunk + 2 * pad) {                                    // one-shot (piper :785)
                cp.chunks = {ChunkSpec{z.get(), 0, frames, 0, 0, gain}};
                decode_chunks(v, cp, r);
                n = 1; if (!emit(p, r.i16[0], 0)) return;
            } else {                                                                // AdaptiveMelChunker (piper :886-912)
                long long last = 0, step = 1; bool more = true;
                cp.fade = 42;                                                       // trim + crossfade(42)
                while (more) {
                    const long long cs = std::min<long long>(chunk * step, 1024);
                    const long long start = last == 0 ? 0 : last - 2 * pad, spad = last == 0 ? 0 : pad;
                    const long long cend = last + cs + pad;
                    long long end = cend, epad = pad;
                    if (frames - cend <= 44) { end = frames; epad = 0; more = false; }
                    step++; last = cend;
                    cp.chunks = {ChunkSpec{z.get(), start, end, spad, epad, gain}};
                    decode_chunks(v, cp, r);
                    n++; if (!emit(p, r.i16[0], 0)) return;
                }
            }
            produced += n;
            if (p.appended_silence_ms) { std::vector<int16_t> none; if (!emit(p, none, sil)) return; }
        }
    } else throw Error(INVALID_SYNTHESIS_MODE, "Invalid synthesis mode");
    p.callback(finished_event());
}

// whole-file peak normalisation like Audio::save_to_file -> to_i16_vec over the concatenated sentences
void write_wav_f32(const char* path, const float* s, size_t n, int sr) {
    std::vector<int16_t> pcm(n);
    if (n) {
        float mx = s[0], mn = s[0];
        for (size_t i = 1; i < n; i++) { mx = fmaxf(mx, s[i]); mn = fminf(mn, s[i]); }
        const float abs_max = fmaxf(fmaxf(fabsf(mx), fabsf(mn)), 1.1920929e-07f);
        const float scale = 32767.0f / abs_max;
        for (size_t i = 0; i < n; i++) pcm[i] = (int16_t)fminf(fmaxf(s[i] * scale, -32768.0f), 32767.0f);
    }
    FILE* f = fopen(path, "wb");
    if (!f) throw Error(OPERATION_ERROR, std::string("cannot open `") + path + "` for writing");
    const uint32_t bytes = (uint32_t)(2 * n), riff = 36 + bytes, fmt = 16, br = (uint32_t)sr * 2;
    const uint16_t pcmf = 1, ch = 1, ba = 2, bits = 16;
    fwrite("RIFF", 1, 4, f); fwrite(&riff, 4, 1, f); fwrite("WAVEfmt ", 1, 8, f); fwrite(&fmt, 4, 1, f);
    fwrite(&pcmf, 2, 1, f); fwrite(&ch, 2, 1, f); fwrite(&sr, 4, 1, f); fwrite(&br, 4, 1, f); fwrite(&ba, 2, 1, f);
    fwrite(&bits, 2, 1, f); fwrite("data", 1, 4, f); fwrite(&bytes, 4, 1, f); fwrite(pcm.data(), 1, bytes, f);
    fclose(f);
}

// f32 waveforms of one batched pass through the context's page-locked staging (speak-to-file: the file is normalised
// as a whole, so the per-sentence device conversion does not apply)
std::vector<std::vector<float>> speak_sentences_f32(Voice* v, const std::vector<std::string>& ph) {
    std::vector<long long> ids; std::vector<size_t> offs{0};
    for (auto& s : ph) { auto r = v->phonemes_to_ids(s.c_str()); ids.insert(ids.end(), r.begin(), r.end()); offs.push_back(ids.size()); }
    std::unique_ptr<Job> j(create_job(v, ids.data(), offs.data(), ph.size(), nullptr, nullptr, nullptr, false));
    j->run(nullptr, 0);
    Context& C = *j->ctx;
    const FrameLayout& l = j->frames;
    C.pin.reserve((size_t)l.total_samples * 4);
    float* all = C.pin.get<float>((size_t)l.total_samples);
    SB_CUDA(cudaMemcpyAsync(all, j->d_wav, (size_t)l.total_samples * 4, cudaMemcpyDeviceToHost, C.stream));
    SB_CUDA(cudaStreamSynchronize(C.stream));
    std::vector<std::vector<float>> out;
    for (size_t b = 0; b < ph.size(); b++)
        out.emplace_back(all + l.fsegs[b].out_off, all + l.fsegs[b].out_off + (size_t)j->y_len[b] * v->a.hop());
    return out;
}

}  // namespace

extern "C" {

void libsonataFreeString(int8_t* string_ptr) { free(string_ptr); }
void libsonataFreePiperSynthConfig(PiperSynthConfig* c) { free(c); }
void libsonataFreeSynthesisEvent(SynthesisEvent event) { if (event.error_ptr) free(event.error_ptr); free(event.data); }

SonataVoice* libsonataLoadVoiceFromConfigPath(const char* config_path_ptr, ExternError* out_error) {
    SonataVoice* r = nullptr;
    guarded(out_error, [&] {
        if (!config_path_ptr) throw Error(INVALID_UTF8_SEQUENCE, "Invalid utf-8 input.");
        const char* d = getenv("SONATA_B200_DEVICE");
        r = new SonataVoice{std::shared_ptr<Voice>(load_voice(config_path_ptr, d ? atoi(d) : 0))};
    });
    return r;
}
// drops this handle's reference; a synthesis still running on a worker thread keeps the voice alive until it returns
void libsonataUnloadSonataVoice(SonataVoice* voice_ptr) { delete voice_ptr; }

void libsonataGetAudioInfo(SonataVoice* voice_ptr, AudioInfo* info, ExternError* out_error) {
    guarded(out_error, [&] { info->sample_rate = (uint32_t)voice_ptr->v->sample_rate; info->num_channels = 1; info->sample_width = 2; });
}
PiperSynthConfig* libsonataGetPiperDefaultSynthConfig(SonataVoice* voice_ptr, ExternError* out_error) {
    PiperSynthConfig* c = nullptr;
    guarded(out_error, [&] {
        c = (PiperSynthConfig*)malloc(sizeof(PiperSynthConfig));
        const SynthConfig& f = voice_ptr->v->factory_cfg;      // speaker: Some(0) (piper/src/lib.rs:444-451)
        *c = PiperSynthConfig{0u, f.length_scale, f.noise_scale, f.noise_w};
    });
    return c;
}
void libsonataSetPiperSynthConfig(SonataVoice* voice_ptr, PiperSynthConfig c, ExternError* out_error) {
    guarded(out_error, [&] {   // capi always passes Some(speaker) (capi/src/lib.rs:175-184) -> unknown ids are errors
        Voice* v = voice_ptr->v.get();
        std::unique_lock<std::shared_mutex> g(v->cfg_mu);
        v->cfg.length_scale = c.length_scale; v->cfg.noise_scale = c.noise_scale; v->cfg.noise_w = c.noise_w;
        bool found = false;
        for (auto& kv : v->speaker_id_map) if (kv.second == (long long)c.speaker) found = true;
        if (!found) throw Error(OPERATION_ERROR, "No speaker was found with the given id `" + std::to_string(c.speaker) + "`");
        v->cfg.speaker = c.speaker; v->cfg.has_speaker = true;
    });
}

void libsonataSpeak(SonataVoice* voice_ptr, const char* text_ptr, SynthesisParams params, ExternError* out_error) {
    guarded(out_error, [&] {
        if (!text_ptr) throw Error(INVALID_UTF8_SEQUENCE, "Invalid utf-8 input.");
        std::shared_ptr<Voice> v = voice_ptr->v;
        const std::string text(text_ptr);
        if (params.nonblocking) {
            std::thread([v, text, params] {                      // callback fires on a foreign thread (capi :374-381);
                try { do_synthesize(v.get(), text, params); }    // the thread owns a reference to the voice
                catch (const Error& e) { params.callback(error_event(e.code, e.what())); }
                catch (const std::exception& e) { params.callback(error_event(UNKNOWN_ERROR, e.what())); }
                catch (...) { params.callback(error_event(UNKNOWN_ERROR, "unknown error")); }
            }).detach();
        } else {
            try { do_synthesize(v.get(), text, params); }
            catch (const Error& e) {
                if (e.code == INVALID_SYNTHESIS_MODE || e.code == INVALID_UTF8_SEQUENCE) throw;
                params.callback(error_event(e.code, e.what()));  // stream errors arrive as events (capi :428-432)
            }
        }
    });
}

uint8_t libsonataSpeakToFile(SonataVoice* voice_ptr, const char* text_ptr, SynthesisParams params,
                             const char* out_filename_ptr, ExternError* out_error) {
    uint8_t ok = 0;
    guarded(out_error, [&] {                                      // errors are swallowed into 0/1 (capi :331-335)
        try {
            if (!text_ptr || !out_filename_ptr) throw Error(INVALID_UTF8_SEQUENCE, "Invalid utf-8 input.");
            check_output_config(params);
            Voice* v = voice_ptr->v.get();
            auto ph = split_sentences(text_ptr);
            std::vector<float> all;
            const float vol = gain_of(params);
            if (!ph.empty()) for (auto& w : speak_sentences_f32(v, ph)) {
                w.resize(w.size() + silence_of(params, v->sample_rate), 0.f);
                for (float& x : w) x *= vol;
                all.insert(all.end(), w.begin(), w.end());
            }
            if (all.empty()) throw Error(OPERATION_ERROR, "No speech data to write");
            write_wav_f32(out_filename_ptr, all.data(), all.size(), v->sample_rate);
            ok = 1;
        } catch (const std::exception&) { ok = 0; }
    });
    return ok;
}

}  // extern "C"
