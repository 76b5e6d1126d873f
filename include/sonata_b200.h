/*
 * sonata_b200.h — C ABI of libsonata_b200.so: the H100-native replacement for the one hot path of
 * mush42/sonata, the Piper/VITS phoneme -> waveform synthesis that the reference delegates to
 * onnxruntime (`ort::Session::run`, crates/sonata/models/piper/src/lib.rs:362-379).
 *
 * A Rust `impl SonataModel for H100Vits` (or any FFI host) binds exactly these symbols; each entry
 * point cites the reference interface it replaces.  Plain pointers and sizes only — no torch /
 * CUDA types cross this boundary.  All functions are thread-safe per voice (the reference calls
 * `speak_one_sentence` concurrently from rayon workers on one model, synth/src/lib.rs:316-320).
 *
 * Error convention (mirrors ffi_support's ExternError used by libsonata, capi/libsonata.h:41-49):
 * every fallible call returns 0 on success or an error code and, when `err` is non-NULL, fills
 * `err->code` / `err->message` (heap string, free with sb200_string_free).  Codes reuse
 * libsonata's: 17 FAILED_TO_LOAD_RESOURCE, 18 PHONEMIZATION_ERROR, 19 OPERATION_ERROR
 * (capi/libsonata.h:10-16; SonataError variants at core/src/lib.rs:19-24).
 */
#ifndef SONATA_B200_H
#define SONATA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB200_OK 0
#define SB200_FAILED_TO_LOAD_RESOURCE 17
#define SB200_PHONEMIZATION_ERROR 18
#define SB200_OPERATION_ERROR 19

typedef struct sb200_voice sb200_voice;     /* = Arc<dyn SonataModel> holding a VitsModel (piper/src/lib.rs:291-297) */
typedef struct sb200_job sb200_job;         /* one batched synthesis in flight */
typedef struct sb200_latent sb200_latent;   /* = EncoderOutputs {z, y_mask} (piper/src/lib.rs:671-677) */

typedef struct sb200_error {
    int32_t code;
    char* message;
} sb200_error;

/* = sonata_core::Audio {samples: Vec<f32>, info.sample_rate, inference_ms} (audio/ops/src/samples.rs:208-214).
 * `data` is library-owned pinned host memory; release with sb200_audio_free. */
typedef struct sb200_audio {
    float* data;
    size_t len;
    float inference_ms;     /* fractional ms (the reference truncates to whole ms, piper/src/lib.rs:380) */
    uint32_t sample_rate;
} sb200_audio;

/* = PiperSynthesisConfig (piper/src/lib.rs:160-166); has_speaker==0 <=> speaker: None */
typedef struct sb200_synth_config {
    int64_t speaker;
    int32_t has_speaker;
    float noise_scale;
    float length_scale;
    float noise_w;
} sb200_synth_config;

/* = AudioInfo (audio/ops/src/samples.rs:9-14; values fixed at piper/src/lib.rs:282-288) */
typedef struct sb200_audio_info {
    uint32_t sample_rate;
    uint32_t num_channels;
    uint32_t sample_width;
} sb200_audio_info;

/* ---- library ---- */
const char* sb200_version(void);
void sb200_string_free(char* s);
void sb200_audio_free(sb200_audio* a);
int32_t sb200_device_count(void);

/* ---- voice: sonata_piper::from_config_path (piper/src/lib.rs:88-110) ----
 * `config_path` is the Piper `<voice>.onnx.json`; weights are read from the sibling `<voice>.svw`
 * (where the reference opens `<voice>.onnx`).  `device` = CUDA ordinal; -1 loads the config only
 * (host-side queries and id mapping work, every synthesis call fails with OPERATION_ERROR). */
int32_t sb200_voice_load(const char* config_path, int32_t device, sb200_voice** out, sb200_error* err);
/* Drops the caller's handle.  Jobs and latents created from the voice share ownership of it (the reference holds the
 * model behind an Arc, capi/src/lib.rs:314,375): they stay valid and may be freed afterwards, in any order. */
void sb200_voice_free(sb200_voice* v);

/* SonataModel::audio_output_info (core/src/lib.rs:83) */
int32_t sb200_audio_output_info(const sb200_voice* v, sb200_audio_info* out, sb200_error* err);
/* SonataModel::get_default_synthesis_config / get_fallback_ / set_fallback_ (core/src/lib.rs:88-90;
 * piper/src/lib.rs:444-462, 215-231: unknown speaker id -> OPERATION_ERROR) */
int32_t sb200_get_default_synthesis_config(const sb200_voice* v, sb200_synth_config* out, sb200_error* err);
int32_t sb200_get_fallback_synthesis_config(const sb200_voice* v, sb200_synth_config* out, sb200_error* err);
int32_t sb200_set_fallback_synthesis_config(sb200_voice* v, const sb200_synth_config* cfg, sb200_error* err);
/* SonataModel::get_language / properties["quality"] / supports_streaming_output (piper/src/lib.rs:180-196, 649-651).
 * Returned strings are heap copies: sb200_string_free. */
int32_t sb200_get_language(const sb200_voice* v, char** out, sb200_error* err);
int32_t sb200_get_quality(const sb200_voice* v, char** out, sb200_error* err);
int32_t sb200_supports_streaming_output(const sb200_voice* v);
/* SonataModel::get_speakers / speaker_name_to_id (piper/src/lib.rs:466-471): returns -1 when unknown */
int32_t sb200_num_speakers(const sb200_voice* v);
int64_t sb200_speaker_name_to_id(const sb200_voice* v, const char* name);

/* VitsModelCommons::phonemes_to_input_ids (piper/src/lib.rs:232-250): [bos] + (id(ch), pad)* + [eos];
 * unknown characters are dropped silently, only the first id of a map entry is used.
 * `*ids` is malloc'ed (free with sb200_ids_free). */
int32_t sb200_phonemes_to_input_ids(const sb200_voice* v, const char* phonemes_utf8, int64_t** ids, size_t* n,
                                    sb200_error* err);
void sb200_ids_free(int64_t* ids);
/* sb200_phonemes_to_input_ids plus, per id, where it came from: src_char[i] is the index, in Unicode characters of
 * `phonemes_utf8`, of the character id i was mapped from.  A pad id belongs to the character before it; bos and eos get
 * -1; dropped characters own no id.  Both arrays are malloc'ed (free each with sb200_ids_free). */
int32_t sb200_phonemes_to_input_ids_map(const sb200_voice* v, const char* phonemes_utf8, int64_t** ids,
                                        int64_t** src_char, size_t* n, sb200_error* err);

/* ---- synthesis ---- */
/* SonataModel::speak_one_sentence(phonemes: String) (piper/src/lib.rs:439-443) */
int32_t sb200_speak_one_sentence(sb200_voice* v, const char* phonemes_utf8, sb200_audio* out, sb200_error* err);
/* SonataModel::speak_batch(Vec<String>) (piper/src/lib.rs:425-437).  Same per-utterance result as B
 * sequential calls (the reference loops B=1 runs), computed as one batched pass. */
int32_t sb200_speak_batch(sb200_voice* v, const char* const* phonemes_utf8, size_t batch, sb200_audio* outs,
                          sb200_error* err);
/* VitsModel::infer_with_values(Vec<i64>) (piper/src/lib.rs:342-399) */
int32_t sb200_speak_ids(sb200_voice* v, const int64_t* ids, size_t n, sb200_audio* out, sb200_error* err);
/* batched infer_with_values: utterance b = ids_packed[offsets[b] .. offsets[b+1]) */
int32_t sb200_speak_batch_ids(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                              sb200_audio* outs, sb200_error* err);
/* sb200_speak_batch_ids with one synthesis config per utterance (speaker and scales, the per-request options of the
 * reference's CLI and gRPC service), still as one batched pass.  cfgs[b] applies to utterance b; NULL = the voice's
 * fallback config for every utterance, i.e. sb200_speak_batch_ids.  Each entry is checked like
 * sb200_set_fallback_synthesis_config (a speaker must be in the voice's speaker_id_map; has_speaker == 0 means
 * speaker 0); an invalid entry fails the call with OPERATION_ERROR naming the utterance.  Utterance b's result equals
 * a single-utterance call with cfgs[b] as the fallback config, except for the on-device noise of an unseeded utterance:
 * its draws depend on the utterance's position in the batch (see sb200_speak_batch_ids_seeded). */
int32_t sb200_speak_batch_ids_configs(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                      const sb200_synth_config* cfgs, sb200_audio* outs, sb200_error* err);

/* ---- per-phoneme durations: control them, and read when each id is spoken ----
 * Duration controls are per id, packed like ids_packed (one entry per id of the batch):
 *   scale_packed[i]  (finite, >= 0): id i lasts ceil((exp(logw) * length_scale) * scale) frames, the product rounded in
 *                    that order, so a scale of exactly 1.0 gives the bits of a call without scales;
 *   frames_packed[i] (-1 or >= 0) : >= 0 fixes id i's frame count (its predicted duration is still computed and
 *                    ignored); -1 keeps the predicted count.
 * Either array may be NULL (none of that kind).  All-1.0 scales and all -1 frames give the same bits as no controls.
 * A bad entry fails with OPERATION_ERROR naming the utterance and the id.  0 frames are allowed: the id is skipped; an
 * utterance whose ids all get 0 frames is 1 frame long, as a prediction summing to 0 always was.
 * Frames per id (the reference's `p_duration`) come packed like ids_packed; samples of id i = frames * 256. */
/* sb200_speak_batch_ids_configs with duration controls; id_frames_out (NULL: not wanted) receives the frames per id,
 * packed like ids_packed.  With NULL controls and NULL id_frames_out this is sb200_speak_batch_ids_configs, bit for bit.
 * Utterance b equals its single-utterance call with the same config and controls, except for the on-device noise of an
 * unseeded utterance: its draws depend on the utterance's position in the batch. */
int32_t sb200_speak_batch_ids_durations(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                        const sb200_synth_config* cfgs, const float* scale_packed,
                                        const int32_t* frames_packed, sb200_audio* outs, int32_t* id_frames_out,
                                        sb200_error* err);

/* ---- noise seeds: reproducible default-noise synthesis ----
 * The graph draws eps_w [T_x][2] (scaled by noise_w) and eps_z [T_y][inter] (scaled by noise_scale).  Unseeded, they
 * are Philox draws of the voice's call counter and the utterance's place in the packed batch.  A seeded utterance's
 * draws are a function of its seed, the tensor, the row (id or frame index) and the column only, so the utterance
 * equals itself run alone, bit for bit, whatever shares its batch, on every backend and every voice handle of the same
 * file, and the noise of frame t does not depend on how many frames follow it.
 * seeds[b] is utterance b's seed (any 64-bit value) when seeded[b] is 1; seeded[b] = 0 keeps its positional noise
 * (bit for bit what a call without seeds gives it); seeded == NULL with seeds != NULL seeds every utterance; seeds ==
 * NULL is a call without seeds.  A flag other than 0 / 1 fails with OPERATION_ERROR naming the utterance. */
/* sb200_speak_batch_ids_durations with noise seeds; NULL seeds is that call, bit for bit. */
int32_t sb200_speak_batch_ids_seeded(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                     const sb200_synth_config* cfgs, const float* scale_packed,
                                     const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                     sb200_audio* outs, int32_t* id_frames_out, sb200_error* err);

/* ---- output sample rate: results resampled on the device ----
 * An output rate is 8000, 11025, 16000, 22050, 24000, 32000, 44100 or 48000 Hz; 0 or the voice's own rate means no
 * resampling, bit for bit what a call without rates returns.  Any other value fails with OPERATION_ERROR naming the
 * utterance.  The resampler is scipy.signal.resample_poly's default: with up/down the reduced ratio out/in, H = 10 *
 * max(up, down) and h = firwin(2H + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up (designed in double, rounded to
 * f32), an utterance of n samples becomes ceil(n * up / down) samples,
 *     y[j] = sum_i x[i] * h[j*down + H - i*up]  over 0 <= i < n with 0 <= j*down + H - i*up <= 2H,
 * each sum one fmaf chain in ascending i, so a resampled utterance has the same bits in any batch.
 * sb200_speak_batch_ids_seeded with output_rates[b] the rate of utterance b (outs[b].sample_rate reports it); NULL
 * rates is that call, bit for bit. */
int32_t sb200_speak_batch_ids_rates(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                    const sb200_synth_config* cfgs, const float* scale_packed,
                                    const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                    const uint32_t* output_rates, sb200_audio* outs, int32_t* id_frames_out,
                                    sb200_error* err);

/* ---- loudness: each utterance measured (ITU-R BS.1770-4, one channel) and scaled to a target on the device ----
 * Loudness is measured on the signal the caller receives (after resampling, at the output rate).  K-weighting is
 * libebur128's any-rate design in double: a high shelf (f0 = 1681.974450955533 Hz, G = 3.999843853973347 dB,
 * Q = 0.7071752369554196, Vb = Vh^0.4996667741545416) then a high-pass (f0 = 38.13547087602444 Hz,
 * Q = 0.5003270373238773), both with K = tan(pi f0 / rate).  With the step S = (rate + 5) / 10 samples, block j covers
 * samples [jS, jS + 4S) (floor((n - 4S) / S) + 1 blocks when n >= 4S, else none) and has z_j = sum y^2 / 4S over the
 * K-weighted signal y, l_j = -0.691 + 10 log10(z_j).  The absolute gate keeps l_j > -70; with Gr = -0.691 +
 * 10 log10(mean z over those) - 10, the integrated loudness L = -0.691 + 10 log10(mean z over the blocks with
 * l_j > -70 and l_j > Gr), -inf when no block passes (silence, or under 400 ms).  Filter, energies and gates run in
 * double.  The gain g = min(10^((T - L) / 20), 1 / peak) (peak: the largest |x|) is computed in double, rounded to f32
 * and stepped down an ulp while f32(peak * g) > 1, and every sample becomes f32(x * g): normalisation never takes the
 * sample peak above full scale.  L = -inf or peak = 0 gives g = 1 and the utterance keeps its bits.  An utterance's L,
 * g and samples do not depend on its batch.  A target is a finite value in [-70, 0] LUFS, or NaN for none; any other
 * value fails with OPERATION_ERROR naming the utterance.  When some utterance has a target every utterance is
 * measured, and one without a target keeps its bits (g = 1).  The i16 results (sb200_job_fetch_i16,
 * sb200_job_copy_out format 1) convert an utterance with a target at the fixed scale, trunc(clamp(y * 32767, -32768,
 * 32767)), so its level survives; the others keep to_i16_vec.
 * sb200_speak_batch_ids_rates with target_lufs[b] the target of utterance b; lufs_out / gain_out (either may be NULL)
 * receive each utterance's L and g when some utterance has a target.  NULL targets is that call, bit for bit. */
int32_t sb200_speak_batch_ids_loudness(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                       const sb200_synth_config* cfgs, const float* scale_packed,
                                       const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                       const uint32_t* output_rates, const float* target_lufs, sb200_audio* outs,
                                       int32_t* id_frames_out, double* lufs_out, float* gain_out, sb200_error* err);

/* ---- pitch and tempo: each utterance's waveform warped by two ratios on the device ----
 * pitch p in [0.5, 2] multiplies every frequency of the utterance and keeps its duration; tempo t in [0.25, 4] plays it
 * t times faster and keeps its pitch (delivered length about n / t).  NaN or exactly 1 asks for nothing; any other
 * value outside its range fails with OPERATION_ERROR naming the utterance, before any device work.  An utterance that
 * asks for neither keeps its bits.  The stage runs at the voice's rate R on the decoder's waveform x[0 .. n), before any
 * resampling and loudness, which see its output as they see a waveform.  With alpha = (double)p / (double)t:
 *  1. Time stretch by alpha (skipped when p == t), WSOLA: Hs = R / 100, N = 2 Hs, D = R / 160 (integer divisions),
 *     n1 = floor(n alpha + 0.5), frames k < F = ceil(n1 / Hs) at a_k = floor(k Hs / alpha + 0.5) (double), a virtual frame
 *     -1 at a = -Hs with offset 0.  With q[i] = trunc(clamp(x[i], -1, 1) * 32767) (0 outside x), delta_0 = 0 and for
 *     k >= 1 delta_k is the delta in [-D, D] maximising sum_{i < N} q[a_{k-1} + delta_{k-1} + Hs + i] q[a_k + delta + i]
 *     in 64-bit integers, ties to the smaller |delta|, then to the negative one.  With w[i] = 0.5 - 0.5 cos(2 pi i / N),
 *     s[m] = w[r] x[a_k + delta_k + r] + w[r + Hs] x[a_{k-1} + delta_{k-1} + r + Hs] for k = m / Hs, r = m - k Hs, in f32.
 *  2. Pitch resampling by p (skipped when p == 1): n2 = floor(n1 / p + 0.5), y[j] = sum_i s[i] h(j p - i) with
 *     h(u) = c sinc(c u) (0.42 + 0.5 cos(pi u / W) + 0.08 cos(2 pi u / W)) for |u| < W, c = min(1, 1 / p), W = 16 / c;
 *     positions and phases in double, taps rounded to f32, one fmaf chain in ascending i.
 * The offsets are exact integers and the waveform stages have a fixed evaluation order, so a warped utterance has the
 * same bits in any batch.  Per-id frame counts stay frame counts of the unwarped utterance.
 * sb200_speak_batch_ids_loudness with pitch[b] / tempo[b] the ratios of utterance b (either array may be NULL); NULL and
 * NULL is that call, bit for bit. */
int32_t sb200_speak_batch_ids_prosody(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                      const sb200_synth_config* cfgs, const float* scale_packed,
                                      const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                      const uint32_t* output_rates, const float* target_lufs, const float* pitch,
                                      const float* tempo, sb200_audio* outs, int32_t* id_frames_out, double* lufs_out,
                                      float* gain_out, sb200_error* err);

/* ---- job API: the same batched pass split into its host<->device steps (bench / multi-GPU plumbing) ----
 * create  : copies ids to the device (H2D).  `eps_w` / `eps_z` optionally inject the graph's two
 *           RandomNormalLike draws (time-major: eps_w[b] = f32[T_x][2], eps_z[b] = f32[T_y][inter]);
 *           NULL -> Philox noise on the device (skipped when the matching scale is 0).
 * run     : all kernels; the waveform stays in HBM (optionally written into caller device memory
 *           `d_out`, capacity in floats, e.g. an NCCL send buffer); returns device time of the pass.
 * fetch   : D2H of the per-utterance waveforms into pinned host memory. */
int32_t sb200_job_create(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                         const float* const* eps_w, const float* const* eps_z, const size_t* eps_z_frames,
                         sb200_job** out, sb200_error* err);
/* keep every intermediate of the next run fetchable through sb200_job_debug_fetch (tests only) */
int32_t sb200_job_set_debug(sb200_job* job, int32_t on);
/* Per-utterance synthesis configs for the next sb200_job_run: cfgs[0 .. batch), or NULL for the voice's fallback config
 * (what a new job starts with, read at create time) for every utterance.  Entries are checked like
 * sb200_set_fallback_synthesis_config; an invalid one fails with OPERATION_ERROR naming the utterance and leaves the
 * job's configs unchanged.  Philox noise (no eps_w / eps_z given) of an unseeded utterance depends on its batch
 * position, as it always has: injected noise or a seed (sb200_job_set_seeds) makes a mixed batch equal its utterances
 * run alone. */
int32_t sb200_job_set_configs(sb200_job* job, const sb200_synth_config* cfgs, sb200_error* err);
/* Duration controls (see sb200_speak_batch_ids_durations) for the next sb200_job_run; NULL / NULL restores the default
 * (a job without controls, what a new job starts with).  Every entry is checked first; an invalid one fails with
 * OPERATION_ERROR naming the utterance and the id, and leaves the job's controls as they were. */
int32_t sb200_job_set_durations(sb200_job* job, const float* scale_packed, const int32_t* frames_packed, sb200_error* err);
/* Noise seeds (see sb200_speak_batch_ids_seeded) for the next sb200_job_run; seeds == NULL restores positional noise
 * (what a new job starts with).  Seeds on a job created with injected eps_w / eps_z fail with OPERATION_ERROR, as does
 * a bad flag; either leaves the job's seeds as they were.  With debug on, the run's noise is fetchable as "eps_w"
 * ([T_x][2]) and "eps_z" ([T_y][inter]) when its scale is not 0 for some utterance. */
int32_t sb200_job_set_seeds(sb200_job* job, const uint64_t* seeds, const int32_t* seeded, sb200_error* err);
/* Output rates (see sb200_speak_batch_ids_rates) for the next sb200_job_run: rates[0 .. batch), or NULL for none (what
 * a new job starts with).  An unsupported entry fails with OPERATION_ERROR naming the utterance and leaves the job's
 * rates as they were.  After a run with rates, every result call reports the resampled signal: the d_out of
 * sb200_job_run (its capacity counts resampled samples), sb200_job_fetch (sample_rate per utterance),
 * sb200_job_fetch_i16, sb200_job_copy_out (both formats) and the samples and out_offsets of sb200_job_lengths; its
 * frames stay frame counts.  sb200_job_profile reports the resampling launch as the region "resample". */
int32_t sb200_job_set_output_rates(sb200_job* job, const uint32_t* rates, sb200_error* err);
/* Loudness targets (see sb200_speak_batch_ids_loudness) for the next sb200_job_run: target_lufs[0 .. batch), or NULL
 * for none (what a new job starts with; so are targets that are all NaN).  A bad entry fails with OPERATION_ERROR naming
 * the utterance and leaves the job's targets as they were.  A run with targets measures after the decoder and any
 * resampling, scales the job's result in place (d_out included), and sb200_job_profile reports the launch as the
 * region "loudness". */
int32_t sb200_job_set_loudness(sb200_job* job, const float* target_lufs, sb200_error* err);
/* Each utterance's integrated loudness L (LUFS, -inf when no block passes the gates) and applied gain g of the last run
 * into lufs[0 .. batch) / gain[0 .. batch) (either may be NULL).  Fails when that run had no targets. */
int32_t sb200_job_loudness(const sb200_job* job, double* lufs, float* gain, sb200_error* err);
/* Pitch and tempo ratios (see sb200_speak_batch_ids_prosody) for the next sb200_job_run: pitch[0 .. batch) and
 * tempo[0 .. batch), either or both NULL for none (what a new job starts with; so are ratios that are all NaN or 1).  A
 * bad entry fails with OPERATION_ERROR naming the utterance and leaves the job's ratios as they were.  After a run with
 * ratios every result call reports the warped signal, as after a run with output rates, and sb200_job_profile reports
 * the offset chain and the overlap-add as the region "stretch" and the pitch resampler as "pitch". */
int32_t sb200_job_set_prosody(sb200_job* job, const float* pitch, const float* tempo, sb200_error* err);
/* Each utterance's stretched length n1, delivered length before any output-rate resampling n2 and WSOLA frame count F of
 * the last run into n1[0 .. batch) / n2 / frames (each may be NULL).  Fails when that run had no ratios. */
int32_t sb200_job_prosody(const sb200_job* job, int64_t* n1, int64_t* n2, int32_t* frames, sb200_error* err);
/* Frames per id of the last run, packed like ids_packed, into out_packed[0 .. capacity): one device->host copy of the
 * whole batch's cumulative durations, made on the first call after a run.  Fails before a run, or when capacity is
 * smaller than the number of ids. */
int32_t sb200_job_id_frames(sb200_job* job, int32_t* out_packed, size_t capacity, sb200_error* err);
int32_t sb200_job_run(sb200_job* job, float* d_out, size_t d_out_capacity, float* device_ms, sb200_error* err);
int32_t sb200_job_fetch(sb200_job* job, sb200_audio* outs, sb200_error* err);
size_t sb200_job_batch(const sb200_job* job);
/* per-utterance results available after run: frames (T_y), samples (256*T_y), offset into d_out */
/* Peak-normalised 16-bit PCM of every utterance of a finished job, converted on the device (half the device->host
 * bytes).  Mirrors AudioSamples::to_i16_vec / as_wave_bytes (crates/audio/ops/src/samples.rs:51-78) bit for bit.
 * outs[b] receives a malloc'ed buffer of lens[b] samples: free with sb200_i16_free. */
int32_t sb200_job_fetch_i16(sb200_job* job, int16_t** outs, size_t* lens, sb200_error* err);
void sb200_i16_free(int16_t* p);
/* G.711 audio for telephony (SIP/RTP PCMU = mu-law, payload type 0; PCMA = A-law, payload type 8), one byte per sample.
 * The bytes are G.711 of exactly the i16 samples sb200_job_fetch_i16 returns, after utterance b is scaled by gains[b]
 * (NULL = 1; each must be finite): to_i16_vec, or the fixed scale for an utterance with a loudness target.  The
 * encoding runs in the same two launches as the i16 conversion; nothing is encoded on the host.  law:
 * SB200_G711_MULAW (0) or SB200_G711_ALAW (1), as CPython's audioop.lin2ulaw / lin2alaw encode a 16-bit sample
 * (silence, sample 0, is 0xFF in mu-law and 0xD5 in A-law).  outs[b] receives a malloc'ed buffer of lens[b] bytes:
 * free with sb200_bytes_free.  A bad law or gain fails with OPERATION_ERROR before anything runs, a gain naming its
 * utterance. */
#define SB200_G711_MULAW 0
#define SB200_G711_ALAW 1
int32_t sb200_job_fetch_g711(sb200_job* job, int32_t law, const float* gains, uint8_t** outs, size_t* lens,
                             sb200_error* err);
void sb200_bytes_free(uint8_t* p);
/* Lossless FLAC, one complete native stream per utterance (RFC 9639, streamable subset; free with sb200_bytes_free).
 * Its samples are exactly the i16 samples sb200_job_fetch_i16 returns, after utterance b is scaled by gains[b] (NULL =
 * 1; each must be finite, as for sb200_job_fetch_g711), at the utterance's delivered sample rate.  The stream:
 *   - `fLaC`, one metadata block header (last = 1, type 0 STREAMINFO, length 34), STREAMINFO: min = max block size
 *     4096, the exact min / max frame size (0 without frames), the rate, 1 channel, 16 bits, the total samples and an
 *     all-zero MD5 ("not computed");
 *   - fixed-blocksize frames of 4096 samples (the last one shorter): sync 0xFFF8, block-size code 0b1100 (the last
 *     frame: 0b0110 / 0b0111 with 8- / 16-bit size - 1), the rate's code (11025 Hz: 0b1101 with a 16-bit Hz field),
 *     mono, 16 bits, the UTF-8-coded frame number and CRC-8;
 *   - one subframe (no wasted bits): CONSTANT when every sample is equal, else the smallest of FIXED 0-4, LPC 1-8
 *     (12-bit coefficients, shift 0..15) and VERBATIM, ties in that order; residuals in Rice partitions of order 0-8
 *     with each partition's optimal parameter (method 0b00, or 0b01 when one exceeds 14), no escapes;
 *   - zero padding to a byte and CRC-16.
 * The analysis, layout and packing run on the device; the frame sizes come back first, then only the compressed bytes.
 * A frame's bytes depend only on its samples and its position in its stream. */
int32_t sb200_job_fetch_flac(sb200_job* job, const float* gains, uint8_t** outs, size_t* lens, sb200_error* err);
/* The same encoder over a host buffer x[0 .. n) at sample_rate, on `device`: *out receives a malloc'ed stream of *len
 * bytes (free with sb200_bytes_free); n = 0 gives the 42-byte header-only stream.  A rate other than the eight output
 * rates (8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000) fails with OPERATION_ERROR before any device work. */
int32_t sb200_flac_encode(int32_t device, const int16_t* x, size_t n, uint32_t sample_rate, uint8_t** out, size_t* len,
                          sb200_error* err);
int32_t sb200_job_lengths(const sb200_job* job, int64_t* frames, int64_t* samples, int64_t* out_offsets);
/* Copy the result of a finished job into CALLER-OWNED host memory, utterances back to back in batch order.
 * format 0: f32 samples (what infer_with_values returns, piper/src/lib.rs:382-392);
 * format 1: i16 PCM, peak-normalised per utterance on the device (= AudioSamples::to_i16_vec, samples.rs:51-75;
 *           what libsonata hands to its callback, capi/src/lib.rs:416-438) -- half the device->host bytes;
 * format 2 / 3: G.711 mu-law / A-law of the format-1 samples (sb200_job_fetch_g711 with gains 1), one byte per sample.
 * Any other format fails with OPERATION_ERROR before anything runs.
 * `dst` may be ordinary or page-locked memory (see sb200_host_register), e.g. a slice of a segment shared by the
 * per-GPU worker processes of one frontend.  *written = bytes written; fails if `capacity_bytes` is too small. */
int32_t sb200_job_copy_out(sb200_job* job, void* dst, size_t capacity_bytes, int32_t format, size_t* written,
                           sb200_error* err);
/* Page-lock / unlock caller memory for DMA (cudaHostRegister) so that hosts without CUDA bindings (Rust, ctypes)
 * can pin a result segment once and reuse it.  Returns 0 on success. */
int32_t sb200_host_register(void* ptr, size_t bytes, sb200_error* err);
int32_t sb200_host_unregister(void* ptr);
void sb200_job_free(sb200_job* job);

/* ---- streaming: VitsStreamingModel (piper/src/lib.rs:480-669) ----
 * encode = infer_encoder (:537-574): ids -> latent z [T_y][inter] kept on the device.
 * decode_chunk = decoder.onnx on z[:, :, lo:hi] (:793-840) -> 256*(hi-lo) samples (no crossfade here). */
int32_t sb200_encode_ids(sb200_voice* v, const int64_t* ids, size_t n, sb200_latent** out, sb200_error* err);
int64_t sb200_latent_frames(const sb200_latent* z);
int32_t sb200_decode_chunk(sb200_voice* v, const sb200_latent* z, int64_t frame_lo, int64_t frame_hi,
                           sb200_audio* out, sb200_error* err);
void sb200_latent_free(sb200_latent* z);

/* ---- many realtime streams at once: SpeechStreamer (piper/src/lib.rs:765-858) for K clients, as the gRPC server's
 * SynthesizeUtteranceRealtime (grpc/src/main.rs:356-383) holds them, in one pass per step ----
 * Batched infer_encoder (:537-574): one encoder pass over `batch` utterances -> outs[b], each freed with
 * sb200_latent_free in any order (they share one device allocation, released with the last) and sharing ownership of
 * the voice like sb200_encode_ids' latents.  cfgs: one per utterance as for sb200_speak_batch_ids_configs (NULL = the
 * fallback config for every utterance); a bad entry fails the call naming the utterance.  As there, the on-device noise
 * draws of an unseeded utterance depend on its position in the batch (see sb200_encode_batch_ids_seeded). */
int32_t sb200_encode_batch_ids_configs(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                       const sb200_synth_config* cfgs, sb200_latent** outs, sb200_error* err);
/* sb200_encode_batch_ids_configs with duration controls (see sb200_speak_batch_ids_durations); NULL / NULL is that call,
 * bit for bit.  Each latent keeps its ids' frame counts: sb200_latent_id_frames. */
int32_t sb200_encode_batch_ids_durations(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                         const sb200_synth_config* cfgs, const float* scale_packed,
                                         const int32_t* frames_packed, sb200_latent** outs, sb200_error* err);
/* sb200_encode_batch_ids_durations with noise seeds (see sb200_speak_batch_ids_seeded); NULL seeds is that call, bit for
 * bit.  A seeded latent equals the `z` of the same utterance synthesised with the same seed. */
int32_t sb200_encode_batch_ids_seeded(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                      const sb200_synth_config* cfgs, const float* scale_packed,
                                      const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                      sb200_latent** outs, sb200_error* err);
/* The encoder's `p_duration` (piper/src/lib.rs:675, 706-717) as frames per id of the latent's utterance (their sum is
 * its frame count, except that an utterance whose ids all got 0 frames is 1 frame long).  Returns the number of ids;
 * writes them to out only when capacity is at least that (call with NULL, 0 to learn the size). */
int64_t sb200_latent_id_frames(const sb200_latent* z, int32_t* out, size_t capacity);
/* n calls of sb200_decode_chunk (decoder.onnx on z[:, :, lo:hi], :793-840) as ONE decoder pass: outs[k] gets
 * 256*(hi[k]-lo[k]) samples, bit for bit what sb200_decode_chunk(zs[k], lo[k], hi[k]) returns.  Every latent must come
 * from `v` and satisfy 0 <= lo < hi <= frames; errors name the chunk.  n = 0 does nothing. */
int32_t sb200_decode_chunks(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi, size_t n,
                            sb200_audio* outs, sb200_error* err);
/* The same pass, each chunk leaving as what libsonata's SYNTH_MODE_REALTIME emits for it: trim_lo_frames[k] /
 * trim_hi_frames[k] overlap frames dropped (NULL = none; piper :811-826), crossfade(fade) (samples.rs:144-157; 0 = none),
 * linear gain[k] (NULL = 1; synth/src/lib.rs:84-86), then to_i16_vec (samples.rs:51-75) normalised to the chunk's own
 * peak.  outs[k] receives a malloc'ed buffer of lens[k] samples: free with sb200_i16_free. */
int32_t sb200_decode_chunks_i16(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi,
                                const int64_t* trim_lo_frames, const int64_t* trim_hi_frames, size_t n, int32_t fade,
                                const float* gain, int16_t** outs, size_t* lens, sb200_error* err);
/* sb200_decode_chunks_i16's pass, each chunk leaving as the G.711 bytes (law as for sb200_job_fetch_g711) of the i16
 * samples that call returns for it, from the same launches: outs[k] receives a malloc'ed buffer of lens[k] bytes, free
 * with sb200_bytes_free.  A bad law fails with OPERATION_ERROR before anything runs. */
int32_t sb200_decode_chunks_g711(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi,
                                 const int64_t* trim_lo_frames, const int64_t* trim_hi_frames, size_t n, int32_t fade,
                                 const float* gain, int32_t law, uint8_t** outs, size_t* lens, sb200_error* err);

/* ---- streams at an output sample rate (see sb200_speak_batch_ids_rates) ----
 * A resampler is one stream's state on the device: the last K - 1 <= 2H/up of its inputs (K taps per phase) and the
 * counts of inputs consumed and outputs emitted.  out_rate must be a supported rate other than the voice's own (a
 * stream at the voice's rate needs none); otherwise OPERATION_ERROR.  It shares ownership of the voice. */
typedef struct sb200_resampler sb200_resampler;
int32_t sb200_resampler_create(sb200_voice* v, uint32_t out_rate, sb200_resampler** out, sb200_error* err);
void sb200_resampler_free(sb200_resampler* r);
/* sb200_decode_chunks_i16's pass and post-path (trims, crossfade(fade), gain) per chunk, then chunk k appended to its
 * stream's resampler resamplers[k] (NULL: the chunk leaves at the voice's rate after the post-path).  Chunk k emits
 * every output whose inputs have all arrived (the rest, 10-28 inputs at the supported rates, are held back) and, when
 * last[k] is 1 (last NULL: none), every output left, reading zeros past the stream's end; the resampler then takes no
 * more chunks.  A chunk may emit 0 samples.  The concatenation of a stream's outputs is, bit for bit, its whole input
 * resampled at once (sb200_debug_resample).  format 0: outs[k] is f32; 1: i16 normalised to the emitted chunk's own
 * peak (to_i16_vec); 2 / 3: G.711 mu-law / A-law bytes of those i16 samples, except that gain[k] then scales the
 * resampled samples just before their conversion (a volume on the delivered audio) rather than the chunk before it.  outs[k] is malloc'ed, lens[k] samples:
 * free with free() (sb200_i16_free / sb200_buffer_free / sb200_bytes_free).  Another format fails with OPERATION_ERROR.
 * A resampler appearing twice, made for another voice or already flushed fails with OPERATION_ERROR naming the chunk,
 * before any state changes. */
int32_t sb200_decode_chunks_resampled(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi,
                                      const int64_t* trim_lo_frames, const int64_t* trim_hi_frames, size_t n,
                                      int32_t fade, const float* gain, sb200_resampler* const* resamplers,
                                      const int32_t* last, int32_t format, void** outs, size_t* lens, sb200_error* err);

/* ---- streams with a pitch and a tempo (see sb200_speak_batch_ids_prosody) ----
 * A prosody stream is one stream's pitch / tempo state on the device: the tail of its input the WSOLA search and the
 * overlap-add still read (fewer than max(ceil(2 Hs / alpha), Hs) + 2 D + N samples), the tail of the stretched signal
 * the pitch resampler still reads (at most 2 W + 4 samples, W = 16 max(1, pitch) <= 32), the deltas of its last two
 * frames, and its counts.  pitch in [0.5, 2] and tempo in [0.25, 4] as for the batch calls (NaN or 1: none); neutral
 * ratios, or ratios out of range, fail with OPERATION_ERROR.  It shares ownership of the voice. */
typedef struct sb200_prosody_stream sb200_prosody_stream;
int32_t sb200_prosody_stream_create(sb200_voice* v, float pitch, float tempo, sb200_prosody_stream** out,
                                    sb200_error* err);
void sb200_prosody_stream_free(sb200_prosody_stream* s);
/* The "stretch" and "pitch" device time (ms) of the last chunk pass the stream was in (0: none ran). */
int32_t sb200_prosody_stream_profile(const sb200_prosody_stream* s, float* stretch_ms, float* pitch_ms);
/* sb200_decode_chunks_resampled with a prosody stream per chunk, warps[k] (NULL: none; warps NULL: none at all, which
 * is sb200_decode_chunks_resampled bit for bit).  Chunk k's samples after the post-path (trims, crossfade(fade) and,
 * except for G.711, gain[k]) are appended to warps[k]; what it emits then goes to resamplers[k] (or leaves at the
 * voice's rate) and to the conversion, with gain[k] where sb200_decode_chunks_resampled applies it.
 * Contract: the concatenation of what a prosody stream emits is, bit for bit, sb200_debug_prosody of the concatenation
 * of the samples appended to it.  Those are the chunks after this call's post-path on the device, which are the chunks
 * sb200_decode_chunks_resampled returns for a NULL resampler: their crossfade table is computed by this library
 * (sinf), so on the faded samples they can differ by an ulp from a crossfade applied on the host with another sine
 * (as a plain Python stream's chunks are).  Emission rule, with a_k = floor(k Hs / alpha + 0.5) (a_{-1} = -Hs) and C the inputs
 * consumed: frame k's delta is known once max(a_{k-1} + D + Hs + N, a_k + D + N) <= C (frames 0 .. K - 1, each known
 * one in order); stretched samples min(K Hs, floor(C alpha + 0.5)) are computed (C when pitch == tempo); output j is
 * emitted once ceil(j pitch + W) <= that count (every stretched sample when pitch is 1).  None of this depends on the
 * stream's final length.  The chunk with last[k] = 1 emits everything up to n2, reading zeros past the stream's end,
 * and the stream then takes no more chunks.  A chunk may emit 0 samples.  A prosody stream appearing twice, made for
 * another voice or already flushed, or a last flag other than 0 / 1, fails with OPERATION_ERROR naming the chunk before
 * any device work or state change. */
int32_t sb200_decode_chunks_warped(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi,
                                   const int64_t* trim_lo_frames, const int64_t* trim_hi_frames, size_t n, int32_t fade,
                                   const float* gain, sb200_resampler* const* resamplers,
                                   sb200_prosody_stream* const* warps, const int32_t* last, int32_t format, void** outs,
                                   size_t* lens, sb200_error* err);

/* ---- introspection for tests / bench ---- */
/* Copy a named intermediate of the LAST run of `job` to host (time-major fp32, valid rows of
 * utterance b only).  Names: "x","stats","logw","z_p","z","dec.pre","dec.up<i>","dec.mrf<i>", and the first encoder
 * layer's attention "qkv0","att0"; on the tensor-core attention also "p0" (head-0 probabilities) and "vt0" (V, returned
 * channel-major as [hidden][T]).  Duration predictor: "dp.g" (the flows' conditioning, [T][hidden]) and, per coupling
 * flow s = 0, 1, 2 in application order, "dp.f<s>.in" / "dp.f<s>.out" (the two-channel z before / after it, [T][2]),
 * "dp.f<s>.h" (the DDSConv output, [T][hidden]) and "dp.f<s>.h29" (the spline parameters, [T][32], 29 used).
 * Returns rows via *rows, cols via *cols; data malloc'ed (free with sb200_buffer_free). */
int32_t sb200_job_debug_fetch(sb200_job* job, const char* name, size_t b, float** data, size_t* rows, size_t* cols,
                              sb200_error* err);
void sb200_buffer_free(float* p);
/* cumulative durations (int32 per id) of utterance b */
int32_t sb200_job_debug_durations(sb200_job* job, size_t b, int32_t** cum, size_t* n, sb200_error* err);

typedef struct sb200_region_stat {
    char name[32];
    double ms;            /* device time between the region's CUDA events, last run */
    double flops;         /* algorithmic FLOPs (valid rows only, 2 per MAC) */
    double bytes;         /* layer-wise algorithmic bytes (each operand read once, result written once) */
    int32_t launches;
} sb200_region_stat;
/* region statistics of the last run of `job`; returns the number written (<= cap) */
int32_t sb200_job_profile(const sb200_job* job, sb200_region_stat* out, int32_t cap);
/* Test hook: the launch configuration the planner of backend 1 (wgmma bf16x2 conv) / 2 (wgmma 3xTF32 conv) would choose
 * for one convolution of `rows` output rows -- nothing is allocated or launched, so it also works without a GPU.
 * out16, backend 1: {nt, image rows, m-tiles, n-tiles, ring stages, smem bytes, window rows, grid CTAs, weights resident
 * (0/1), CTAs per SM, 0...}; backend 2: {nth, image rows, m-tiles, n-tiles, ring stages, chunk K-blocks, smem bytes, window
 * rows, 0...}.  Returns 0, or 19 if unsupported. */
int32_t sb200_debug_plan(int32_t backend, int64_t rows, int32_t cin, int32_t cout, int32_t k, int32_t dil, int32_t act,
                         int32_t has_res, int32_t accumulate, int32_t* out16);
/* Test hook: the same plan of backend 1, and whether its epilogue operands (residual, accumulated output) are staged in
 * shared memory while the tile's MMAs run: *staging_bytes is their shared memory per CTA, 0 when not staged.  Returns 0,
 * or 19 if unsupported. */
int32_t sb200_debug_plan_staging(int64_t rows, int32_t cin, int32_t cout, int32_t k, int32_t dil, int32_t act,
                                 int32_t has_res, int32_t accumulate, int32_t* staging_bytes);
/* Test hook: at most `cap` CTAs per launch of backend 1's persistent conv kernel from now on in this process (0: no cap;
 * the launch still takes one CTA per column tile).  Results do not depend on it.  Returns the previous cap. */
int32_t sb200_debug_conv_grid_cap(int32_t cap);
/* one convolution on caller data through backend 0 (fp32 CUDA cores), 1 (wgmma bf16x2) or 2 (wgmma 3xTF32), for kernel
 * unit tests: y[rows][cout] (=|+=) scale * (act(bias + conv_k,dil(lrelu_slope(x))) + res); w is [cout][cin][k];
 * act 0 none, 1 relu, 2 tanh*sigmoid gate (y is [rows][cout/2]); rows >= valid_rows are masked. */
int32_t sb200_debug_conv(int32_t device, int32_t backend, const float* x, int32_t rows, int32_t cin, const float* w,
                         const float* bias, int32_t cout, int32_t k, int32_t dil, float in_slope, int32_t act,
                         const float* res, float scale, int32_t accumulate, float* y, int32_t valid_rows,
                         sb200_error* err);
/* sb200_debug_conv with the engine's full row map and both output buffers.  Row q is valid iff
 * q < seg_end[q / gran] * seg_mul (seg_end has one entry per granule of `rows`, as the engine's segment tables); invalid
 * rows come out 0, or keep y's contents where that buffer accumulates.  Output columns n < split go to
 * y0[rows][min(split, cout or cout/2)] (accumulated when acc0), the rest to y1[rows][cout - split] (when acc1);
 * split = cout (or < 0) means y0 only. */
int32_t sb200_debug_conv_ex(int32_t device, int32_t backend, const float* x, int32_t rows, int32_t cin, const float* w,
                            const float* bias, int32_t cout, int32_t k, int32_t dil, float in_slope, int32_t act,
                            const float* res, float scale, const int32_t* seg_end, int32_t gran, int32_t seg_mul,
                            float* y0, int32_t acc0, int32_t split, float* y1, int32_t acc1, sb200_error* err);
/* A whole 64-channel HiFi-GAN ResBlock2 stage through its fused kernel (backend 1), for kernel unit tests:
 * y[rows][64] = (1/nbr) sum_b (x1_b + conv_{ks[b], dils[2b+1]}(lrelu_0.1(x1_b)) + bias),
 * x1_b = x + conv_{ks[b], dils[2b]}(lrelu_0.1(x)) + bias, each conv as sb200_debug_conv_ex runs it with that residual and
 * scale (1 / nbr on the second conv, which accumulates from the second branch on).  w holds the 2 nbr weights
 * [64][64][ks[b]] back to back in the order (branch, conv), bias the 2 nbr biases [64].  Row validity as in
 * sb200_debug_conv_ex; invalid rows come out 0.  Honours sb200_debug_conv_grid_cap. */
int32_t sb200_debug_resblock2_stage(int32_t device, const float* x, int32_t rows, int32_t nbr, const int32_t* ks,
                                    const int32_t* dils, const float* w, const float* bias, const int32_t* seg_end,
                                    int32_t gran, int32_t seg_mul, float* y, sb200_error* err);
/* Test hook: the fused ResBlock2 stage kernel's plan for such a stage over `rows` rows -- nothing is allocated or
 * launched.  out8 = {tile rows, x window rows, x1 rows, weight ring slots, dynamic shared memory bytes, grid CTAs,
 * threads per CTA, registers per CTA}.  Returns 0, or 19 if the kernel does not take the stage. */
int32_t sb200_debug_resblock2_plan(int64_t rows, int32_t nbr, const int32_t* ks, const int32_t* dils, int32_t* out8);
/* The duration predictor's spline inverse (10 bins, tails at +-5) on caller data, for kernel unit tests: z is [rows][2],
 * h29 [rows][ldh >= 29] holds per row 10 width logits, 10 height logits and 9 derivative logits, used as given (the
 * engine divides the width / height logits by sqrt(hidden) first).  z[r][tcol] is replaced by its inverse for rows
 * r < valid_rows and set to 0 for the rest; z[r][1 - tcol] is left alone.  z is updated in place. */
int32_t sb200_debug_spline(int32_t device, const float* h29, int32_t ldh, float* z, int32_t rows, int32_t tcol,
                           int32_t valid_rows, sb200_error* err);
/* The duration kernel on caller data: per segment b (rows [seg_off[b], seg_off[b] + seg_len[b]) of z [rows][2]),
 * logw = (z[:,0] - m0) * exp(-logs0), cum = inclusive scan of ceil(exp(logw) * length_scale), y_len[b] = max(sum, 1).
 * cum and y_len saturate at INT32_MAX.  logw / cum rows outside every segment keep what the caller passed in. */
int32_t sb200_debug_durations(int32_t device, const float* z, int32_t rows, const int32_t* seg_off, const int32_t* seg_len,
                              int32_t nseg, float m0, float logs0, float length_scale, float* logw, int32_t* cum,
                              int32_t* y_len, sb200_error* err);
/* Test hook: the resampling filter from in_rate to out_rate (see sb200_speak_batch_ids_rates), no device needed.
 * *up / *down receive the reduced ratio, and taps[0 .. 2H] the f32 taps in natural order when cap >= 2H + 1
 * (H = 10 * max(up, down)).  Returns 0, or 19 when out_rate is not a supported rate or equals in_rate. */
int32_t sb200_debug_resample_filter(int32_t in_rate, int32_t out_rate, float* taps, size_t cap, int32_t* up,
                                    int32_t* down);
/* Test hook, no device needed: the samples a stream resampled from in_rate to out_rate emits per chunk when its chunks
 * bring chunk_lens[0 .. n) inputs and the last one flushes it.  emitted[k] receives chunk k's count.  Returns 0, or 19
 * for an unsupported rate or a negative length. */
int32_t sb200_debug_resample_emit(int32_t in_rate, int32_t out_rate, const int64_t* chunk_lens, size_t n,
                                  int64_t* emitted);
/* The resampling kernel over one caller buffer x[0 .. n) from in_rate to out_rate: y receives ceil(n * up / down)
 * samples, bit for bit what a job resampling an utterance of those samples returns. */
int32_t sb200_debug_resample(int32_t device, const float* x, size_t n, int32_t in_rate, int32_t out_rate, float* y,
                             sb200_error* err);
/* Test hook, no device needed: the K-weighting design at `rate` (see sb200_speak_batch_ids_loudness) into coeffs[0 .. 10):
 * the shelf's b0, b1, b2, a1, a2, then the high-pass's (a0 = 1).  Returns 0, or 19 for a rate outside 8000 .. 384000. */
int32_t sb200_debug_loudness_filter(int32_t rate, double* coeffs);
/* The loudness kernel over one caller buffer x[0 .. n) at `rate`, measured only: *lufs receives its integrated loudness,
 * bit for bit what a job measures for an utterance of those samples. */
int32_t sb200_debug_loudness(int32_t device, const float* x, size_t n, int32_t rate, double* lufs, sb200_error* err);
/* Test hook, no device needed: the prosody plan (see sb200_speak_batch_ids_prosody) of n samples at `rate` with the two
 * ratios: shape6 receives Hs, N, D, n1, n2, F, and positions[0 .. min(F, cap)) the analysis positions a_k.  Returns 0, or
 * 19 for a ratio out of range or a rate outside 1000 .. 48000. */
int32_t sb200_debug_prosody_plan(int32_t rate, int64_t n, float pitch, float tempo, int64_t* shape6, int64_t* positions,
                                 size_t cap);
/* The prosody kernels over one caller buffer x[0 .. n) at `rate`: y[0 .. n2) receives the result, bit for bit what a job
 * gives an utterance of those samples, offsets[0 .. F) (NULL: not wanted) its delta_k and stretched[0 .. n1) (NULL: not
 * wanted) the signal after stage 1 when that stage runs.  Fails when a destination is smaller than the plan says. */
int32_t sb200_debug_prosody(int32_t device, const float* x, size_t n, int32_t rate, float pitch, float tempo, float* y,
                            size_t cap, int32_t* offsets, size_t offsets_cap, float* stretched, size_t stretched_cap,
                            sb200_error* err);
/* Test hook, no device needed: the samples a prosody stream with these ratios at `rate` emits per chunk (the rule of
 * sb200_decode_chunks_warped) when its chunks bring chunk_lens[0 .. n_chunks) inputs and the last one ends it.
 * emitted[k] receives chunk k's count.  Returns 0, or 19 for bad ratios, a bad rate or a negative length. */
int32_t sb200_debug_prosody_stream_plan(int32_t rate, float pitch, float tempo, const int64_t* chunk_lens, size_t n_chunks,
                                        int64_t* emitted);
/* A fresh prosody stream on `device` fed x[0 .. sum chunk_lens) in chunks of chunk_lens[0 .. n_chunks), the last one
 * ending it, with no decoder involved: y receives the concatenated outputs (cap: its size), lens[k] chunk k's count,
 * and offsets[0 .. F) (NULL: not wanted) every frame's delta as its chunk computed it. */
int32_t sb200_debug_prosody_stream(int32_t device, const float* x, const int64_t* chunk_lens, size_t n_chunks,
                                   int32_t rate, float pitch, float tempo, float* y, size_t cap, int64_t* lens,
                                   int32_t* offsets, size_t offsets_cap, sb200_error* err);
/* Test hook: G.711 (law as for sb200_job_fetch_g711) of x[0 .. n) into out[0 .. n).  device -1 runs the host copy of
 * the encoders (no device needed); otherwise the encoders run on that device over the buffer. */
int32_t sb200_debug_g711(int32_t device, int32_t law, const int16_t* x, size_t n, uint8_t* out, sb200_error* err);
/* kernels launched by this library since load (host-side counter) */
uint64_t sb200_launch_count(void);
/* select the contraction backend: 0 = fp32 CUDA-core implicit GEMM, 1 = wgmma (3xTF32) where
 * implemented; returns the previous value */
int32_t sb200_set_backend(sb200_voice* v, int32_t backend);

#ifdef __cplusplus
}
#endif
#endif /* SONATA_B200_H */
