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

/* ---- pitch contours: a pitch ratio per id, each id keeping its duration ----
 * A contour gives each id of an utterance its own pitch ratio, packed like ids_packed: a finite value in [0.5, 2], or
 * NaN or exactly 1 for none.  Every frequency in the samples an id produces is multiplied by its ratio, and with the
 * utterance's tempo t (1 without one) each id lasts its unwarped length / t.  A contour combines with a tempo but not
 * with the utterance's pitch ratio: an utterance with both fails with OPERATION_ERROR naming it, and a bad entry fails
 * naming the utterance and the id, before any device work.  A contour of NaN / 1 only asks for nothing.  In double
 * (Hs, N, D, the quantisation, the tie rule, the window and the sinc kernel as for sb200_speak_batch_ids_prosody), on
 * the decoder's n = 256 T_y samples:
 *  1. Pieces.  Id i covers input samples [256 C_{i-1}, 256 C_i) (C: cumulative frames).  Ids with 0 frames are dropped,
 *     and runs of consecutive remaining ids with equal f32 ratios (NaN -> 1) merge into one piece: pieces r = 1 .. m with
 *     0 = B_0 < .. < B_m = n and ratios p_r.  An utterance whose ids all have 0 frames is one piece with ratio 1.  One
 *     piece is planned as the utterance ratio p_1 (so a uniform contour has the bits of that pitch ratio).
 *  2. Stretch (skipped when every alpha_r = 1): alpha_r = (double)p_r / (double)t, S_0 = 0,
 *     S_r = S_{r-1} + (B_r - B_{r-1}) * alpha_r, n1 = floor(S_m + 0.5), F = ceil(n1 / Hs).  Frame k lies in the piece
 *     with S_{r-1} <= k Hs < S_r (the last piece: k Hs >= S_{m-1}) and a_k = floor(B_{r-1} + (k Hs - S_{r-1}) / alpha_r
 *     + 0.5); the virtual frame -1 stays at -Hs.  The offsets and the overlap-add are those of the utterance ratios.
 *  3. Pitch (skipped when every p_r = 1): Q_0 = 0, Q_r = Q_{r-1} + (S_r - S_{r-1}) / p_r for r < m,
 *     n2 = floor(Q_{m-1} + (n1 - S_{m-1}) / p_m + 0.5).  Output j lies in the piece with Q_{r-1} <= j < Q_r (the last
 *     one open-ended) at pos = S_{r-1} + (j - Q_{r-1}) * p_r, and y[j] = sum_i s[i] h_r(pos - i) over 0 <= i < n1 with
 *     |pos - i| < W_r, c_r = min(1, 1 / p_r), W_r = 16 / c_r; phases in double, taps rounded to f32, one fmaf chain in
 *     ascending i.
 *  4. Delivered ends.  Id i, ending at input sample b with B_{r-1} < b <= B_r (r = 1 for b = 0), ends at
 *     floor(Q_{r-1} + ((b - B_{r-1}) * alpha_r) / p_r + 0.5); the last id ends at n2.  With an output rate up / down a
 *     delivered end beta is at ceil(beta * up / down) of the resampled signal, as frame boundaries are.
 * Every expression is evaluated as written, each operation rounded (no fused multiply-add), so with one piece each one is
 * the utterance-ratio formula.  With t = 1 every end but the last is the unwarped 256 C_i, and the last, n2, is within
 * one sample of n.  Utterances without a contour get the same ends from the one piece of their ratios.
 * sb200_speak_batch_ids_prosody with pitch_packed (NULL: none) the contours of the batch, packed like ids_packed, and
 * bounds_out (NULL: not wanted) each id's delivered end before any output-rate resampling, packed like ids_packed.
 * NULL pitch_packed and NULL bounds_out is that call, bit for bit. */
int32_t sb200_speak_batch_ids_contour(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                      const sb200_synth_config* cfgs, const float* scale_packed,
                                      const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                      const uint32_t* output_rates, const float* target_lufs, const float* pitch,
                                      const float* tempo, const float* pitch_packed, sb200_audio* outs,
                                      int32_t* id_frames_out, int64_t* bounds_out, double* lufs_out, float* gain_out,
                                      sb200_error* err);

/* ---- formant ratios: the spectral envelope moved on its own ----
 * The pitch ratios and contours above multiply every frequency, the formants (the spectral envelope) included, so a
 * shifted voice sounds like a smaller or larger speaker.  A formant ratio phi per utterance (NaN: none; else a finite
 * value in [0.5, 2], or OPERATION_ERROR naming the utterance before any device work) gives the delivered audio the
 * voice's own envelope with every frequency multiplied by phi: phi = 1 with a pitch ratio or contour keeps the
 * formants where they were (so unlike the other ratios, an explicit 1 asks for something when the utterance has a
 * pitch), and phi != 1 without one moves them at the same pitch and duration.  The stage runs at the voice's rate R
 * on the n2 samples y the pitch stage hands out (its stretched signal with a tempo only, the decoder's waveform with
 * neither), after it and before any output-rate resampling and loudness.  It keeps the length: n2, the delivered ends,
 * the frame counts and the alignments are those without it.  In double:
 *  1. Frames.  N = 1024, H = 256, periodic Hann w[i] = 0.5 - 0.5 cos(2 pi i / N).  Frame m in [-3, ceil(n2 / H)) reads
 *     y[m H + i], i < N, zero outside [0, n2); each output sample lies in exactly 4 frames.
 *  2. Frame ratios.  c_m = clamp(m H + N / 2, 0, n2 - 1).  p_m is the utterance's pitch ratio (1 without one), or with
 *     a contour the p_r of the piece with Q_{r-1} <= c_m < Q_r (step 3 of sb200_speak_batch_ids_contour).
 *     r_m = p_m / phi, Q_m = floor(Q0 / p_m + 0.5) with Q0 = floor(R / 250): a 4 ms cutoff on the unshifted voice
 *     (half the period of a 120 Hz voice), whose harmonics and formants y carries p_m times further apart.  A 2 ms
 *     cutoff smooths formants of 80 - 120 Hz bandwidth away: it neither keeps them through a pitch shift nor moves
 *     them at a fixed pitch.
 *  3. Envelope.  X = rfft(w frame), P = |X|^2 (bins 0 .. N/2), eps = 1e-10 mean(P) + 1e-30, Lambda = log(P + eps) / 2,
 *     c = irfft(Lambda) (the real cepstrum), lifter l[0] = 1, l[q] = l[N - q] = (1 + cos(pi q / Q_m)) / 2 for
 *     1 <= q < Q_m, else 0, and E = Re rfft(c l), bins 0 .. N/2.
 *  4. Gain.  Bin k reads u = k r_m: E^ = E[N/2] when u >= N/2, else E[i] + (u - i)(E[i + 1] - E[i]) with i = floor(u);
 *     g_k = clamp(E^ - E[k], -G, G) with G = 1.2 ln 10 (24 dB as a natural-log amplitude).
 *  5. Synthesis.  z_m = irfft(X e^g); out[j] = (sum_m w[j - m H] z_m[j - m H]) / 1.5 over its 4 frames in ascending m,
 *     rounded to f32 once.
 * An utterance runs the stage only when phi is finite and some frame has r_m != 1; any other keeps its bits (one with
 * phi == its pitch ratio and no contour among them).  The kernels compute in double with their own FFTs and a fixed
 * order per utterance, so an utterance has the same bits in any batch; a sample is within half an f32 ulp of the
 * float64 specification's value plus 1e-11 (tests/formant_reference.py).  Realtime streams take a formant ratio through
 * sb200_prosody_stream_create_formant, with the same bits as this call.
 * sb200_speak_batch_ids_contour with formants (NULL: none) one ratio per utterance.  NULL formants is that call, bit for
 * bit. */
int32_t sb200_speak_batch_ids_formants(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                       const sb200_synth_config* cfgs, const float* scale_packed,
                                       const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                       const uint32_t* output_rates, const float* target_lufs, const float* pitch,
                                       const float* tempo, const float* pitch_packed, const float* formants,
                                       sb200_audio* outs, int32_t* id_frames_out, int64_t* bounds_out,
                                       double* lufs_out, float* gain_out, sb200_error* err);

/* ---- speaker blends: a voice between the speakers of a multi-speaker voice ----
 * A speaker reaches the model through one vector g (the reference's emb_g(sid)).  A blend of an utterance or stream is
 * n >= 1 pairs (s_i, u_i): distinct speaker ids of the voice (values of its speaker_id_map) and finite f32 weights
 * u_i >= 0, at least one of them > 0.  Any other blend (an unknown or repeated id, a negative, NaN or infinite weight,
 * all weights zero, an empty blend, or any blend on a single-speaker voice) fails with OPERATION_ERROR before any device
 * work, naming the utterance (or stream) and the speaker or weight, and leaves the job or batch as it was.
 *  1. Canonical form: drop the pairs with u_i = 0 and sort the rest by s ascending; U = sum of (double) u_i in that
 *     order, and w_i = (float)((double) u_i / U).
 *  2. Embedding: acc = 0.0f, then acc = fmaf(w_i, emb_g[s_i][k], acc) for each i in canonical order; g[k] = acc.
 *  3. Conditioning: the effective biases base[r] + sum_k W[r][k] g[k] of every speaker-conditioned 1x1 conv (the
 *     duration predictor's, every flow WaveNet's and the vocoder input's), computed as for a plain speaker with g in
 *     place of emb_g(sid): in a batch pass, in an encoder pass and in every decoder chunk pass of its latents.
 *  4. The blend replaces the config's speaker; the config's noise_scale, length_scale and noise_w still apply.
 * So a blend whose canonical form is one speaker s (any positive weight, with or without zero-weight extras) has w = 1
 * and g = emb_g[s]: the bits of that speaker.  Blends with the same canonical form (reordered, with zero weights added,
 * or every weight scaled by a power of two) give the same bits, and a blended utterance has the same bits in any batch
 * (with seeded or injected noise).  Equal canonical blends of a pass share one speaker slot, and a one-speaker blend
 * shares the slot of that plain speaker; a pass in which no slot blends two or more speakers runs as it does without
 * blends, with the same launches.
 * A blend table is three arrays: blend_speakers and blend_weights, and blend_offsets[0 .. batch] (offsets[0] = 0):
 * utterance b's pairs are [offsets[b], offsets[b + 1]), and an empty range means no blend for that utterance.
 * sb200_speak_batch_ids_formants with a blend table (NULL blend_offsets: none).  NULL is that call, bit for bit. */
int32_t sb200_speak_batch_ids_blends(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                     const sb200_synth_config* cfgs, const float* scale_packed,
                                     const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                     const uint32_t* output_rates, const float* target_lufs, const float* pitch,
                                     const float* tempo, const float* pitch_packed, const float* formants,
                                     const int64_t* blend_speakers, const float* blend_weights,
                                     const size_t* blend_offsets, sb200_audio* outs, int32_t* id_frames_out,
                                     int64_t* bounds_out, double* lufs_out, float* gain_out, sb200_error* err);

/* ---- volume contours: a level in dB per id ----
 * A volume contour gives each id of an utterance a level, packed like ids_packed: a finite value in [-60, 20] dB,
 * -inf for silence (gain 0), or NaN or exactly 0 for no change.  Any other value fails with OPERATION_ERROR naming the
 * utterance and the id, before any device work; a contour of NaN / 0 only asks for nothing.  The stage runs at the
 * voice's rate R on the n2 samples x the formant stage hands out (the pitch stage's output without one, the decoder's
 * waveform without prosody), after those stages and before any output-rate resampling and loudness, which see its
 * output as they see a waveform.  It changes no length, delivered end, frame count or alignment.  In double, each
 * operation rounded (no fused multiply-add):
 *  1. Pieces.  Id i covers the delivered samples [E_{i-1}, E_i), E_{-1} = 0, with E the ends of step 4 of
 *     sb200_speak_batch_ids_contour (what sb200_job_prosody_bounds reports; 256 C_i without pitch, tempo or contour;
 *     the last id always ends at n2).  Ids whose span is empty are dropped, and runs of consecutive ids with equal f32
 *     levels (NaN -> 0) merge: pieces r = 1 .. m with boundaries 0 = B_0 < B_1 < .. < B_m = n2 and levels v_r, and
 *     g_r = f32(10^(v_r / 20)) computed on the host (-inf: 0).
 *  2. Gain curve.  L = 2 (R / 200) samples (integer division: 220 at 22.05 kHz, 160 at 16 kHz, about 10 ms).  Boundary
 *     r (1 <= r < m) ramps the samples B_r - L/2 <= j < B_r + L/2 with t = (j - B_r + L/2 + 0.5) / L and
 *     S_r(j) = t t (3 - 2 t).  G_j = g_a + sum (g_{r+1} - g_r) S_r(j) over the boundaries whose ramp covers j, in
 *     ascending r, with a the piece before the first of them (the piece holding j when none does), rounded to f32 once.
 *  3. Output.  y_j = x_j G_j, one f32 multiply, with no clamp.
 * So a contour that merges into one piece is the utterance times g_1 bit for bit, an utterance whose pieces all have
 * gain 1 runs nothing and keeps its bits, and a contoured utterance has the same bits in any batch.  A loudness target
 * normalises the contoured utterance as a whole, so the contour's relative levels survive it.  The executable
 * specification is tests/volume_reference.py.  Realtime streams take a contour through
 * sb200_prosody_stream_create_volume, with the same bits as this call.
 * sb200_speak_batch_ids_blends with volume_db_packed (NULL: none) the contours of the batch, packed like ids_packed.
 * NULL is that call, bit for bit. */
int32_t sb200_speak_batch_ids_volume(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                     const sb200_synth_config* cfgs, const float* scale_packed,
                                     const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                     const uint32_t* output_rates, const float* target_lufs, const float* pitch,
                                     const float* tempo, const float* pitch_packed, const float* formants,
                                     const int64_t* blend_speakers, const float* blend_weights,
                                     const size_t* blend_offsets, const float* volume_db_packed, sb200_audio* outs,
                                     int32_t* id_frames_out, int64_t* bounds_out, double* lufs_out, float* gain_out,
                                     sb200_error* err);

/* ---- breaks: a pause in milliseconds after any id ----
 * A break image gives each id of an utterance a pause after it, packed like ids_packed (f32): a finite value in
 * (0, 10000] ms, or NaN or exactly 0 for none.  Any other value (negative, +-inf, above 10 s) fails with
 * OPERATION_ERROR naming the utterance and the id, before any device work, as does an utterance whose paused length
 * would pass 2^31 - 1 samples.  The stage runs at the voice's rate R on the n2 samples x the volume stage hands out
 * (the formant stage's, the pitch stage's or the decoder's without one), after it and before any output-rate
 * resampling, loudness target, live meter and encoder, which see its output as they see a waveform.  In double, each
 * operation rounded (no fused multiply-add):
 *  1. Lengths.  N_i = floor(ms_i R / 1000 + 0.5); a break with N_i = 0 asks for nothing.
 *  2. Positions.  Break i sits at E_i, id i's delivered end before breaks (the ends of step 4 of
 *     sb200_speak_batch_ids_contour, what sb200_job_prosody_bounds reported before breaks: 256 C_i without prosody; the
 *     last end is n2).  Breaks at equal positions merge in ascending id order, their lengths summed: breaks k = 1 .. m at
 *     P_1 < .. < P_m of lengths M_k, with running totals D_k = M_1 + .. + M_k, D_0 = 0.
 *  3. Fades.  F = R / 200 (integer division, volume's half ramp), S(t) = t t (3 - 2 t).  Input sample j gets h_j: 1.0
 *     multiplied, in ascending k, by S(((P_k - j) - 0.5) / F) for every k with P_k - F <= j < P_k (fade-out) and by
 *     S(((j - P_k) + 0.5) / F) for every k with P_k <= j < P_k + F (fade-in), rounded to f32 once; y_j = x_j h_j, one
 *     f32 multiply, no clamp.
 *  4. Output.  n2 + D_m samples: input sample j lands at j + D_{k(j)}, k(j) = #{k : P_k <= j}, and outputs
 *     [P_k + D_{k-1}, P_k + D_k) hold +0.0f.  A break at n2 is trailing silence; one at 0 (after ids with no samples)
 *     leading silence.
 *  5. Delivered ends.  E'_i = E_i + sum of M_k over P_k <= E_i: a pause belongs to the id it follows, so alignments stay
 *     contiguous from sample 0 and the last end is the delivered length.  bounds_out, sb200_job_prosody_bounds and the
 *     stream bounds report E' (at an output rate: ceil(E' up / down)).  The volume stage still uses E.
 * An image of NaN / 0 only, or whose breaks all round to 0 samples, runs nothing and keeps every bit; an utterance with
 * breaks has the same bits in any batch; a loudness target normalises the paused utterance as a whole (its silent
 * blocks fall under the absolute gate); the i16 route's peak scale does not move.  When some utterance of a batch asks,
 * every utterance goes through the one break launch (one that does not ask is copied).  sb200_job_lengths, the fetches
 * (f32, i16, G.711, FLAC), sb200_job_copy_out and the d_out capacity all count the paused signal.  The executable
 * specification is tests/break_reference.py.  Realtime streams take breaks through sb200_prosody_stream_create_breaks.
 * sb200_speak_batch_ids_volume with breaks_ms_packed (NULL: none); NULL is that call, bit for bit. */
int32_t sb200_speak_batch_ids_breaks(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                     const sb200_synth_config* cfgs, const float* scale_packed,
                                     const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                     const uint32_t* output_rates, const float* target_lufs, const float* pitch,
                                     const float* tempo, const float* pitch_packed, const float* formants,
                                     const int64_t* blend_speakers, const float* blend_weights,
                                     const size_t* blend_offsets, const float* volume_db_packed,
                                     const float* breaks_ms_packed, sb200_audio* outs, int32_t* id_frames_out,
                                     int64_t* bounds_out, double* lufs_out, float* gain_out, sb200_error* err);

/* ---- target durations: fit an utterance, or spans of it, to a duration in milliseconds ----
 * A target table gives utterance b the spans k in [fit_offsets[b], fit_offsets[b + 1]) (fit_offsets: batch + 1
 * entries from 0, as blend_offsets): ids [fit_first[k], fit_end[k]) of the utterance (0-based, end exclusive) and the
 * duration fit_ms[k] they should take.  A whole utterance is the span [0, n_ids), bos and eos included.  Spans must be
 * non-empty, inside the utterance, ascending and disjoint, and fit_ms finite in (0, 600000], or NaN for a span that
 * asks for nothing; any other entry fails with OPERATION_ERROR naming the utterance and the span, before any device
 * work, as does a span that asks on an utterance with a tempo ratio (the two set the same length).  Solving span S at
 * the voice's rate R:
 *  1. T = floor(ms R / 1000 + 0.5) samples, in double.
 *  2. P = the break samples of S's ids (step 1 of sb200_speak_batch_ids_breaks: a pause belongs to the id it follows).
 *  3. Each predicted id i of S gets c_i(u) = ceil(w_i u) frames for an f32 factor u, where w_i = (exp(logw_i)
 *     length_scale) scale_i is rounded exactly as without a target, and the multiply by u is one more f32 multiply,
 *     applied last.  An id with a fixed count (frames_packed >= 0) keeps it; counts saturate at INT_MAX.
 *  4. L(u) = 256 sum c_i(u) + P samples (the hop times S's frames), in int64.
 *  5. u* is the largest f32 u in [0.5, 2] with L(u) <= T: the longest delivery that does not overrun the slot.  When
 *     even L(0.5) > T, u* = 0.5 and the span is over its target.  Every c_i is nondecreasing in u, so u* is unique and
 *     any u of its plateau gives the same counts.  A span without a predicted id asks for nothing (u* = 1).
 * Ids outside every span keep their counts; without a span that asks, nothing is multiplied, launched or copied, and
 * every bit is that of a call without targets.  u* is found on the device between the duration predictor and the
 * durations' scan (one warp per span, bisection over the f32 bit patterns of [0.5, 2]: at most 25 integer sums), so a
 * fitted utterance has the bits of the same utterance run with frames_packed fixed to its fitted counts, in any batch.
 * Everything after the durations composes as it does with fixed counts: pitch ratios and contours, formants, volume,
 * breaks, output rates, loudness, G.711 and FLAC; the delivered ends are what bounds_out reports.  fit_factor_out /
 * fit_len_out (per span, either may be NULL) receive u* and L(u*) in samples at R (NaN and -1 for a span that asks
 * nothing).  The executable specification is tests/fit_reference.py.  Realtime streams are fitted in their encoder
 * pass (sb200_encode_batch_ids_targets).  sb200_speak_batch_ids_breaks with a target table (NULL fit_offsets: none);
 * NULL is that call, bit for bit. */
int32_t sb200_speak_batch_ids_fit(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                  const sb200_synth_config* cfgs, const float* scale_packed,
                                  const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                  const uint32_t* output_rates, const float* target_lufs, const float* pitch,
                                  const float* tempo, const float* pitch_packed, const float* formants,
                                  const int64_t* blend_speakers, const float* blend_weights,
                                  const size_t* blend_offsets, const float* volume_db_packed,
                                  const float* breaks_ms_packed, const int64_t* fit_first, const int64_t* fit_end,
                                  const float* fit_ms, const size_t* fit_offsets, sb200_audio* outs,
                                  int32_t* id_frames_out, int64_t* bounds_out, double* lufs_out, float* gain_out,
                                  float* fit_factor_out, int64_t* fit_len_out, sb200_error* err);

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
/* A pitch contour (see sb200_speak_batch_ids_contour) for the next sb200_job_run, packed like ids_packed, or NULL for none
 * (what a new job starts with; so is a contour that is all NaN or 1).  Checked like sb200_job_set_durations: a bad entry
 * fails with OPERATION_ERROR naming the utterance and the id, and an utterance with a pitch ratio set by
 * sb200_job_set_prosody fails naming the utterance; either leaves the job as it was.  A run with a contour copies the
 * batch's cumulative durations to the host with the frame counts, and after it every result call reports the warped
 * signal, as after a run with ratios. */
int32_t sb200_job_set_pitch_contour(sb200_job* job, const float* pitch_packed, sb200_error* err);
/* Formant ratios (see sb200_speak_batch_ids_formants) for the next sb200_job_run, one per utterance, or NULL for none
 * (what a new job starts with; so are ratios that are all NaN).  A bad entry fails naming the utterance and leaves the
 * job as it was.  A ratio of 1 asks for something on an utterance with a pitch ratio or contour.  The result keeps
 * its layout: the stage changes no length or offset. */
int32_t sb200_job_set_formants(sb200_job* job, const float* formants, sb200_error* err);
/* A volume contour (see sb200_speak_batch_ids_volume) for the next sb200_job_run, packed like ids_packed, or NULL for
 * none (what a new job starts with; so is a contour that is all NaN or 0).  Checked like sb200_job_set_pitch_contour: a
 * bad entry fails with OPERATION_ERROR naming the utterance and the id, and leaves the job as it was.  A run with a
 * contour copies the batch's cumulative durations to the host with the frame counts, and sb200_job_profile reports the
 * stage as the region "volume".  The result keeps its layout: the stage scales it in place. */
int32_t sb200_job_set_volume_contour(sb200_job* job, const float* volume_db_packed, sb200_error* err);
/* Breaks (see sb200_speak_batch_ids_breaks) for the next sb200_job_run, packed like ids_packed, or NULL for none (what a
 * new job starts with; so is an image that is all NaN or 0).  A bad entry fails with OPERATION_ERROR naming the
 * utterance and the id, and leaves the job as it was.  A run with breaks copies the batch's cumulative durations to the
 * host, and sb200_job_profile reports the stage as the region "break".  The result's lengths, offsets and
 * sb200_job_prosody_bounds count the pauses. */
int32_t sb200_job_set_breaks(sb200_job* job, const float* breaks_ms_packed, sb200_error* err);
/* Target durations (see sb200_speak_batch_ids_fit) for the next sb200_job_run, or NULL fit_offsets for none (what a new
 * job starts with; so is a table whose spans all ask nothing).  A bad entry fails with OPERATION_ERROR naming the
 * utterance and the span, and leaves the job's targets as they were.  A run with targets reports the fit as the
 * profile region "fit" and, with debug set, keeps each span's predicted w_i fetchable as "fit.w" (X level, one column;
 * rows outside the spans and of fixed ids are not written). */
int32_t sb200_job_set_targets(sb200_job* job, const int64_t* fit_first, const int64_t* fit_end, const float* fit_ms,
                              const size_t* fit_offsets, sb200_error* err);
/* u* and L(u*) of every span of the last run's targets, packed as the table (capacity: its spans; either may be NULL);
 * fails when the last run had none. */
int32_t sb200_job_targets(const sb200_job* job, float* fit_factor, int64_t* fit_len, size_t capacity, sb200_error* err);
/* Speaker blends (see sb200_speak_batch_ids_blends) for the next sb200_job_run as a blend table, or NULL offsets for none
 * (what a new job starts with).  Every entry is checked first; a bad one fails with OPERATION_ERROR naming the utterance
 * and leaves the job's blends as they were. */
int32_t sb200_job_set_speaker_blends(sb200_job* job, const int64_t* blend_speakers, const float* blend_weights,
                                     const size_t* blend_offsets, sb200_error* err);
/* Each id's delivered end in the last run (see sb200_speak_batch_ids_contour), at the voice's rate, packed like
 * ids_packed, into out_packed[0 .. capacity).  Fails before a run, or when capacity is smaller than the number of ids. */
int32_t sb200_job_prosody_bounds(sb200_job* job, int64_t* out_packed, size_t capacity, sb200_error* err);
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

/* ---- Watermark: a keyed provenance mark on everything a voice delivers (tests/watermark_reference.py) ----
 * Set on the voice, not per call: once set, every job of the voice is marked, through every batch route (f32, i16,
 * G.711, FLAC, output rates, loudness targets), and every realtime stream made while it is set
 * (sb200_watermark_stream_create).
 *
 * Where: at each utterance's delivered rate R, after the last waveform stage (the resampler with an output rate, else
 * breaks, volume, formant, pitch or the decoder) and before loudness and the encoders, over exactly the samples the
 * caller receives.  n counts them from 0 at the utterance's first delivered sample (pauses count).  Loudness and the
 * peak-scaled i16 conversion only apply a gain afterwards, and detection does not depend on gain.
 * Chips: P = 4096.  c_j[m] = +1 when bit 0 of word 0 of Philox4x32-10 with counter (m, j, 0, 0) and key
 * (key mod 2^32, key >> 32) is 1, else -1, for j in {0, 1}, m in [0, P).  c0 is the sync sequence; c1 carries the
 * payload s as a cyclic shift: c[n] = c0[n mod P] + c1[(n - s) mod P], one of {-2, 0, 2}.
 * Envelope: blocks of B = floor(R / 100) samples (the last may be shorter, L_k its length); q[n] the sample quantised
 * as the pitch stage quantises it, (int)(clamp(x, -1, 1) * 32767) with an f32 product and a truncating cast;
 * S_k = sum of q^2 over block k in int64; E_k = min(S_{k-1} / L_{k-1}, S_k / L_k) in double, block -1 taken as block 0.
 * So the 10 ms after speech, and silences and pauses, get no mark.
 * Gain: alpha = 10^(strength_db / 20) in double on the host; a_k = (float)((alpha * sqrt(E_k * 0.5)) / 32767), each
 * double operation correctly rounded; y[n] = x[n] + a_k * c[n] as one f32 multiply and one f32 add.  The mark's power
 * is alpha^2 E_k.  Nothing is clamped; lengths, ends, alignments and prosody bounds do not change.
 * Scope: a provenance mark, not a tamper-proof one (folding many marked clips estimates the P-periodic sequence).  It
 * survives gain, i16, G.711, FLAC, cropping and additive noise; it is not designed to survive resampling, time-scaling,
 * pitch-shifting or lossy codecs after delivery.  A file that joins separately marked utterances splits its evidence
 * over several offsets, so detecting each utterance is stronger than detecting the whole file. */
typedef struct sb200_watermark {
    uint64_t key;
    int32_t payload;     /* [0, 4096) */
    float strength_db;   /* finite, in [-40, -10] */
} sb200_watermark;
/* wm == NULL turns the mark off.  A bad payload or strength fails with OPERATION_ERROR naming the field and leaves the
 * voice as it was.  The first use of a key builds its two chip tables on the voice's device.  A job reads the setting
 * once, when it starts to run. */
int32_t sb200_voice_set_watermark(sb200_voice* v, const sb200_watermark* wm, sb200_error* err);
/* *on receives 1 and *out the setting when the voice marks, else *on = 0 (out untouched). */
int32_t sb200_voice_watermark(const sb200_voice* v, sb200_watermark* out, int32_t* on, sb200_error* err);
typedef struct sb200_watermark_result {
    int32_t marked;      /* 1: z0 >= 6.5 */
    int32_t payload;     /* (o0 - o1) mod P when marked and z1 >= 6.5, else -1 */
    int32_t offset;      /* o0: the clip start's position mod P */
    double z0, z1;
} sb200_watermark_result;
/* Detection in clips packed[offsets[b] .. offsets[b + 1]) for b < batch, f32 (fmt 0, quantised as above) or i16
 * (fmt 1) samples, each possibly cropped anywhere, on `device`:
 *   fold F[m] = sum of q[i] over i = m mod P (int64, exact); X = FFT_P(F); W = X / |X| (0 where |X| = 0);
 *   r_j[o] = sum_m w[m] c_j[(m + o) mod P] = Re IFFT(conj(W) FFT_P(c_j)) [o];
 *   o_j = argmax r_j (smallest o on ties); z_j = (r_j[o_j] - mu_j) / sigma_j, mu_j and sigma_j the population mean and
 *   standard deviation of the other P - 1 lags (z_j = 0 when sigma_j = 0).
 * Without a mark the standardised lags are about N(0, 1), so a false detection per clip and key is bounded by about
 * P Q(6.5) = 1.6e-7.  A bad format fails with OPERATION_ERROR before any device work. */
int32_t sb200_watermark_detect(int32_t device, uint64_t key, int32_t fmt, const void* packed, const size_t* offsets,
                               size_t batch, sb200_watermark_result* out, sb200_error* err);

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
/* sb200_encode_batch_ids_seeded with a blend table (see sb200_speak_batch_ids_blends); NULL is that call, bit for bit.
 * Each latent keeps its utterance's canonical blend (or plain speaker), and every decoder chunk pass of it conditions on
 * that blend. */
int32_t sb200_encode_batch_ids_blends(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                      const sb200_synth_config* cfgs, const float* scale_packed,
                                      const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                      const int64_t* blend_speakers, const float* blend_weights,
                                      const size_t* blend_offsets, sb200_latent** outs, sb200_error* err);
/* sb200_encode_batch_ids_blends with a target table (see sb200_speak_batch_ids_fit; NULL fit_offsets: none, that call
 * bit for bit): each latent's frames are fitted in the encoder pass, and its chunks then decode unchanged.
 * breaks_ms_packed (NULL: none, checked as sb200_speak_batch_ids_breaks checks them) are the pauses the latents'
 * prosody streams will insert; the fit counts them in P, and the pass inserts none.  fit_factor_out / fit_len_out as
 * there. */
int32_t sb200_encode_batch_ids_targets(sb200_voice* v, const int64_t* ids_packed, const size_t* offsets, size_t batch,
                                       const sb200_synth_config* cfgs, const float* scale_packed,
                                       const int32_t* frames_packed, const uint64_t* seeds, const int32_t* seeded,
                                       const int64_t* blend_speakers, const float* blend_weights,
                                       const size_t* blend_offsets, const float* breaks_ms_packed,
                                       const int64_t* fit_first, const int64_t* fit_end, const float* fit_ms,
                                       const size_t* fit_offsets, float* fit_factor_out, int64_t* fit_len_out,
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
/* ---- streams with a pitch contour (see sb200_speak_batch_ids_contour) ----
 * A prosody stream for latent z's sentence with pitch_per_id[0 .. n_ids) (one ratio per id of z, n_ids its id count;
 * values as for sb200_speak_batch_ids_contour, NaN or 1: none) and a tempo (NaN or 1: none).  Its plan is fixed at
 * creation from the latent's frames: n = 256 T_y inputs, id i ending at 256 C_i (C: cumulative frames), pieces, knots
 * and delivered ends as in sb200_speak_batch_ids_contour.  A bad ratio fails naming the id, a contour and tempo that
 * together ask for nothing, a wrong n_ids or another voice's latent fail too, all with OPERATION_ERROR before any device
 * work.  The piece table is uploaded once, into the stream's own allocation.
 * Contract: join the chunks a contoured stream emits through sb200_decode_chunks_warped; the result is, bit for bit,
 * sb200_debug_prosody_contour (n, ends = 256 C_i, the ratios and the tempo) of the joined samples appended to it (the
 * chunks after the post-path, as for a ratio stream), then resampled and converted as without a contour.  The joined
 * trimmed chunks of a stream cover frames [0, T_y) exactly, so the chunk that ends the stream must bring the total to
 * n and no chunk may take it past n; otherwise that pass fails with OPERATION_ERROR (internal) before any device work,
 * and the stream is left as it was.  A contour that merges into one piece
 * is the ratio stream of that pitch (same chunk counts, same bits).
 * Emission rule, generalising sb200_decode_chunks_warped's (which it is with one piece): pieces r = 1 .. m with knots
 * B, S, Q as in sb200_speak_batch_ids_contour, alpha_r = p_r / t, W_r = 16 / min(1, 1 / p_r) and W_max = max_r W_r; C
 * the inputs consumed.  a_k is step 2's (a_{-1} = -Hs) and frame K's delta is known once
 * max(a_{K-1} + D + Hs + N, a_K + D + N) <= C.  Stretched samples min(K Hs, floor(sigma(C) + 0.5)) are computed, where
 * sigma(C) = S_{r-1} + (C - B_{r-1}) * alpha_r in the piece with B_{r-1} <= C < B_r (sigma(n) = S_m).  Output j, at
 * step 3's pos_j in its piece r(j), is emitted once ceil(pos_j + W_{r(j)}) <= that count, as a prefix (W changes at a
 * piece's first output).  Between chunks the stream holds the inputs from max(0, min(a_{K-2} + Hs, a_{K-1}) - D) on,
 * fewer than max(ceil(2 Hs / alpha_min), Hs) + 2 D + N + 4 of them (alpha_min = min_r alpha_r), and the stretched
 * samples from floor(pos_J - W_max) + 1 on (J: the first output not emitted; a later output in a wider piece reaches
 * below pos_J - W_{r(J)}), at most 2 ceil(W_max) + 4 <= 68.  The last chunk emits everything up to n2.  Every
 * expression is evaluated as written, each operation rounded (no fused multiply-add). */
int32_t sb200_prosody_stream_create_contour(sb200_voice* v, const sb200_latent* z, const float* pitch_per_id,
                                            size_t n_ids, float tempo, sb200_prosody_stream** out, sb200_error* err);
/* Each id's delivered end (step 4 of sb200_speak_batch_ids_contour; after its pauses for a stream with breaks) at the
 * voice's rate, known at creation: the ends the batch path reports for the same latent.  out[0 .. n_ids); fails with
 * OPERATION_ERROR for a stream made without a contour or breaks, or a capacity below the id count. */
int32_t sb200_prosody_stream_bounds(const sb200_prosody_stream* s, int64_t* out, size_t capacity, sb200_error* err);
/* ---- streams with a formant ratio (see sb200_speak_batch_ids_formants) ----
 * A prosody stream with a formant ratio phi (NaN: none; else a finite value in [0.5, 2]) on top of a pitch ratio and a
 * tempo (pitch_per_id NULL: a ratio stream, z may be NULL), or of latent z's contour pitch_per_id[0 .. n_ids) and a
 * tempo (as sb200_prosody_stream_create_contour; pitch must then be NaN or 1), or of neither.  Unlike the other
 * creators it accepts ratios that ask for nothing when phi asks for something: a formant-only stream, which changes the
 * timbre of a plain stream.  The stage runs only when formant_asks holds: phi finite and some frame with p_m / phi != 1
 * (a contour stream knows n2 at creation); a stream whose phi asks for nothing (phi NaN, or equal to its pitch ratio
 * without a contour) is the stream without phi: the same chunk counts, bits and launches.  A bad phi fails naming it,
 * as do ratios and a phi that all ask for nothing and every failure of the other creators, all with OPERATION_ERROR
 * before any device work.  Lengths, sb200_prosody_stream_bounds and the delivered ends do not depend on phi.
 * Contract: join the chunks such a stream emits through sb200_decode_chunks_warped; the result is, bit for bit, the y
 * of sb200_debug_formant over the joined samples appended to the stream (the chunks after the post-path, as for a ratio
 * stream) with the stream's pitch, tempo, contour (ends = 256 C_i) and phi, then resampled and converted as without phi.
 * Emission rule: let G be the formant stage's inputs so far (the outputs the pitch stage has emitted or, without pitch
 * and tempo, the samples appended), N = 1024 and H = 256.  A chunk that does not end the stream emits the stage's outputs
 * [0, E), E = H max(0, floor((G - (N - H)) / H)): every hop whose 4 frames lie inside the input.  Those frames neither
 * read past G nor reach the clamp of their centres at n2 - 1, so nothing before the last chunk depends on n2.  The last
 * chunk emits everything up to n2, reading zeros past the end.  Between chunks the stream holds its inputs from
 * max(0, E - 3 H) on, fewer than N + 3 H = 1792 of them: the 3 H before E recompute the frames whose overlap-add
 * reaches E.  The stage holds back G - E = 768 .. 1023 samples on top of the pitch stage's hold-back (35 - 46 ms at
 * 22.05 kHz, 48 - 64 ms at 16 kHz).  A one-shot stream's single chunk is its last, so it emits everything. */
int32_t sb200_prosody_stream_create_formant(sb200_voice* v, const sb200_latent* z, float pitch,
                                            const float* pitch_per_id, size_t n_ids, float tempo, float formant,
                                            sb200_prosody_stream** out, sb200_error* err);
/* The "formant" device time (ms) of the last chunk pass the stream was in (0: its stage did not run). */
int32_t sb200_prosody_stream_profile_formant(const sb200_prosody_stream* s, float* formant_ms);
/* ---- streams with a volume contour (see sb200_speak_batch_ids_volume) ----
 * sb200_prosody_stream_create_formant with volume_db_per_id[0 .. n_ids) (NULL: none), one level per id of latent z
 * (required with a contour; n_ids its id count, shared with pitch_per_id when both are given).  Like the formant
 * creator it accepts ratios and a phi that ask for nothing when the contour asks for something: a volume-only stream.
 * A contour that asks for nothing gives the stream sb200_prosody_stream_create_formant gives: the same chunk counts,
 * bits and launches.  The ends and pieces are fixed at creation from the latent's frames (the ends the batch path
 * gives for the same latent, ratios and contour) and the piece table is uploaded once, into the stream's own
 * allocation.  A bad level fails naming the id, as do a wrong n_ids and another voice's latent, all with
 * OPERATION_ERROR before any device work.
 * Emission: G_j depends only on j and the ends, so the stage holds nothing back.  Every sample the stages before it
 * emit is scaled at its delivered position, in the chunk pass's region "volume", after "formant" and before
 * resampling and any meter.  Contract: join the chunks such a stream emits through sb200_decode_chunks_warped or
 * sb200_decode_chunks_metered; the result is, bit for bit, the batch contract applied to the joined chunks the same
 * stream yields without the contour, then resampled, metered and converted as without it. */
int32_t sb200_prosody_stream_create_volume(sb200_voice* v, const sb200_latent* z, float pitch,
                                           const float* pitch_per_id, size_t n_ids, float tempo, float formant,
                                           const float* volume_db_per_id, sb200_prosody_stream** out,
                                           sb200_error* err);
/* The "volume" device time (ms) of the last chunk pass the stream was in (0: its stage did not run). */
int32_t sb200_prosody_stream_profile_volume(const sb200_prosody_stream* s, float* volume_ms);
/* ---- streams with breaks (see sb200_speak_batch_ids_breaks) ----
 * sb200_prosody_stream_create_volume with breaks_ms_per_id[0 .. n_ids) (NULL: none), one break per id of latent z
 * (required with breaks).  Ratios, a phi and a volume contour that ask for nothing are accepted when a break asks: a
 * break-only stream.  Breaks that ask for nothing give the stream sb200_prosody_stream_create_volume gives.  The
 * positions and lengths are fixed at creation from the latent's frames and the table is uploaded once, into the
 * stream's own allocation; the stream must then be fed exactly its latent's frames.  A bad break fails naming the id.
 * Emission: with J the samples the stage has received so far, after every chunk pass it has emitted exactly
 * O(J) = J + sum of M_k over P_k <= J samples, so a chunk whose input reaches P_k emits break k's zeros in that pass; the
 * stage holds nothing back, adds no latency and changes no chunk count, and the last chunk brings the total to
 * n2 + D_m.  It runs in the chunk pass's region "break", after "volume" and before resampling and any meter.
 * Contract: join the chunks such a stream emits through sb200_decode_chunks_warped or sb200_decode_chunks_metered; the
 * result is, bit for bit, the batch contract applied to the joined chunks the same stream yields without breaks, then
 * resampled, metered and converted as without them.  sb200_prosody_stream_bounds gives E' for such a stream. */
int32_t sb200_prosody_stream_create_breaks(sb200_voice* v, const sb200_latent* z, float pitch,
                                           const float* pitch_per_id, size_t n_ids, float tempo, float formant,
                                           const float* volume_db_per_id, const float* breaks_ms_per_id,
                                           sb200_prosody_stream** out, sb200_error* err);
/* The "break" device time (ms) of the last chunk pass the stream was in (0: its stage did not run). */
int32_t sb200_prosody_stream_profile_breaks(const sb200_prosody_stream* s, float* break_ms);

/* ---- live loudness: a stream held to a target by a causal BS.1770 meter carried on the device ----
 * A loudness stream (a meter) belongs to a voice, and so to its device, and meters one delivered rate r.  Its target T
 * (LUFS) is finite and in [-70, 0]; its maximum gain M (dB) is finite and in [0, 40] (20 is the usual choice).  Its input
 * x_0, x_1, .. is the concatenation of the f32 samples that every chunk passed with it would deliver without it: after
 * the post-path (trims, crossfade), the prosody and formant stages and resampling, before the chunk's gain and before
 * conversion.  Across chunks, and across the sentences of one request, the signal just continues.
 * With S = (r + 5) / 10 and q_c the sum of y^2 over step c (samples [cS, (c + 1)S)) of the K-weighted signal, computed
 * as sb200_debug_loudness's kernel computes it (each step filtered from zero state to e_c, states chained as
 * s_{c+1} = A^S s_c + e_c, then y^2 summed in sample order from the true s_c; the same bits as the batch kernel's q_c):
 * - the reading at step boundary m >= 1 (time mS) uses x[0, mS) only.  For m >= 4 it is the gated integrated loudness
 *   L_m over blocks 0 .. m - 4 with the batch gates and reduction order: sb200_debug_loudness(x, mS, r), bit for bit.
 *   For 1 <= m <= 3, before the first 400 ms block exists, it is provisional:
 *   L_m = -0.691 + 10 log10((q_0 + .. + q_{m-1}) / (mS)), summed left to right, and -inf when that is <= -70 or the
 *   sum is 0.
 * - gains at the boundaries: a_0 = 1 for a new meter (a meter that continues keeps its last a); for m >= 1,
 *   a_m = a_{m-1} when L_m = -inf, else f32(min(10^((T - L_m)/20), 10^(M/20))), computed in double.
 * - sample i of step m >= 1 gets G_i = f32(a_{m-1} + (a_m - a_{m-1}) (i - mS + 1) / S), in double as written with each
 *   operation rounded: a linear ramp across each 100 ms step.  Step 0 gets a_0.  The output is
 *   y_i = clamp(x_i * G_i, -1, 1) (an f32 product); the meter counts the samples it clamped.
 * So G_i depends only on samples before mS: the meter holds nothing back and adds no latency, and every chunk delivers
 * exactly as many samples as it would without it.  The result does not depend on how the signal is chunked, or on what
 * shares the pass.  When a request ends at n samples, its last reading is the batch meter's L of x[0, floor(n/S) S).
 * The first 100 ms of a new meter play at gain 1, readings before 400 ms are provisional, and peaks are held by the
 * clamp, not by a look-ahead limiter.  A meter keeps q of at most 2^16 steps (about 109 minutes of audio).
 * out_rate: r (0: the voice's rate; else one of the output rates). */
typedef struct sb200_loudness_stream sb200_loudness_stream;
int32_t sb200_loudness_stream_create(sb200_voice* v, uint32_t out_rate, float target_lufs, float max_gain_db,
                                     sb200_loudness_stream** out, sb200_error* err);
void sb200_loudness_stream_free(sb200_loudness_stream* s);
/* The meter's last reading (LUFS; -inf before any or without one), its last gain a, the samples it has metered and
 * clamped, and the "loudness" device time (ms) of the last chunk pass it was in.  Any pointer may be NULL. */
int32_t sb200_loudness_stream_state(const sb200_loudness_stream* s, double* lufs, float* gain, int64_t* samples,
                                    int64_t* clipped, float* ms, sb200_error* err);
/* sb200_decode_chunks_warped with meters[k] (NULL entries: none; meters NULL: that call, bit for bit) metering chunk
 * k's delivered samples as above, in the pass's "loudness" region after resampling.  A metered chunk's gain[k] scales y
 * after the meter, in every format; its i16 is trunc(clamp(y * 32767)) at the fixed scale, not peak-normalised, and
 * G.711 encodes those samples.  Joined, what a metered stream delivers (f32) is, bit for bit,
 * sb200_debug_loudness_stream over the joined chunks the same stream delivers without a meter, however they are
 * chunked.  Each of these fails with OPERATION_ERROR naming the chunk, before any device work or state change: a meter
 * made for another voice, a meter used twice in one call, a chunk whose delivered rate is not the meter's, a meter
 * whose history would pass 2^16 steps. */
int32_t sb200_decode_chunks_metered(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi,
                                    const int64_t* trim_lo_frames, const int64_t* trim_hi_frames, size_t n, int32_t fade,
                                    const float* gain, sb200_resampler* const* resamplers,
                                    sb200_prosody_stream* const* warps, sb200_loudness_stream* const* meters,
                                    const int32_t* last, int32_t format, void** outs, size_t* lens, sb200_error* err);
/* Watermarked realtime streams.  sb200_watermark_stream_create reads the voice's watermark once: *out is a stream that
 * marks with that setting to its end, or NULL when the voice marks nothing (such a stream stays unmarked to its end).
 * out_rate: the stream's delivered rate (0: the voice's).  sb200_decode_chunks_marked is sb200_decode_chunks_metered
 * with one such stream (or NULL) per chunk: what the chunk delivers after resampling goes through the watermark stage
 * before its meter and conversion, at stream positions n counted from the stream's first delivered sample.  After a
 * pass in which a stream's stage has received J samples it has emitted floor(J / B) B of them (B = rate / 100), and
 * all of them once a chunk with last = 1 ends it: it holds back fewer than B samples, and its chunk count does not
 * change.  The joined chunks equal the whole-signal mark of the joined unmarked chunks, bit for bit.  A chunk's
 * stream must be delivered at the chunk's rate and may appear once per pass. */
typedef struct sb200_watermark_stream sb200_watermark_stream;
int32_t sb200_watermark_stream_create(sb200_voice* v, uint32_t out_rate, sb200_watermark_stream** out,
                                      sb200_error* err);
void sb200_watermark_stream_free(sb200_watermark_stream* s);
/* the "watermark" device time (ms) of the last chunk pass the stream was in; 19 for a null argument */
int32_t sb200_watermark_stream_profile(const sb200_watermark_stream* s, float* ms);
int32_t sb200_decode_chunks_marked(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi,
                                   const int64_t* trim_lo_frames, const int64_t* trim_hi_frames, size_t n, int32_t fade,
                                   const float* gain, sb200_resampler* const* resamplers,
                                   sb200_prosody_stream* const* warps, sb200_loudness_stream* const* meters,
                                   sb200_watermark_stream* const* marks, const int32_t* last, int32_t format, void** outs,
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
/* One stage of one chunk of sb200_debug_decode_chunks: rows x cols floats, time-major. */
typedef struct sb200_chunk_capture {
    char name[32];
    size_t chunk;         /* index of the chunk in the call */
    size_t rows, cols;
    float* data;
} sb200_chunk_capture;
/* Test hook: sb200_decode_chunks' pass over chunks zs[k] frames [lo[k], hi[k]) with every decoder stage captured; the
 * same kernels run and the waveforms are bit for bit that call's.  *caps receives *n_caps records, for each chunk in
 * order: "z" (the latent rows the pass gathered, [hi - lo][inter]), "dec.pre", "dec.up<i>", "dec.mrf<i>" (the names,
 * channel order and rows per frame of sb200_job_debug_fetch) and "wav" (the chunk's samples, one column).  Each holds
 * the chunk's own (hi - lo) * U rows.  Records and data are one malloc'ed block: free *caps with free(). */
int32_t sb200_debug_decode_chunks(sb200_voice* v, const sb200_latent* const* zs, const int64_t* lo, const int64_t* hi,
                                  size_t n, sb200_chunk_capture** caps, size_t* n_caps, sb200_error* err);

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
/* A fresh meter (see sb200_loudness_stream_create) at `rate` with target_lufs and max_gain_db on `device`, fed x in
 * chunks of chunk_lens[0 .. n_chunks) samples, one loudness launch per chunk: y receives the metered samples (as many as
 * x), lufs_steps / gain_steps every reading L_m and gain a_m, m = 1 .. floor(total / S), and *clipped the clamp count. */
int32_t sb200_debug_loudness_stream(int32_t device, const float* x, const size_t* chunk_lens, size_t n_chunks,
                                    int32_t rate, float target_lufs, float max_gain_db, float* y, double* lufs_steps,
                                    float* gain_steps, int64_t* clipped, sb200_error* err);
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
/* Test hook, no device needed: the plan of a pitch contour (see sb200_speak_batch_ids_contour) over n samples at `rate`
 * whose id i ends at input sample ends[i] (non-decreasing, the last one at n unless all are 0) with ratio ratios[i], and
 * the tempo: shape6 receives Hs, N, D, n1, n2, F, positions[0 .. min(F, cap)) the a_k and bounds[0 .. n_ids) (NULL: not
 * wanted) each id's delivered end.  Returns 0, or 19 for a bad ratio, tempo, end or rate. */
int32_t sb200_debug_prosody_contour_plan(int32_t rate, int64_t n, const int64_t* ends, const float* ratios, size_t n_ids,
                                         float tempo, int64_t* shape6, int64_t* positions, size_t cap, int64_t* bounds);
/* The prosody kernels over one caller buffer x[0 .. n) with that contour: y[0 .. n2), offsets[0 .. F) and
 * stretched[0 .. n1) as for sb200_debug_prosody, bit for bit what a job gives an utterance of those samples and ends. */
int32_t sb200_debug_prosody_contour(int32_t device, const float* x, size_t n, int32_t rate, const int64_t* ends,
                                    const float* ratios, size_t n_ids, float tempo, float* y, size_t cap,
                                    int32_t* offsets, size_t offsets_cap, float* stretched, size_t stretched_cap,
                                    sb200_error* err);
/* Test hook: the blended embedding g (gin floats) and the effective biases (cond_rows floats) a pass computes for the
 * blend of pairs (speakers[i], weights[i]), i < n, checked as in sb200_speak_batch_ids_blends, through the same launches:
 * bit for bit what a pass conditions on.  Fails when g_cap or bias_cap is too small. */
int32_t sb200_debug_speaker_blend(sb200_voice* v, const int64_t* speakers, const float* weights, size_t n, float* g,
                                  size_t g_cap, float* bias, size_t bias_cap, sb200_error* err);
/* The prosody chain and the formant stage over one caller buffer x[0 .. n) at `rate`: the pitch / tempo ratios (NaN or
 * 1: none) or, with ends and ratios (n_ids entries; pitch must then be NaN), that contour and the tempo, then formant
 * ratio phi.  pre[0 .. n2) receives the signal the formant stage reads, y[0 .. n2) its output (pre itself when the
 * stage does not run), n2_out the length; bit for bit what a job gives an utterance of those samples and ends. */
int32_t sb200_debug_formant(int32_t device, const float* x, size_t n, int32_t rate, float pitch, float tempo,
                            const int64_t* ends, const float* ratios, size_t n_ids, float phi, float* pre, float* y,
                            size_t cap, int64_t* n2_out, sb200_error* err);
/* The volume stage over one caller buffer x[0 .. n) at `rate`, whose id i ends at delivered sample ends[i]
 * (non-decreasing, the last at n) with levels[i] (n_ids entries, checked as sb200_speak_batch_ids_volume checks them):
 * y[0 .. n) receives the result, x itself when the pieces ask for nothing; bit for bit what a job gives an utterance
 * of those samples and ends. */
int32_t sb200_debug_volume(int32_t device, const float* x, size_t n, const int64_t* ends, const float* levels,
                           size_t n_ids, int32_t rate, float* y, sb200_error* err);
/* The break stage over one caller buffer x[0 .. n) at `rate`, whose id i ends at ends[i] (non-decreasing, the last at
 * n) with a break of ms[i] after it (n_ids entries, checked as sb200_speak_batch_ids_breaks checks them): *n_out
 * receives the paused length and y[0 .. *n_out) the result (cap: y's room; too little fails after *n_out is set); bit
 * for bit what a job gives an utterance of those samples and ends. */
/* The fit kernel over caller values: w[0 .. n) the ids' w_i, frames (NULL: all predicted) their fixed counts as
 * frames_packed, and n_spans spans [first[k], end[k]) with budget[k] = floor((T - P) / 256) frames.  factor[0 .. n)
 * receives the factor image (1 outside the spans), u_out / frames_out per span u* and its frames (L(u*) = 256 frames +
 * P); any output may be NULL.  Bit for bit what the synthesis path's fit does with those w. */
int32_t sb200_debug_fit(int32_t device, const float* w, size_t n, const int32_t* frames, const int64_t* first,
                        const int64_t* end, const int64_t* budget, size_t n_spans, float* factor, float* u_out,
                        int64_t* frames_out, sb200_error* err);
int32_t sb200_debug_breaks(int32_t device, const float* x, size_t n, const int64_t* ends, const float* ms, size_t n_ids,
                           int32_t rate, float* y, size_t cap, int64_t* n_out, sb200_error* err);
/* The watermark stage over one caller buffer x[0 .. n) delivered at `rate` (8000 .. 48000), marked with *wm (checked as
 * sb200_voice_set_watermark checks it): y[0 .. n) receives the result; bit for bit what a job gives an utterance of
 * those samples. */
int32_t sb200_debug_watermark(const float* x, size_t n, int32_t rate, const sb200_watermark* wm, float* y,
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
/* Test hook, no device needed: a contoured prosody stream (see sb200_prosody_stream_create_contour) over n inputs at
 * `rate` whose id i ends at ends[i], fed chunk_lens[0 .. n_chunks), the last one ending it.  counts[5 k .. 5 k + 5)
 * receives chunk k's outputs emitted, then the frames known, the stretched samples computed and the inputs and
 * stretched samples held after it.  Returns 0, or 19 for bad ratios or ends, a neutral contour and tempo, a bad rate,
 * a negative length or chunks that do not add up to n. */
int32_t sb200_debug_prosody_contour_stream_plan(int32_t rate, int64_t n, const int64_t* ends, const float* ratios,
                                                size_t n_ids, float tempo, const int64_t* chunk_lens, size_t n_chunks,
                                                int64_t* counts);
/* sb200_debug_prosody_stream for a fresh contoured stream over x[0 .. sum chunk_lens), n = sum chunk_lens, with those
 * ends, ratios and tempo. */
int32_t sb200_debug_prosody_contour_stream(int32_t device, const float* x, const int64_t* chunk_lens, size_t n_chunks,
                                           int32_t rate, const int64_t* ends, const float* ratios, size_t n_ids,
                                           float tempo, float* y, size_t cap, int64_t* lens, int32_t* offsets,
                                           size_t offsets_cap, sb200_error* err);
/* Test hook, no device needed: the samples a stream of sb200_prosody_stream_create_formant emits per chunk at `rate`,
 * with pitch and tempo, or (ends, ratios: n_ids entries; n_ids 0: none) a contour over n = sum chunk_lens inputs, and
 * formant ratio `formant`, when its chunks bring chunk_lens[0 .. n_chunks) inputs and the last one ends it.  emitted[k]
 * receives chunk k's count.  Fails with the creator's errors, or for a negative length. */
int32_t sb200_debug_formant_stream_plan(int32_t rate, float pitch, float tempo, const int64_t* ends, const float* ratios,
                                        size_t n_ids, float formant, const int64_t* chunk_lens, size_t n_chunks,
                                        int64_t* emitted, sb200_error* err);
/* That stream, fresh on `device`, fed x[0 .. sum chunk_lens) in those chunks with no decoder involved: y receives the
 * concatenated outputs (cap: its size) and lens[k] chunk k's count. */
int32_t sb200_debug_formant_stream(int32_t device, const float* x, const int64_t* chunk_lens, size_t n_chunks,
                                   int32_t rate, float pitch, float tempo, const int64_t* ends, const float* ratios,
                                   size_t n_ids, float formant, float* y, size_t cap, int64_t* lens, sb200_error* err);
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
