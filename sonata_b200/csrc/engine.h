// Host runtime of libsonata_b200: voice (weights + config), per-call contexts, batched job.
// This is the C++ stand-in for the reference's Rust `VitsModel` (piper/src/lib.rs:291-478): it
// owns what `ort::Session` owns there (weights, execution resources) and mirrors the model-side
// state (`ModelConfig`, `RwLock<PiperSynthesisConfig>`).
#pragma once
#include "common.cuh"
#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

namespace sb200 {

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define SB_CUDA(x)                                                                                       \
    do {                                                                                                 \
        cudaError_t e__ = (x);                                                                           \
        if (e__ != cudaSuccess)                                                                          \
            throw ::sb200::Error(19, std::string("CUDA error: ") + cudaGetErrorString(e__) + " at " +    \
                                         __FILE__ + ":" + std::to_string(__LINE__));                     \
    } while (0)

struct HostTensor {
    std::vector<int> dims;
    std::vector<float> f;
    std::vector<int> i;
    bool is_int = false;
    size_t numel() const { size_t n = 1; for (int d : dims) n *= (size_t)d; return n; }
};

struct Arch {
    int hidden, inter, filter, heads, layers, kernel, window, n_vocab, resblock, up_init, flow_n, wn_layers,
        flow_kernel, dp_kernel, dp_bins, sample_rate;
    std::vector<int> up_rates, up_kernels, res_kernels;
    std::vector<std::vector<int>> res_dils;
    int hop() const { int h = 1; for (int u : up_rates) h *= u; return h; }
};

// One convolution layer: its shape (conv_layout) and the weight images of the kernels that can run it.  A layer carries
// only the images of its kernels, and Runner::conv picks the kernel from the images it finds.
struct ConvW {
    float* w = nullptr;                      // fp32 [ntaps][cin][ldw] (conv_simt.cu); null on the phase-fused ConvTranspose
    float* bias = nullptr;
    float* wtc = nullptr; int tc_nt = 0;     // bf16 hi/lo swizzled weight images (conv_tc.cu): flow and decoder layers
    float* wtf = nullptr;                    // tf32 hi/lo images (conv_tf.cu): text-encoder / duration-predictor layers
    int cin = 0, cout = 0, ldw = 0, ntaps = 0;
    int macs = 0;                            // multiply-adds per output row (profile counters)
    int cond_off = -1;                       // multi-speaker voices: offset of this conv's per-call effective bias (Runner::cond)
    int tap_off[SB_MAX_TAPS] = {0};
    int min_off = 0, span = 0;
};

// Tap offsets (t - (k-1)/2) * dil, t < k, of a centred Conv1d of kernel size k.
std::vector<int> centred_taps(int k, int dil);
// The shape of a conv with taps `offs` and no weights: ntaps, tap_off, min_off, span, macs = ntaps * cin * cout, and ldw
// padded to conv_simt's column tile (pad_ldw) or equal to cout.
ConvW conv_layout(int cin, int cout, const std::vector<int>& offs, bool pad_ldw = true);
// Column tile of conv_tc's weight image for `cout` output columns; 0: the kernel takes no such layer.
int tc_tile_for(int cout);

// What a call site adds to a layer: input activation, epilogue and outputs (the ConvArgs fields of the same names).
struct ConvCall {
    float in_slope = 1.f; int act = ACT_NONE; float scale = 1.f;
    const float* res = nullptr; int ldres = 0;
    float* y0 = nullptr; int ldy0 = 0; int acc0 = 0; int split = -1;     // split < 0: every column goes to y0
    float* y1 = nullptr; int ldy1 = 0; int acc1 = 0;
    int orow_mul = 1, orow_add = 0;
    float* yt = nullptr; int yt_col0 = 0, ldyt = 0;     // conv_tf only: column tiles >= yt_col0 stored transposed
};
// Launch arguments of layer `w` over the rows of `map`, reading x [map.rows][ldx]; the bias is the layer's own.
ConvArgs conv_args(const ConvW& w, const float* x, int ldx, const RowMap& map, const ConvCall& c);

struct EncLayer { ConvW qkv, o, ffn1, ffn2; float *relk, *relv, *g1, *b1, *g2, *b2; };
struct DDSW { float* wdw[3]; float* bdw[3]; ConvW c1x1[3]; float *g1[3], *b1[3], *g2[3], *b2[3]; };
struct CFlowW { float* pre_w; float* pre_b; DDSW dds; ConvW proj; int ccol, tcol; };
struct CouplingW { ConvW pre; std::vector<ConvW> in, rs; ConvW post; int cond_off, tgt_off; };
struct ResBW { int k; std::vector<int> dils; std::vector<ConvW> c1, c2; };
// A ResBlock2 stage (branches res[b], convs c1[0] and c1[1]) of 64 channels as one launch (resblock_tc.cu):
// y = mean over b of x1_b + conv(lrelu(x1_b)), x1_b = x + conv(lrelu(x)), bit-identical to the six conv_tc launches.
// resblock2_tc_plan: false when the stage's shape is not one the kernel takes; out8 (or null) = {tile rows, x window
// rows, x1 rows, weight ring slots, dynamic shared memory bytes, grid CTAs for `rows`, threads, registers of one CTA}.
bool resblock2_tc_plan(const std::vector<ResBW>& res, int rows, int* out8);
void launch_resblock2_tc(const std::vector<ResBW>& res, const float* x, float* y, const RowMap& map, cudaStream_t st);
// phase: one fp32 conv per output phase (backend 0, or when fused has no image); fused: all phases as one N = u*cout
// conv with bf16 images only (backends 1 and 2)
struct UpStageW { int u, k, cin, cout; std::vector<ConvW> phase; ConvW fused; std::vector<ResBW> res; };

struct SynthConfig { long long speaker = 0; bool has_speaker = false; float noise_scale = 0.667f, length_scale = 1.f, noise_w = 0.8f; };

// resample_poly's default filter for in_rate -> out_rate (resample.cu): up / down the reduced ratio, H = 10 max(up, down)
// and 2H + 1 taps; on the device the taps are stored phase-major, K per phase (ResampleSeg).
struct ResampleFilter { int up = 1, down = 1, H = 0, K = 0; float* taps = nullptr; };
// The output rates a caller may ask for.  A rate of 0 or equal to the voice's own means no resampling.
bool output_rate_supported(long long rate);
// The filter's ratio and shape (no taps) for in_rate -> out_rate; throws OPERATION_ERROR prefixed by `who` when out_rate
// is not a supported rate or the ratio is too large for the kernel.  in_rate == out_rate is not a resampling ratio.
ResampleFilter resample_ratio(int in_rate, long long out_rate, const std::string& who);
// The 2H + 1 taps in natural order, designed in double (firwin with a Kaiser(5.0) window, times up), rounded to f32.
std::vector<float> resample_taps(int up, int down);
// The phase-major image of `h`: [up][K], zero past 2H.
std::vector<float> resample_phase_major(const std::vector<float>& h, int up, int K);

// Loudness normalisation (loudness.cu).  Rates the K-weighting filter is designed for: 8 kHz .. 384 kHz.
bool loudness_rate_supported(long long rate);
// Fills s.S = (rate + 5) / 10, the cascade s.k (libebur128's design in double) and s.AS = A^S; throws OPERATION_ERROR
// for an unsupported rate.
void loudness_design(long long rate, LoudSeg& s);
// Checks targets t[0 .. B) (null: none): NaN is no target, anything else must be finite and in [-70, 0] LUFS, or the
// call fails naming the utterance.  Returns whether some utterance has a target.
bool check_loudness_targets(const float* t, size_t B);

// Pitch and tempo (prosody.cu).  What one utterance of n samples at `rate` becomes with its two ratios: the WSOLA
// frame sizes (synthesis hop Hs = rate / 100, frame N = 2 Hs, search radius D = rate / 160), the stretch factor
// alpha = pitch / tempo, the stretched length n1 = floor(n alpha + 0.5) in F = ceil(n1 / Hs) frames (stage skipped when
// pitch == tempo: n1 = n, F = 0) and the delivered length n2 = floor(n1 / pitch + 0.5) (stage skipped when pitch is 1).
struct ProsodyShape { int Hs, N, D, F; long long n1, n2; bool stretch, pitch; double alpha, p; };
// NaN or 1 asks for nothing.  Throws OPERATION_ERROR for a rate without frame sizes or a result too long to index.
ProsodyShape prosody_shape(int rate, long long n, float pitch, float tempo);
// Checks pitch[0 .. B) and tempo[0 .. B) (either may be null): NaN or 1 is none, anything else must be finite and in
// [0.5, 2] (pitch) or [0.25, 4] (tempo), or the call fails naming the utterance.  Returns whether some utterance asks.
bool check_prosody(const float* pitch, const float* tempo, size_t B);
// The three prosody launches over segments laid out back to back: each segment's ProsodySeg, the sizes of the offsets,
// the stretched scratch and the output, what the launches are sized by and what the profile counts.
struct Voice;
struct ProsodyStream;
struct ProsodyStep;
struct ProsodyPlan {
    std::vector<ProsodySeg> segs;
    std::vector<ProsodyShape> shapes;
    long long s_total = 0, y_total = 0, d_total = 0, max_ola = 0, max_pitch = 0, steps = 0;
    long long in_total = 0, max_in = 0, max_keep = 0;     // streams: the input windows, the staging and carry sizes
    int smem_ints = 0;
    double stretch_flops = 0, stretch_bytes = 0, pitch_flops = 0, pitch_bytes = 0;
    // Appends the segment wav[in_off, in_off + n) with shape `sh`.
    void add(const ProsodyShape& sh, long long in_off, long long n);
    // Appends stream ps's window for its chunk pass step t; its input window goes to wav[in_total ..) of the pass.
    void add_stream(const ProsodyStream& ps, const ProsodyStep& t);
};

// One stream's pitch and tempo state (prosody.cu): the shape of its ratios, its counts (inputs consumed, frames whose
// delta is known, stretched samples computed, outputs emitted, and the history held of the inputs and the stretched
// signal) and, on the device, two sets of buffers read and written alternately: the input tail (at most cap_in), the
// stretched tail (at most cap_s, with both stages) and the deltas of the last two known frames.
struct ProsodyCounts { long long consumed = 0, frames = 0, stretched = 0, emitted = 0; int h_in = 0, h_s = 0; };
struct ProsodyStream {
    Voice* v = nullptr;
    int device = 0, rate = 0;
    float pitch = 1.f, tempo = 1.f;
    ProsodyShape sh{};                    // Hs, N, D, alpha, p and the stages (lengths unused)
    int cap_in = 0, cap_s = 0;
    void* mem = nullptr;
    float* in_hist[2] = {nullptr, nullptr}; float* s_hist[2] = {nullptr, nullptr}; int* d_hist[2] = {nullptr, nullptr};
    int cur = 0;
    ProsodyCounts c;
    bool ended = false;
    float last_ms[2] = {0.f, 0.f};        // the "stretch" and "pitch" device time of the last pass it was in
    ~ProsodyStream();
};
// What one chunk pass does to a stream: n_in new inputs, the frames [k0, k1), stretched samples [m0, m1) and outputs
// [j0, j1) it computes, the first absolute positions of its input and stretched windows (x0, s0), where the tails the
// next pass reads start (in_from, s_from), and the counts after it.  Computed on the host from the counts alone.
struct ProsodyStep {
    long long n_in, x0, s0, m0, m1, j0, j1, in_from, s_from;
    int k0, k1;
    ProsodyCounts next;
};
// Checks the ratios (one must ask for something) and sizes the history; no device memory.
void prosody_stream_init(ProsodyStream& ps, int rate, float pitch, float tempo);
ProsodyStream* create_prosody_stream(Voice* v, int device, int rate, float pitch, float tempo);
// The emission rule (include/sonata_b200.h, sb200_decode_chunks_warped).  Throws OPERATION_ERROR only on an internal
// inconsistency.
ProsodyStep prosody_stream_step(const ProsodyStream& ps, long long n_in, bool last);
// The stage / carry entry of chunk `chunk` for step t of ps.
ProsodyCarry prosody_carry(const ProsodyStream& ps, const ProsodyStep& t, int chunk);
// The launches of a stream pass's "stretch" region: staging, the offset chain, the overlap-add and the carry.  The
// pitch stage is launch_prosody_pitch over the same tables.
void launch_prosody_stream_stretch(const ProsodyPlan& p, const ProsodySeg* segs, const ProsodyCarry* cs,
                                   const float* src, const FrameSeg* fsegs, const PcmPost* posts, int hop, float* x,
                                   float* s, int* offsets, float* y, cudaStream_t st);
// After the pass has synchronised: the counts become t's and the buffers swap.
void prosody_stream_advance(ProsodyStream& ps, const ProsodyStep& t, bool last);
// Outputs per chunk of a stream with these ratios whose chunks bring chunk_lens[0 .. n) inputs, the last one ending it.
std::vector<long long> prosody_stream_plan(int rate, float pitch, float tempo, const long long* chunk_lens, size_t n);

struct Context;   // stream + arenas for one in-flight call

struct Voice {
    // ---- config (ModelConfig, piper/src/lib.rs:143-158) ----
    std::string config_path, key, quality, language_code, espeak_voice;
    int sample_rate = 22050;
    int num_speakers = 1;
    int num_symbols = 0;
    bool streaming = false;
    std::map<std::string, long long> speaker_id_map;
    std::unordered_map<uint32_t, long long> phoneme_first_id;   // char (code point) -> first id
    SynthConfig factory_cfg;
    mutable std::shared_mutex cfg_mu;     // RwLock<PiperSynthesisConfig> (piper/src/lib.rs:292)
    SynthConfig cfg;

    // ---- weights ----
    int device = 0;
    Arch a;
    std::vector<void*> dev_allocs;
    float* emb = nullptr;
    std::vector<EncLayer> enc;
    ConvW enc_proj;
    ConvW dp_pre, dp_proj;
    DDSW dp_dds;
    std::vector<CFlowW> dp_flows;   // in application order (CF4, CF3, CF2)
    float ea_m0 = 0, ea_logs0 = 0;
    std::vector<CouplingW> flows;   // in application order (f = n-1 .. 0)
    ConvW conv_pre;
    std::vector<UpStageW> ups;
    // multi-speaker conditioning (num_speakers > 1): see the end of load_voice
    float* emb_g = nullptr; int gin = 0, emb_rows = 0;
    float *cond_w = nullptr, *cond_base = nullptr; int cond_rows = 0;
    float* conv_post_w = nullptr;   // [7][C_last]
    int c_last = 0;

    int backend = 1;                // 1 (default): wgmma everywhere (bf16x2 split for flow + decoder, chunk-flushed 3xTF32 for the text
                                    // encoder + duration predictor); 2: wgmma flow + decoder, fp32 CUDA cores for encoder + predictor;
                                    // 0: fp32 CUDA cores everywhere.  Runner::conv applies it to the images each layer carries.
    unsigned long long noise_seed = 0x5eed5eedULL;
    std::mutex pool_mu;
    std::vector<Context*> pool;
    std::atomic<unsigned long long> call_counter{0};
    std::mutex rs_mu;
    std::map<long long, ResampleFilter> rs_filters;   // by output rate, taps on the device: built on first use

    ~Voice();
    Context* acquire();
    void release(Context* c);
    // Piper's [bos, (id, pad)*, eos] ids of a phoneme string.  src_char (optional) receives, per id, the index in
    // Unicode characters of the input character it came from (a pad belongs to the character before it; bos and eos
    // get -1).
    std::vector<long long> phonemes_to_ids(const char* utf8, std::vector<long long>* src_char = nullptr) const;
};

Voice* load_voice(const std::string& config_path, int device);
// The voice's filter to `out_rate` with its phase-major taps on the voice's device, built and cached on first use.
const ResampleFilter& voice_resampler(Voice& v, long long out_rate, const std::string& who);
ConvW debug_make_conv(Voice& v, const float* w, const float* bias, int cout, int cin, int k, int dil);

struct Region { std::string name; cudaEvent_t e0, e1; double flops = 0, bytes = 0; int launches = 0; float ms = 0; };

// Bump allocator over one device (or page-locked host) buffer.  A dry arena hands out no memory and only counts bytes:
// a workspace is carved once dry to learn its size, reserve()d, then carved for real (engine.cu plan()).
struct Arena {
    bool pinned = false;    // page-locked host memory instead of device memory
    bool dry = false;
    char* base = nullptr;
    size_t cap = 0, used = 0;
    void* alloc(size_t bytes) {
        const size_t a = (used + 255) & ~(size_t)255;
        used = a + bytes;
        if (dry) return nullptr;
        if (used > cap) throw Error(19, "internal: arena overflow");
        return base + a;
    }
    template <typename T> T* get(size_t n) { return reinterpret_cast<T*>(alloc(n * sizeof(T))); }
    void reserve(size_t bytes);   // empties the arena and makes room for `bytes` (growing frees the old buffer)
    void release();
};

struct Context {
    int device = 0;
    cudaStream_t stream = nullptr;
    Arena dev_id;       // id level of a pass: lives until the job is freed (stats, durations, speaker biases, captures)
    Arena dev_frame;    // frame level of a pass (latent, flow, decoder, waveforms), or one streaming decoder chunk
    Arena pin{true};    // page-locked staging: tables on the way in, results on the way out
    std::vector<cudaEvent_t> events; size_t events_used = 0;
    cudaEvent_t ev_begin = nullptr, ev_end = nullptr;
    cudaEvent_t next_event();
    ~Context();
};

struct Level {          // one time resolution of the packed batch
    RowMap map;
    long long valid_rows = 0;
    const int* bias_slot = nullptr;   // speaker slot of every granule (multi-speaker voices), for the conditioned convs
};

// The frame level of a pass, one segment per utterance (a job) or chunk (a chunk pass), and its speaker slots.
struct FrameLayout {
    std::vector<FrameSeg> fsegs;
    int RY = 0;
    long long total_samples = 0;
    std::vector<int> slot_of;         // per segment: its speaker slot (index into slot_sid; 0 on single-speaker voices)
    std::vector<int> slot_sid;        // per slot: the speaker id, distinct, in order of first use (empty: one speaker)
};

struct Job {
    Voice* v = nullptr;
    Context* ctx = nullptr;
    std::vector<SynthConfig> cfgs;    // one per utterance: the voice's fallback config unless set_job_configs changed it
    size_t B = 0;
    bool debug = false;
    bool encode_only = false;     // stop after the flow (streaming 'encoder.onnx' half)
    float* z_dev = nullptr;
    unsigned long long noise_call = 0;
    // host copies of inputs
    std::vector<long long> ids; std::vector<size_t> offs;
    // per-id duration controls, packed like ids (empty: none; set_job_durations)
    std::vector<float> dur_scale; std::vector<int> dur_frames;
    std::vector<int> id_frames;       // frames per id of the last run, packed like ids: filled by job_id_frames
    std::vector<std::vector<float>> eps_w, eps_z; std::vector<size_t> eps_z_frames;
    std::vector<NoiseSeed> seeds;     // one per utterance, empty when none is seeded (set_job_seeds)
    std::vector<int> out_rates;       // one per utterance, 0 = the voice's rate; empty when none resamples
                                      // (set_job_output_rates)
    std::vector<float> loud_target;   // one LUFS target per utterance, NaN = none; empty when none has one
                                      // (set_job_loudness)
    std::vector<float> pitch, tempo;  // one ratio per utterance each, NaN = none; both empty when no utterance asks
                                      // (set_job_prosody)
    std::vector<ProsodyShape> pros_ran;   // each utterance's shape in the last run (empty: it ran no prosody stage)
    // Loudness of the last run: the targets it ran with (empty: it measured nothing), each utterance's integrated
    // loudness and the gain applied to it
    std::vector<float> loud_ran; std::vector<double> loud_lufs; std::vector<float> loud_gain;
    // X layout
    int RX = 0; std::vector<SegInfo> xsegs; int max_tx = 0;
    // Y layout
    FrameLayout frames; std::vector<int> y_len;
    // tensor-core attention (conv_tf.cu grouped GEMMs): tile tables built with the X layout, same for every layer
    std::vector<TfTile> tiles_s, tiles_o;      // Q.K^T tiles, P.V tiles
    int att_tp = 0;                            // key columns of a score row (multiple of 96)
    int att_nth_s = 64, att_nth_o = 96;   // column tiles of the two attention GEMMs (narrower when the job is small)
    // device results read after the pass (context arenas)
    int* d_cum = nullptr;
    float* d_wav = nullptr;
    // What the job hands out: utterance b is d_wav[osegs[b].out_off ..) of osegs[b].len * out_hop samples, and
    // d_osegs mirrors osegs on the device.  Without prosody or output rates these are fsegs, the hop and total_samples;
    // with either, one segment of len = its delivered samples per utterance at out_hop = 1.
    std::vector<FrameSeg> osegs; int out_hop = 1; long long out_total = 0;
    std::vector<int> osr;             // sample rate of each handed-out utterance
    FrameSeg* d_osegs = nullptr;
    std::map<std::string, std::pair<float*, int>> dbg;   // name -> (device ptr, cols)
    std::map<std::string, int> dbg_level;                // name -> U (rows per frame), 0 for X level, -1 for an X-level
                                                         // buffer stored transposed ([cols][RX])
    std::vector<Region> regions;
    float last_ms = 0;
    bool ran = false;

    ~Job();
    void run(float* d_out, size_t d_out_cap);
};

Job* create_job(Voice* v, const long long* ids, const size_t* offs, size_t B, const float* const* eps_w,
                const float* const* eps_z, const size_t* eps_z_frames, bool debug);
// Checks a synthesis config against the voice like sb200_set_fallback_synthesis_config: a speaker, when given, must be
// a value of the voice's speaker_id_map.  `who` prefixes the error message.
void check_config(const Voice& v, const SynthConfig& c, const std::string& who);
// Per-utterance configs of the job's next run: cfgs[0 .. B), or the voice's fallback config for every utterance when
// cfgs is null.  Every entry is checked first; on an error the job keeps its configs.
void set_job_configs(Job& j, const SynthConfig* cfgs);
// Per-id duration controls of the job's next run, each packed like the job's ids (one entry per id) or null: scales
// (finite, >= 0) multiply the predicted duration before its ceil, frames (-1 = predicted, or >= 0) replace it.  Every
// entry is checked first; an error names the utterance and the id, and leaves the job's controls as they were.  Null
// and null restores the default (no controls, the kernel reads none).
void set_job_durations(Job& j, const float* scale, const int* frames);
// Per-utterance noise seeds of the job's next run: utterance b is seeded when seeded[b] is 1 (every utterance when
// seeded is null), and its eps_w / eps_z are then keyed draws of seeds[b] that do not depend on the batch
// (kernels_misc.cu randn_seg_kernel); seeded[b] = 0 keeps its positional noise.  Null seeds restores positional noise
// for all.  Flags other than 0 / 1, or seeds on a job with injected noise, fail naming the utterance and leave the job
// as it was.
void set_job_seeds(Job& j, const unsigned long long* seeds, const int* seeded);
// Per-utterance output rates of the job's next run (rates[0 .. B), 0 or the voice's rate: none), or null for none.
// Every entry is checked first; an unsupported rate fails naming the utterance and leaves the job's rates as they were.
void set_job_output_rates(Job& j, const unsigned* rates);
// Per-utterance loudness targets of the job's next run (targets[0 .. B), NaN: none), or null for none.  With a target,
// every utterance is measured after the decoder and any resampling, and those with one are scaled to it; see
// check_loudness_targets for the checks.  A bad entry leaves the job's targets as they were.
void set_job_loudness(Job& j, const float* targets);
// Per-utterance pitch and tempo ratios of the job's next run (each [0 .. B) or null; NaN or 1: none).  With a ratio, the
// utterance's waveform is time-stretched and pitch-resampled right after the decoder, before any resampling and
// loudness; see check_prosody for the checks.  A bad entry leaves the job's ratios as they were.
void set_job_prosody(Job& j, const float* pitch, const float* tempo);
// Frames per id of the job's last run, packed like its ids: one device->host copy of the batch's cum rows through the
// context's page-locked staging, differenced on the host.  Cached until the next run.
const std::vector<int>& job_id_frames(Job& j);

struct Latent {
    Voice* v = nullptr;
    long long sid = 0;    // speaker of the encoder pass (the reference hands `g` from encoder.onnx to decoder.onnx)
    std::shared_ptr<float> mem;   // device allocation shared by the latents of one encoder pass, freed with the last
    float* z = nullptr;   // device [frames][inter], inside `mem`
    long long frames = 0;
    std::vector<int> id_frames;   // frames per id of the encoder pass (the reference's p_duration)
};
// One encoder pass over B utterances (cfgs: one per utterance, or null for the voice's fallback config; scale / frames:
// per-id duration controls as for set_job_durations, or null; seeds / seeded: noise seeds as for set_job_seeds) -> B
// latents sharing one device allocation.  The caller owns the returned pointers.
std::vector<Latent*> encode_latents(Voice* v, const long long* ids, const size_t* offs, size_t B, const SynthConfig* cfgs,
                                    const float* scale = nullptr, const int* frames = nullptr,
                                    const unsigned long long* seeds = nullptr, const int* seeded = nullptr);
Latent* encode_latent(Voice* v, const long long* ids, size_t n);
// One stream's resampling state: the filter to its output rate, the last inputs (two device buffers of K floats each,
// read and written alternately), and how many inputs it has consumed and outputs it has emitted.
struct Resampler {
    Voice* v = nullptr;
    ResampleFilter f;
    float* hist[2] = {nullptr, nullptr};
    int cur = 0, h = 0;
    long long consumed = 0, emitted = 0;
    bool ended = false;
    ~Resampler();
};
Resampler* create_resampler(Voice* v, long long out_rate);
// Outputs of a stream whose first n inputs have arrived: all ceil(n * up / down) once it has ended, else those whose
// every input has arrived (j * down + H < n * up).
long long resample_emit_end(const ResampleFilter& f, long long n, bool ended);

// One chunk z[lo, hi) of a latent, and what its pass does to it before it leaves.
struct ChunkSpec {
    const Latent* z = nullptr; long long lo = 0, hi = 0;
    long long trim_lo = 0, trim_hi = 0;   // overlap frames dropped by the post-path
    float gain = 1.f;                     // linear gain of the post-path
    Resampler* rs = nullptr;              // the chunk's stream (resample passes; null: none)
    ProsodyStream* ps = nullptr;          // the chunk's pitch / tempo stream (resample passes; null: none)
    int last = 0;                         // 1: the chunk ends its stream, which is flushed
};
// One frame-level decoder pass over chunks of latents of one voice; chunk k equals the same chunk decoded alone, bit for
// bit.  Without `resample` or i16, a chunk leaves as the decoder's waveform, and its trims, gain and the fade must keep
// their defaults.  Otherwise the reference's post-path runs on the device per chunk: drop the trim frames,
// crossfade(fade) (samples.rs:144-157), the gain.  With `resample` the chunk is then appended to its stream's resampler,
// emitting every output it can (a chunk without one leaves at the voice's rate as the post-path leaves it); a resampler
// may appear once per pass and must belong to the voice.  A chunk with a prosody stream (resample passes only) is warped
// first, and what that stream emits is what the resampler, or the voice-rate copy, takes; the same rules hold for
// prosody streams.  i16: to_i16_vec (samples.rs:51-75) normalised to each emitted
// chunk's own peak; mu-law / A-law: the G.711 bytes of those same i16 samples, from the same launches.  Every check runs
// before any device work and any resampler changes; errors name the chunk, except with `single`, which keeps the
// single-chunk entry point's messages.
struct ChunkPass {
    std::vector<ChunkSpec> chunks;
    int fade = 0;
    bool resample = false;
    int format = 0;                       // PcmFormat: 0 f32, 1 i16, 2 mu-law, 3 A-law
    bool single = false;
};
struct ChunkResult {
    std::vector<std::vector<float>> f32;      // format 0
    std::vector<std::vector<int16_t>> i16;    // format 1
    std::vector<std::vector<uint8_t>> g711;   // formats 2 and 3
    float ms = 0;                             // the pass's device time
    float stretch_ms = 0, pitch_ms = 0;       // its "stretch" and "pitch" regions (0: none ran)
};
void decode_chunks(Voice* v, const ChunkPass& p, ChunkResult& out);

void job_pcm16(Job& j, float gain, std::vector<std::vector<int16_t>>& out);
// Peak-normalised 16-bit PCM of every utterance of a finished job (to_i16_vec after a linear gain), converted on the
// device and copied to `dst`: total_samples values laid out like the job's waveforms, in host memory that is best
// page-locked (a DMA copy).  An utterance the last run gave a loudness target converts at the fixed scale 32767.
void job_i16_to_host(Job& j, float gain, int16_t* dst);
// G.711 laws of the C ABI.
constexpr int G711_MULAW = 0, G711_ALAW = 1;
// The PcmFormat of G.711 law `law`; throws OPERATION_ERROR prefixed by `who` for any other value.
int g711_format(long long law, const std::string& who);
// job_i16_to_host's samples, utterance b after gains[b] (null: 1; each must be finite), encoded with G.711 law `law`
// in the same launches: one byte per sample in `dst`, laid out like the job's waveforms.  A bad law or gain fails
// before anything runs.
void job_g711_to_host(Job& j, int law, const float* gains, uint8_t* dst);
// One FLAC stream per utterance of a finished job (flac.cu): the 16-bit samples job_i16_to_host's conversion gives
// after gains[b] (null: 1; each must be finite), encoded on the device at the utterance's delivered rate.  outs[b]
// receives a malloc'ed buffer of lens[b] bytes.  A bad gain fails before anything runs.
void job_flac_to_host(Job& j, const float* gains, uint8_t** outs, size_t* lens);

// ---- FLAC (flac.cu) ----
constexpr int FLAC_STREAMINFO_BYTES = 42;   // `fLaC`, the block header and STREAMINFO
// One stream to encode: samples [off, off + n) of a device buffer of 16-bit samples, at `rate` Hz.
struct FlacStream { long long off = 0, n = 0; long long rate = 0; };
// Whether `rate` has a FLAC frame-header code here: the eight output rates.
bool flac_rate_supported(long long rate);
// A complete FLAC stream (RFC 9639 streamable subset; mono, 16 bits, blocks of 4096) of every entry of `streams`,
// encoded by the kernels of flac.cu on `st`: outs[s] receives a malloc'ed buffer of lens[s] bytes.  The size table is
// read back first, then only the compressed bytes.  An unsupported rate fails before any device work.
void flac_encode(const short* d_x, const std::vector<FlacStream>& streams, cudaStream_t st, uint8_t** outs,
                 size_t* lens);

}  // namespace sb200
