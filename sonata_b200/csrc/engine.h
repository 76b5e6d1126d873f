// Host runtime of libsonata_b200: voice (weights + config), per-call contexts, batched job.
// This is the C++ stand-in for the reference's Rust `VitsModel` (piper/src/lib.rs:291-478): it
// owns what `ort::Session` owns there (weights, execution resources) and mirrors the model-side
// state (`ModelConfig`, `RwLock<PiperSynthesisConfig>`).
#pragma once
#include "common.cuh"
#include <atomic>
#include <cmath>
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
    int yt_keep = 0;                                    // ... and also untransposed to y0
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

// A speaker blend in canonical form (include/sonata_b200.h, sb200_speak_batch_ids_blends): distinct speaker ids in
// ascending order, each with its normalised weight.  A plain speaker s is {s} with weight 1; empty: no blend.
struct SpeakerBlend {
    std::vector<int> s;
    std::vector<float> w;
    bool operator==(const SpeakerBlend& o) const { return s == o.s && w == o.w; }
    static SpeakerBlend plain(long long sid) { return SpeakerBlend{{(int)sid}, {1.f}}; }
};

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
// One stream's live loudness meter (include/sonata_b200.h, sb200_loudness_stream_create): its voice (null for a test
// hook's meter) and device, its delivered rate, target T and maximum gain M, the K-weighting design (d.S, d.k, d.AS);
// on the device two carries read and written alternately (the state at the last complete step boundary, 4 doubles,
// then the samples since it, S floats) and q of every complete step (LS_MAX_STEPS doubles), in one allocation; its
// counts, the gains at its last two boundaries and its last reading, and its "loudness" time of the last pass.
constexpr long long LS_MAX_STEPS = 1 << 16;
struct Voice;
struct LoudnessStream {
    Voice* v = nullptr;
    int device = 0;
    long long rate = 0;
    float target = 0.f, max_gain_db = 20.f;
    LoudSeg d{};
    void* mem = nullptr;
    double* carry[2] = {nullptr, nullptr};
    double* q = nullptr;
    int cur = 0;
    long long samples = 0, steps = 0, clipped = 0;
    float a_prev = 1.f, a = 1.f;
    double lufs = -INFINITY;
    float last_ms = 0.f;
    ~LoudnessStream();
};
// Checks T (finite, in [-70, 0]) and M (finite, in [0, 40]) and the rate, then allocates the meter's device state.
LoudnessStream* create_loudness_stream(Voice* v, int device, long long rate, float target, float max_gain_db);
// The steps a chunk of n more samples completes; throws OPERATION_ERROR prefixed by `who` when they would take the
// meter past LS_MAX_STEPS.
long long loudness_stream_steps(const LoudnessStream& s, long long n, const std::string& who);
// The chunk entry of n samples at y with gain `gain` after the meter; the scratch pointers (win, e, lufs, gains,
// clipped) are the caller's to set.
LoudStreamSeg loudness_stream_seg(const LoudnessStream& s, float* y, long long n, float gain);
// After the pass has synchronised: n samples more, the readings and gains of the boundaries it reached and the samples
// it clamped; the carries swap.
void loudness_stream_advance(LoudnessStream& s, long long n, const double* lufs, const float* gains,
                             unsigned long long clipped);

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
// Checks a pitch contour packed[0 .. offs[B]) of B utterances (utterance b: ids [offs[b], offs[b + 1])): NaN or 1 is
// none, anything else must be finite and in [0.5, 2], and an utterance with a contour must not also have a pitch ratio
// (pitch: one per utterance, or null), or the call fails naming the utterance (and the id).  Returns whether some
// utterance has a contour.
bool check_pitch_contour(const float* packed, const size_t* offs, size_t B, const float* pitch);
// The plan of one utterance of n samples whose id i ends at input sample ends[i] (non-decreasing; the last one at n
// unless every id is empty) with pitch ratio ratios[i] (NaN or 1: none; ratios null: the utterance ratio `pitch` for
// every id) and the utterance's tempo (include/sonata_b200.h, sb200_speak_batch_ids_contour).  Returns the shape;
// pieces receives the piece table and its sentinel when the ids make two or more pieces, and is emptied when they make
// one, which is planned as the utterance ratio it equals.  bounds[0 .. n_ids) (may be null) receives each id's delivered
// end.  Throws OPERATION_ERROR for bad ends, a rate without frame sizes or a result too long to index.
ProsodyShape prosody_contour_plan(int rate, long long n, const long long* ends, const float* ratios, size_t n_ids,
                                  float pitch, float tempo, std::vector<ContourPiece>& pieces, long long* bounds);
// The three prosody launches over segments laid out back to back: each segment's ProsodySeg, the sizes of the offsets,
// the stretched scratch and the output, what the launches are sized by and what the profile counts.  Segments with a
// contour add their piece tables to `pieces`, and the plan then needs a d_total table of analysis positions.
struct Voice;
struct ProsodyStream;
struct ProsodyStep;
// The canonical form of the blend of pairs (s[i], u[i]), i < n, on voice v; throws OPERATION_ERROR prefixed by `who`
// (naming the speaker or the weight) for an empty blend, a single-speaker voice, an unknown or repeated id, a weight that
// is negative or not finite, or weights that are all zero.
SpeakerBlend canonical_blend(const Voice& v, const long long* s, const float* u, size_t n, const std::string& who);
// The canonical blends of a blend table of B utterances or streams (utterance b: pairs [offs[b], offs[b + 1]); an empty
// range: no blend, an empty entry).  `what` names an entry in errors ("utterance", "stream").  Null tables: B empty
// entries.  Every entry is checked before anything is returned.
std::vector<SpeakerBlend> canonical_blends(const Voice& v, const long long* s, const float* u, const size_t* offs,
                                          size_t B, const std::string& what);
struct ProsodyPlan {
    std::vector<ProsodySeg> segs;
    std::vector<ProsodyShape> shapes;
    std::vector<ContourPiece> pieces;
    long long s_total = 0, y_total = 0, d_total = 0, max_ola = 0, max_pitch = 0, steps = 0;
    long long in_total = 0, max_in = 0, max_keep = 0;     // streams: the input windows, the staging and carry sizes
    int smem_ints = 0;
    bool contour = false;                                  // some segment has a contour: a d_total table of positions
    double stretch_flops = 0, stretch_bytes = 0, pitch_flops = 0, pitch_bytes = 0;
    // Appends the segment wav[in_off, in_off + n) with shape `sh` and, when it has one, its contour's piece table.
    void add(const ProsodyShape& sh, long long in_off, long long n, const std::vector<ContourPiece>* contour = nullptr);
    // Appends stream ps's window for its chunk pass step t; its input window goes to wav[in_total ..) of the pass.
    void add_stream(const ProsodyStream& ps, const ProsodyStep& t);
};

// Formant ratios (formant.cu).  Checks phi[0 .. B) (null: none): NaN is none, anything else must be finite and in
// [0.5, 2], or the call fails naming the utterance.  Returns whether some utterance has a ratio.  Unlike a pitch or tempo
// ratio, phi = 1 asks for something whenever the utterance has a pitch ratio or contour.
bool check_formants(const float* phi, size_t B);
// Whether an utterance of n samples after the pitch stage, with pitch ratio p (pc / c_n: its contour's pieces, c_n = 0
// for none) and formant ratio phi, runs the formant stage: phi is not NaN and some frame has p_m / phi != 1.
bool formant_asks(long long n, float phi, double p, const ContourPiece* pc, int c_n);
// The formant launch's segments, read from and written to the same offsets of two buffers laid out alike (the output
// of the stage before it, `total` samples), the copies of the utterances that do not ask ((offset, samples), adjacent
// ones merged), the CTA runs it is sized by and what the profile counts.
// A stream pass's plan instead holds one segment per stream: its window at in[off ..) (in_total samples in all, the
// largest max_in) and the hops it emits at out[y_off ..) (total samples), in runs of FM_STREAM_HOPS.
struct FormantStep;
struct FormantPlan {
    std::vector<FormantSeg> segs;
    std::vector<std::pair<long long, long long>> copies;
    long long total = 0, max_runs = 0;
    long long in_total = 0, max_in = 0;
    double flops = 0, bytes = 0;
    // Appends an utterance of n samples at offset `off` at the voice's `rate`, with its ratios (see FormantSeg).
    void add(int rate, long long off, long long n, float phi, double p, int c_off, int c_n);
    // Appends the copy of an utterance that does not ask.
    void copy(long long off, long long n);
    // Appends stream ps's window for its chunk pass step t.
    void add_stream(const ProsodyStream& ps, const FormantStep& t);
};

// One stream's pitch and tempo state (prosody.cu): the shape of its ratios, its counts (inputs consumed, frames whose
// delta is known, stretched samples computed, outputs emitted, and the history held of the inputs and the stretched
// signal) and, on the device, two sets of buffers read and written alternately: the input tail (at most cap_in), the
// stretched tail (at most cap_s, with both stages) and the deltas of the last two known frames.  A stream with a pitch
// contour knows its whole input length n_total and its plan (prosody_contour_plan) at creation: its piece table, when
// the contour makes two or more pieces, is resident on the device after the buffers (pieces_d); one piece is planned
// as the ratio stream it equals.
struct ProsodyCounts { long long consumed = 0, frames = 0, stretched = 0, emitted = 0; int h_in = 0, h_s = 0; };
struct ProsodyStream {
    Voice* v = nullptr;
    int device = 0, rate = 0;
    float pitch = 1.f, tempo = 1.f;
    ProsodyShape sh{};                    // Hs, N, D, alpha, p and the stages (lengths unused; a contour's: its plan's)
    int cap_in = 0, cap_s = 0;
    long long n_total = -1;               // a contour stream's input length (-1: a ratio stream)
    std::vector<ContourPiece> pieces;     // its piece table and sentinel (empty: one piece, or a ratio stream)
    std::vector<long long> bounds;        // its ids' delivered ends (empty: a ratio stream)
    double w_max = 0;                     // the widest pitch kernel radius of its pieces
    const ContourPiece* pieces_d = nullptr;
    void* mem = nullptr;
    float* in_hist[2] = {nullptr, nullptr}; float* s_hist[2] = {nullptr, nullptr}; int* d_hist[2] = {nullptr, nullptr};
    int cur = 0;
    ProsodyCounts c;
    bool ended = false;
    float last_ms[2] = {0.f, 0.f};        // the "stretch" and "pitch" device time of the last pass it was in
    // The formant stage (formant.cu): phi (NaN: none), whether the stage runs (formant_asks), its inputs taken (the
    // pitch stage's outputs, or the chunks' samples without pitch and tempo) and outputs emitted, the h carried inputs
    // [fm_in - fm_h, fm_in) in fm_hist[cur] (FM_CARRY floats each, after the prosody buffers) and its last region time.
    float formant = NAN;
    bool fm = false;
    long long fm_in = 0, fm_out = 0;
    int fm_h = 0;
    float* fm_hist[2] = {nullptr, nullptr};
    float last_fm_ms = 0.f;
    // The volume stage (volume.cu): the contour's pieces over the delivered samples, fixed at creation (empty: none),
    // resident on the device after the pitch contour's table (vol_d), and its last region time.
    std::vector<VolumePiece> vol;
    const VolumePiece* vol_d = nullptr;
    float last_vol_ms = 0.f;
    // The break stage (breaks.cu): the table of pauses over the delivered samples before them, fixed at creation
    // (empty: none), resident on the device after the volume table (brk_d); the stage's input length brk_n2, inputs
    // taken (J) and outputs emitted, and its last region time.
    std::vector<BreakPiece> brk;
    const BreakPiece* brk_d = nullptr;
    long long brk_n2 = 0, brk_in = 0, brk_out = 0;
    float last_brk_ms = 0.f;
    ~ProsodyStream();
};
// Whether stream ps runs the stretch or pitch stage (a formant-only stream runs neither).
inline bool prosody_stream_warps(const ProsodyStream& ps) { return ps.sh.stretch || ps.sh.pitch; }
// Volume contours (volume.cu).  Checks a volume contour packed[0 .. offs[B]) of B utterances or, with !per_utterance,
// of one stream: a level is NaN or 0 (none), -inf (silence) or a finite value in [-60, 20] dB, or the call fails naming
// the utterance (per_utterance) and the id.  Returns whether some level asks for something.
bool check_volume_contour(const float* packed, const size_t* offs, size_t B, bool per_utterance = true);
// The f32 gain of a level: 1 for NaN, 0 for -inf, else 10^(level / 20) in double.
float volume_gain_of(float level);
// The pieces of a signal of n2 delivered samples whose id i ends at ends[i] (non-decreasing, the last at n2) with
// levels[i] (include/sonata_b200.h, sb200_speak_batch_ids_volume): empty ids dropped, runs of equal levels merged.
// Empty when every piece has gain 1, which asks for nothing.  Throws OPERATION_ERROR for bad ends.
std::vector<VolumePiece> volume_pieces(const long long* ends, const float* levels, size_t n_ids, long long n2);
// The ramp's half length L / 2 = rate / 200 samples (about 5 ms).
inline int volume_half(int rate) { return rate / 200; }
// The volume launch's segments.  at[q]: a job's segment is in place at offset at[q] of the stage's input; a chunk
// pass's is chunk at[q], written at y_off[q] of the pass's own output (total samples).  A job's piece tables are laid
// out back to back in `pieces` (p_off[q]; -1: the segment's pc is already a stream's resident table).
struct VolumePlan {
    std::vector<VolumeSeg> segs;
    std::vector<long long> at, p_off, y_off;
    std::vector<VolumePiece> pieces;
    long long total = 0, max_n = 0;
    double bytes = 0;
    void add(long long at_, long long n, long long j0, int half, const std::vector<VolumePiece>& pc,
             const VolumePiece* pc_d = nullptr);
};
// Pauses (breaks.cu).  Checks breaks packed[0 .. offs[B]) of B utterances or, with !per_utterance, of one stream: a
// break is NaN or 0 (none) or a finite value in (0, 10000] ms, or the call fails naming the utterance (per_utterance)
// and the id.  Returns whether some break asks for something.
bool check_breaks(const float* packed, const size_t* offs, size_t B, bool per_utterance = true);
// The samples of a break of ms milliseconds at `rate`: floor(ms R / 1000 + 0.5) in double, 0 for none.
long long break_samples(float ms, int rate);
// The break table of a signal of n2 delivered samples whose id i ends at ends[i] (non-decreasing, the last at n2) with
// a break of ms[i] after it (include/sonata_b200.h, sb200_speak_batch_ids_breaks): breaks of 0 samples dropped, those
// at equal positions merged.  Empty when none asks.  Throws OPERATION_ERROR, prefixed by `who`, for bad ends and for a
// paused length past 2^31 - 1.
std::vector<BreakPiece> break_plan(const long long* ends, const float* ms, size_t n_ids, long long n2, int rate,
                                   const std::string& who);
// The samples the breaks at or before input position pos add: sum of M_k over P_k <= pos.
long long break_shift(const std::vector<BreakPiece>& bk, long long pos);
// The break launch's segments.  at[q]: a job's segment reads offset at[q] of the stage's input; a chunk pass's is
// chunk at[q].  Every segment writes at y_off[q] of the stage's own output (total samples).  A job's tables are laid out
// back to back in `pieces` (p_off[q]; -1: the segment's table is already a stream's resident one).
struct BreakPlan {
    std::vector<BreakSeg> segs;
    std::vector<long long> at, p_off, y_off;
    std::vector<BreakPiece> pieces;
    long long total = 0, max_n = 0;
    double bytes = 0;
    // Appends a segment of n_in inputs from input position j0 that emits outputs [o0, o0 + n_out).
    void add(long long at_, long long n_in, long long j0, long long o0, long long n_out, int half,
             const std::vector<BreakPiece>& bk, const BreakPiece* bk_d = nullptr);
};

// The most inputs a formant stream carries between passes: fewer than N, and the 3 H that recompute the frames before
// its next hop.
constexpr int FM_CARRY = FM_N + 3 * FM_H;
// What one chunk pass does to a stream's formant stage (include/sonata_b200.h, sb200_prosody_stream_create_formant): its
// inputs become g1, it emits hops [h0, h1) (outputs [e0, e1)) and the next pass carries its inputs from `from` on.
struct FormantStep { long long g1, h0, h1, e0, e1, from; };
FormantStep formant_stream_step(const ProsodyStream& ps, long long g1, bool last);
// The stage / carry entry of chunk `chunk` for step t of ps; direct: where its new inputs are (the pitch stage's output),
// or null for the chunk's samples after the post-path.
FormantCarry formant_carry(const ProsodyStream& ps, const FormantStep& t, int chunk, const float* direct);
// The launches of a stream pass's "formant" region: the staging (and carry), then the stage over every window.
void launch_formant_stream(const FormantPlan& p, const FormantSeg* segs, const FormantCarry* cs, const float* src,
                           const FrameSeg* fsegs, const PcmPost* posts, int hop, float* win, float* y, cudaStream_t st);
// After the pass has synchronised: the stage's counts become t's (prosody_stream_advance swaps the buffers).
void formant_stream_advance(ProsodyStream& ps, const FormantStep& t);
// What one chunk pass does to a stream: n_in new inputs, the frames [k0, k1), stretched samples [m0, m1) and outputs
// [j0, j1) it computes, the first absolute positions of its input and stretched windows (x0, s0), where the tails the
// next pass reads start (in_from, s_from), and the counts after it.  Computed on the host from the counts alone.
struct ProsodyStep {
    long long n_in, x0, s0, m0, m1, j0, j1, in_from, s_from;
    int k0, k1;
    ProsodyCounts next;
};
// Checks the ratios (one must ask for something unless allow_none) and sizes the history; no device memory.
void prosody_stream_init(ProsodyStream& ps, int rate, float pitch, float tempo, bool allow_none = false);
ProsodyStream* create_prosody_stream(Voice* v, int device, int rate, float pitch, float tempo);
// The same for a pitch contour of n_ids ids over n inputs (ends, ratios: as for prosody_contour_plan) and a tempo:
// checks them as check_pitch_contour and check_prosody do (a contour and tempo that ask for nothing are refused), plans
// the pieces and the bounds, and sizes the history by the smallest stretch factor and the widest pitch kernel.
void prosody_stream_init_contour(ProsodyStream& ps, int rate, long long n, const long long* ends, const float* ratios,
                                 size_t n_ids, float tempo, bool allow_none = false);
// A stream with a formant ratio phi (NaN: none) on top of a pitch ratio and a tempo (ratios null) or of a contour of
// n_ids ids over n inputs and a tempo: the checks of the two above, which here accept ratios that ask for nothing when
// phi asks, and phi's own (finite, in [0.5, 2]); a pitch ratio beside a contour, and a stream that asks for nothing at
// all, are refused.
void prosody_stream_init_formant(ProsodyStream& ps, int rate, long long n, const long long* ends, const float* ratios,
                                 size_t n_ids, float pitch, float tempo, float phi, bool allow_none = false);
// The same with a volume contour levels[0 .. n_ids) (null: none) over the stream's delivered samples, with ends
// (n_ids ids over n inputs, required with levels) giving each id's delivered end as prosody_contour_plan does: the
// checks of check_volume_contour, and ratios and a phi that ask for nothing are accepted when the contour asks.
void prosody_stream_init_volume(ProsodyStream& ps, int rate, long long n, const long long* ends, const float* ratios,
                                size_t n_ids, float pitch, float tempo, float phi, const float* levels,
                                bool allow_none = false);
// The same with breaks ms[0 .. n_ids) (null: none) after the ids (ends required with breaks): the checks of
// check_breaks, and ratios, a phi and a contour that ask for nothing are accepted when a break asks.  The table is
// planned over the delivered ends before breaks, and bounds becomes the ends after them.
void prosody_stream_init_breaks(ProsodyStream& ps, int rate, long long n, const long long* ends, const float* ratios,
                                size_t n_ids, float pitch, float tempo, float phi, const float* levels,
                                const float* ms);
ProsodyStream* create_prosody_stream_breaks(Voice* v, int device, int rate, long long n, const long long* ends,
                                            const float* ratios, size_t n_ids, float pitch, float tempo, float phi,
                                            const float* levels, const float* ms);
ProsodyStream* create_prosody_stream_volume(Voice* v, int device, int rate, long long n, const long long* ends,
                                            const float* ratios, size_t n_ids, float pitch, float tempo, float phi,
                                            const float* levels);
ProsodyStream* create_prosody_stream_formant(Voice* v, int device, int rate, long long n, const long long* ends,
                                             const float* ratios, size_t n_ids, float pitch, float tempo, float phi);
// Outputs per chunk of fresh stream ps (no device memory) fed chunk_lens[0 .. n), the last one ending it: what its
// formant stage emits when it runs, else what its pitch stage emits.
std::vector<long long> formant_stream_counts(ProsodyStream& ps, const long long* chunk_lens, size_t n);
ProsodyStream* create_prosody_stream_contour(Voice* v, int device, int rate, long long n, const long long* ends,
                                             const float* ratios, size_t n_ids, float tempo);
// The emission rule (include/sonata_b200.h, sb200_decode_chunks_warped).  Throws OPERATION_ERROR only on an internal
// inconsistency.
ProsodyStep prosody_stream_step(const ProsodyStream& ps, long long n_in, bool last);
// The stage / carry entry of chunk `chunk` for step t of ps.
ProsodyCarry prosody_carry(const ProsodyStream& ps, const ProsodyStep& t, int chunk);
// The launches of a stream pass's "stretch" region: staging, the offset chain, the overlap-add and the carry.  The
// pitch stage is launch_prosody_pitch over the same tables.
void launch_prosody_stream_stretch(const ProsodyPlan& p, const ProsodySeg* segs, const ProsodyCarry* cs,
                                   const float* src, const FrameSeg* fsegs, const PcmPost* posts, int hop, float* x,
                                   float* s, int* offsets, float* y, cudaStream_t st, long long* apos = nullptr);
// After the pass has synchronised: the counts become t's and the buffers swap.
void prosody_stream_advance(ProsodyStream& ps, const ProsodyStep& t, bool last);
// Outputs per chunk of a stream with these ratios whose chunks bring chunk_lens[0 .. n) inputs, the last one ending it.
std::vector<long long> prosody_stream_plan(int rate, float pitch, float tempo, const long long* chunk_lens, size_t n);
// The counts after each chunk of stream ps (fresh, no device memory) fed chunk_lens[0 .. n): 5 per chunk (outputs
// emitted, frames, stretched samples, input and stretched history held).
std::vector<long long> prosody_stream_counts(ProsodyStream& ps, const long long* chunk_lens, size_t n);

// The watermark (watermark.cu; include/sonata_b200.h, sb200_voice_set_watermark): key, payload, strength and the key's
// chip tables on the voice's device (c0 then c1, WM_P signed chars each).
constexpr int WM_P = 4096;
struct Watermark {
    unsigned long long key = 0;
    int payload = 0;
    float strength_db = 0.f;
    const signed char* chips = nullptr;
};
// One stream's watermark (include/sonata_b200.h, sb200_watermark_stream_create): the voice's setting when the stream was
// made, its delivered rate and block, the inputs it has received and the outputs it has emitted (a multiple of blk
// until the last chunk), and on the device two sets, read and written alternately, of the held inputs (fewer than blk)
// and the S of the last block emitted.
struct WatermarkStream {
    Voice* v = nullptr;
    Watermark wm;
    long long rate = 0, blk = 0, in = 0, out = 0;
    void* mem = nullptr;
    float* hold[2] = {nullptr, nullptr};
    long long* s[2] = {nullptr, nullptr};
    int cur = 0;
    bool ended = false;
    float last_ms = 0.f;
    ~WatermarkStream();
};
// The stream of voice v delivered at `rate`: null when the voice does not mark.
WatermarkStream* create_watermark_stream(Voice* v, long long rate);
// Checks a payload in [0, WM_P) and a finite strength in [-40, -10] dB; an error names the field.
void check_watermark(long long payload, float strength_db);
// The key's chip tables, built on the current device in memory the caller frees (cudaFree).
signed char* build_watermark_chips(unsigned long long key);

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
    // under cfg_mu: the watermark when wm_on, and the chip tables of every key ever set (in dev_allocs), kept because
    // a job that started under an earlier key may still read its table
    bool wm_on = false;
    Watermark wm;
    std::map<unsigned long long, const signed char*> wm_chips;

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

// Each workspace hands out its buffers in one carve(dev, pin).  plan() runs it on dry arenas to learn the sizes, makes
// room in the arenas and carves again for real, so no size is written down twice.
template <typename Carve> void plan(Arena& dev, Arena& pin, Carve&& carve) {
    Arena dry_dev, dry_pin;
    dry_dev.dry = dry_pin.dry = true;
    carve(dry_dev, dry_pin);
    dev.reserve(dry_dev.used);
    pin.reserve(dry_pin.used);
    carve(dev, pin);
}

// A table the host fills and the device reads, or the reverse: the device table `d` and its page-locked mirror `h`,
// carved together with one element count, so every copy moves exactly the carved table.  Unset (null) when not carved.
template <typename T> struct Staged {
    T* d = nullptr; T* h = nullptr; size_t n = 0;
    void carve(Arena& dev, Arena& pin, size_t count) { n = count; d = dev.get<T>(n); h = pin.get<T>(n); }
    void upload(cudaStream_t st) const { SB_CUDA(cudaMemcpyAsync(d, h, n * sizeof(T), cudaMemcpyHostToDevice, st)); }
    void download(cudaStream_t st) const { SB_CUDA(cudaMemcpyAsync(h, d, n * sizeof(T), cudaMemcpyDeviceToHost, st)); }
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

// The profile of a pass: each region between begin() and end() records its device time on a pair of the context's
// events and counts the flops, bytes and launches of the launches made inside it.  Without a region list it records
// nothing (the test hooks).
struct Profile {
    Context* c = nullptr; std::vector<Region>* regions = nullptr; cudaStream_t st = nullptr;
    Region* cur = nullptr;
    void begin(const std::string& name);
    void end();
    void count(double flops, double bytes, int launches = 1) {
        if (cur) { cur->flops += flops; cur->bytes += bytes; cur->launches += launches; }
    }
    // After the pass has synchronised: the device time of the region `name` (0 when none ran).
    float ms(const std::string& name) const;
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
    std::vector<int> slot_of;         // per segment: its speaker slot (index into slot_spk; 0 on single-speaker voices)
    std::vector<SpeakerBlend> slot_spk;   // per slot: the canonical blend, distinct, in order of first use (empty: one
                                          // speaker); a plain speaker is the blend of itself
    // Whether some slot blends two or more speakers: only then does the pass form its embeddings in a blend table.
    bool blended() const {
        for (const SpeakerBlend& b : slot_spk)
            if (b.s.size() > 1) return true;
        return false;
    }
};

// One span of a target table (include/sonata_b200.h, sb200_speak_batch_ids_fit): ids [first, end) of its utterance and
// the duration in ms they should take (NaN: none).
struct FitTarget { long long first, end; float ms; };

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
    std::vector<float> contour;       // per-id pitch ratios, packed like ids, NaN or 1 = none; empty when no utterance
                                      // has a contour (set_job_pitch_contour)
    std::vector<float> formant;       // one formant ratio per utterance, NaN = none; empty when none has one
                                      // (set_job_formants)
    std::vector<float> volume;        // per-id levels in dB, packed like ids, NaN or 0 = none; empty when no utterance
                                      // has a volume contour (set_job_volume_contour)
    std::vector<float> breaks;        // per-id pauses in ms, packed like ids, NaN or 0 = none; empty when no utterance
                                      // has one (set_job_breaks)
    std::vector<FitTarget> targets;   // target durations: each utterance's spans, target_offs[b] .. target_offs[b + 1];
    std::vector<size_t> target_offs;  // both empty when no span asks (set_job_targets)
    std::vector<float> fit_u;         // per span of the last run's targets: u* and L(u*) in samples at the voice's
    std::vector<long long> fit_len;   // rate (NaN and -1 for a span that asked nothing); empty when it had none
    std::vector<SpeakerBlend> blends; // one canonical blend per utterance (empty entry: the config's speaker); empty when
                                      // none has one (set_job_blends)
    bool wm_on = false;               // the voice's watermark, read when the run starts
    Watermark wm;
    std::vector<ProsodyShape> pros_ran;   // each utterance's shape in the last run (empty: it ran no prosody stage)
    std::vector<float> pitch_ran, tempo_ran;   // the ratios the last run had (empty: none)
    std::vector<long long> pros_bounds;   // each id's delivered end in the last run when it had a contour, a volume
                                          // contour or breaks (after its pauses; else empty)
    // Loudness of the last run: the targets it ran with (empty: it measured nothing), each utterance's integrated
    // loudness and the gain applied to it
    std::vector<float> loud_ran; std::vector<double> loud_lufs; std::vector<float> loud_gain;
    // X layout
    int RX = 0; std::vector<SegInfo> xsegs;
    // Y layout
    FrameLayout frames; std::vector<int> y_len;
    // tensor-core attention (conv_tf.cu grouped GEMMs): tile tables built with the X layout, same for every layer, of
    // the utterances of at most ATT_TC_MAX ids (the only ones the path takes: Job::run)
    std::vector<TfTile> tiles_s, tiles_o;      // Q.K^T tiles, P.V tiles
    int att_tc_len = 0;                        // the longest of those utterances (0: none)
    int att_tp = 0;                            // key columns of a score row (multiple of 64)
    int att_nth_s = 64, att_nth_o = 96;   // column tiles of the two attention GEMMs (narrower when the job is small)
    // device results read after the pass (context arenas)
    int* d_cum = nullptr;
    float* d_wav = nullptr;
    // What the job hands out: utterance b is d_wav[osegs[b].out_off ..) of osegs[b].len * out_hop samples, and
    // d_osegs mirrors osegs on the device.  Without prosody or output rates these are fsegs, the hop and total_samples;
    // with either, one segment of len = its delivered samples per utterance at out_hop = 1.
    std::vector<FrameSeg> osegs; int out_hop = 1; long long out_total = 0;
    std::vector<int> osr;             // sample rate of each handed-out utterance
    const FrameSeg* d_osegs = nullptr;
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
// Per-id pitch ratios of the job's next run, packed like its ids (NaN or 1: none), or null for none; see
// check_pitch_contour for the checks, which also refuse an utterance with a pitch ratio.  A bad entry leaves the job's
// contour as it was.  Each utterance with a contour runs the prosody stage with its pieces (prosody_contour_plan).
void set_job_pitch_contour(Job& j, const float* packed);
// Per-utterance formant ratios of the job's next run (phi[0 .. B), NaN: none), or null for none; see check_formants.
// An utterance that asks (formant_asks) runs the formant stage after the pitch stage, before any resampling and
// loudness; its length, bounds, alignments and place in the job's result do not change.  A bad entry leaves the job's
// ratios as they were.
void set_job_formants(Job& j, const float* phi);
// Per-id volume levels of the job's next run, packed like its ids (NaN or 0: none), or null for none; see
// check_volume_contour.  A bad entry leaves the job's contour as it was.  Each utterance whose pieces (volume_pieces,
// over its ids' delivered ends) ask runs the volume stage after the formant stage, before any resampling and loudness.
void set_job_volume_contour(Job& j, const float* packed);
// Per-id breaks of the job's next run in ms, packed like its ids (NaN or 0: none), or null for none; see check_breaks.
// A bad entry leaves the job's breaks as they were.  When some utterance's breaks ask for samples, every utterance runs
// the break stage after the volume stage, before any resampling and loudness, and its length, bounds and place in the
// job's result count its pauses.
void set_job_breaks(Job& j, const float* packed);
// Target durations of the job's next run: spans [first[k], end[k]) of ids with ms[k] each, utterance b's spans being
// k in [fit_offs[b], fit_offs[b + 1]), or null fit_offs for none; see check_targets.  A bad entry leaves the job's
// targets as they were.  The run fits each span that asks between the duration predictor and the durations' scan
// (fit_kernel) and keeps u* and L(u*) of every span in fit_u / fit_len.
void set_job_targets(Job& j, const long long* first, const long long* end, const float* ms, const size_t* fit_offs);
// Checks a target table of B utterances (offs: their id offsets) or, with !per_utterance, of one stream: spans
// non-empty, inside the utterance, ascending and disjoint; ms NaN (none) or a finite value in (0, 600000]; no span
// that asks on an utterance whose tempo[b] (null: none) asks.  Errors name the utterance and the span.  Returns whether
// some span asks.
bool check_targets(const long long* first, const long long* end, const float* ms, const size_t* fit_offs,
                   const size_t* offs, size_t B, const float* tempo, bool per_utterance = true);
// The samples of a target of ms milliseconds at `rate`: floor(ms R / 1000 + 0.5) in double.
long long target_samples(float ms, int rate);
// The fit launch of job j: the spans that ask, each with its break samples P and its index into j.targets.
struct FitPlan {
    std::vector<FitSpan> spans;
    std::vector<long long> pause;
    std::vector<size_t> index;
};
FitPlan fit_plan(const Job& j);
// Per-utterance speaker blends of the job's next run (a blend table as for canonical_blends), or null for none.  A blend
// replaces the utterance's config speaker; its noise and length scales still apply.  Every entry is checked first; a bad
// entry fails naming the utterance and leaves the job's blends as they were.
void set_job_blends(Job& j, const long long* s, const float* u, const size_t* offs);
// The blended embedding g [gin] and effective biases [cond_rows] a pass computes for blend b, through the pass's own
// launches, copied to the host.
void debug_speaker_blend(Voice& v, const SpeakerBlend& b, std::vector<float>& g, std::vector<float>& bias);
// Each id's delivered end (prosody_contour_plan) in the job's last run, packed like its ids, at the voice's rate: kept
// from the run when it had a contour, else computed from job_id_frames and the ratios it had.
std::vector<long long> job_prosody_bounds(Job& j);
// Frames per id of the job's last run, packed like its ids: one device->host copy of the batch's cum rows through the
// context's page-locked staging, differenced on the host.  Cached until the next run.
const std::vector<int>& job_id_frames(Job& j);

struct Latent {
    Voice* v = nullptr;
    SpeakerBlend spk;     // canonical blend of the encoder pass, the plain config speaker's without one (the reference
                          // hands `g` from encoder.onnx to decoder.onnx); its chunk passes condition on it
    std::shared_ptr<float> mem;   // device allocation shared by the latents of one encoder pass, freed with the last
    float* z = nullptr;   // device [frames][inter], inside `mem`
    long long frames = 0;
    std::vector<int> id_frames;   // frames per id of the encoder pass (the reference's p_duration)
};
// One encoder pass over B utterances (cfgs: one per utterance, or null for the voice's fallback config; scale / frames:
// per-id duration controls as for set_job_durations, or null; seeds / seeded: noise seeds as for set_job_seeds) -> B
// latents sharing one device allocation.  The caller owns the returned pointers.
// blend_s / blend_u / blend_offs: speaker blends as for set_job_blends, or null.  fit_*: target durations as for
// set_job_targets (their u* and L(u*) into fit_u / fit_len when given), with `breaks` (per id, as for set_job_breaks)
// counted in each span's P: the breaks its latent's prosody stream will insert.
std::vector<Latent*> encode_latents(Voice* v, const long long* ids, const size_t* offs, size_t B, const SynthConfig* cfgs,
                                    const float* scale = nullptr, const int* frames = nullptr,
                                    const unsigned long long* seeds = nullptr, const int* seeded = nullptr,
                                    const long long* blend_s = nullptr, const float* blend_u = nullptr,
                                    const size_t* blend_offs = nullptr, const float* breaks = nullptr,
                                    const long long* fit_first = nullptr, const long long* fit_end = nullptr,
                                    const float* fit_ms = nullptr, const size_t* fit_offs = nullptr,
                                    float* fit_u = nullptr, long long* fit_len = nullptr);
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
    LoudnessStream* ls = nullptr;         // the chunk's live loudness meter (resample passes; null: none)
    WatermarkStream* ws = nullptr;        // the chunk's watermark (resample passes; null: none)
    int last = 0;                         // 1: the chunk ends its stream, which is flushed
};
// One frame-level decoder pass over chunks of latents of one voice; chunk k equals the same chunk decoded alone, bit for
// bit.  Without `resample` or i16, a chunk leaves as the decoder's waveform, and its trims, gain and the fade must keep
// their defaults.  Otherwise the reference's post-path runs on the device per chunk: drop the trim frames,
// crossfade(fade) (samples.rs:144-157), the gain.  With `resample` the chunk is then appended to its stream's resampler,
// emitting every output it can (a chunk without one leaves at the voice's rate as the post-path leaves it); a resampler
// may appear once per pass and must belong to the voice.  A chunk with a prosody stream (resample passes only) is warped
// first, and what that stream emits is what the resampler, or the voice-rate copy, takes; the same rules hold for
// prosody streams.  A chunk with a loudness meter (resample passes only) is metered after all that, in place, and its
// gain applies after the meter, in every format; its i16 / G.711 conversion is at the fixed scale.  i16: to_i16_vec (samples.rs:51-75) normalised to each emitted
// chunk's own peak; mu-law / A-law: the G.711 bytes of those same i16 samples, from the same launches.  Every check runs
// before any device work and any resampler changes; errors name the chunk, except with `single`, which keeps the
// single-chunk entry point's messages.  With `debug` the decoder keeps one buffer per stage and every stage is copied
// out per chunk after the pass (ChunkResult::captures); the launches are the same.  Such a pass is format 0 without
// `resample`.
struct ChunkPass {
    std::vector<ChunkSpec> chunks;
    int fade = 0;
    bool resample = false;
    int format = 0;                       // PcmFormat: 0 f32, 1 i16, 2 mu-law, 3 A-law
    bool single = false;
    bool debug = false;
};
// One stage of a debug chunk pass: "z" (the gathered latent rows), then the DecoderBufs::expose_to names; rows[k] is
// chunk k's (hi - lo) * level rows of `cols` values, time-major.
struct ChunkCapture {
    std::string name;
    int cols = 0, level = 1;
    std::vector<std::vector<float>> rows;
};
struct ChunkResult {
    std::vector<std::vector<float>> f32;      // format 0
    std::vector<std::vector<int16_t>> i16;    // format 1
    std::vector<std::vector<uint8_t>> g711;   // formats 2 and 3
    float ms = 0;                             // the pass's device time
    float stretch_ms = 0, pitch_ms = 0;       // its "stretch" and "pitch" regions (0: none ran)
    float formant_ms = 0;                     // its "formant" region (0: none ran)
    float loudness_ms = 0;                    // its "loudness" region (0: none ran)
    std::vector<ChunkCapture> captures;       // ChunkPass::debug only
};
void decode_chunks(Voice* v, const ChunkPass& p, ChunkResult& out);

// ---- the waveform output stage (output_stage.cu) ----
// After the decoder: prosody (stretch, pitch), formants, volume, breaks, resampling, then loudness in place on what that
// leaves.

// What a stage reads: segment k is buf[segs[k].out_off ..), segs[k].len * hop samples read through posts[k] (trims,
// fade, gain; null: read plainly).  The whole-signal prosody and formant launches read buf at their plans' offsets.
struct Wave {
    float* buf = nullptr;
    const FrameSeg* segs = nullptr;
    const PcmPost* posts = nullptr;
    int hop = 1;
};

// One resample launch over segments laid out back to back: each segment's ResampleSeg, what the launch is sized by and
// what the profile counts.
struct ResamplePlan {
    std::vector<ResampleSeg> segs;
    long long total = 0, max_out = 0; int smem = 0;
    double flops = 0, bytes = 0;
    // Appends a segment of n_in inputs through `f` (null: copied unchanged).  A whole signal emits every output; with a
    // stream's resampler `r` (whose filter is f) the segment continues r's stream, emits every output whose inputs have
    // all arrived, and flushes the stream when `last`.
    void add(const ResampleFilter* f, long long n_in, const Resampler* r = nullptr, bool last = false);
};

// The watermark launch.  Segment q emits n samples of its input at y[y_off ..): the h samples at hold, then the m at
// x[x_off ..), the mark at positions pos0 + i in blocks of blk = R / 100 samples (chips null: copied unchanged).  The
// block before the first is block 0, or with s_in the block whose S is *s_in.  A job's segments are whole utterances,
// read and written at the same offset (h = 0, m = n, pos0 = 0).  A stream's also put the inputs past n into hold_out
// and the S of the last block they emit into s_out (WatermarkStream).
struct WatermarkSeg {
    long long x_off, y_off, n, m, pos0;
    int h, blk, payload;
    double alpha;
    const signed char* chips;
    const float* hold; float* hold_out;
    const long long* s_in; long long* s_out;
};
struct WatermarkStream;
struct WatermarkPlan {
    std::vector<WatermarkSeg> segs;
    long long total = 0, max_runs = 0, max_n = 0;
    double bytes = 0;
    // A job's utterance of n samples at offset off, delivered at `rate`.
    void add(const Watermark& wm, long long off, long long n, int rate);
    // A chunk of m new samples at x_off: with its stream ws, what the stream emits for it (the hold-back rule of
    // include/sonata_b200.h, sb200_watermark_stream_create), else the chunk copied; written at total ..
    void add_chunk(const WatermarkStream* ws, long long x_off, long long m, bool last);
};
void launch_watermark(const WatermarkPlan& p, const WatermarkSeg* segs, const float* x, float* y, cudaStream_t st);
// Detection (include/sonata_b200.h, sb200_watermark_detect) of `batch` clips of fmt 0 (f32) or 1 (i16) samples at
// d_x[offs[b] .. offs[b + 1]) on the device, into out[0 .. batch); the device work runs on st.  F (null: not wanted)
// receives every clip's fold, WM_P int64 each.
struct WatermarkScore { int marked, payload, offset; double z0, z1; };
void watermark_detect(unsigned long long key, int fmt, const void* d_x, const size_t* offs, size_t batch,
                      WatermarkScore* out, cudaStream_t st, long long* F = nullptr);

// The loudness launch over what a job hands out: one segment per utterance at its delivered rate, chunk scratch laid out
// back to back.
struct LoudnessPlan {
    std::vector<LoudSeg> segs;
    long long chunks = 0;
};

// The metered chunks of a chunk pass: chunks[q] has n[q] samples, its window at win_off[q] of the pass's window buffer
// and the steps[q] steps it completes at step_off[q] of its step tables.
struct MeterPlan {
    std::vector<int> chunks;
    std::vector<long long> n, win_off, step_off, steps;
    long long win_total = 0, steps_total = 0;
    void add(int k, const LoudnessStream& s, long long samples, long long completes);
};

// The output stage of one pass.  A job's (plan_job_output) runs each stage on whole utterances; a chunk pass's
// (plan_chunk_output) runs each chunk's streams, one window each, and keeps the chunks and their steps so the streams
// can advance after the pass.  An empty plan of either kind runs nothing.
struct OutputPlan {
    ProsodyPlan pp;
    FormantPlan fp;
    VolumePlan vp;
    BreakPlan bp;
    ResamplePlan rp;
    WatermarkPlan wp;                         // jobs of a marked voice
    LoudnessPlan lp;                          // whole signals
    MeterPlan mp;                             // chunk passes
    std::vector<ChunkSpec> chunks;            // chunk passes: empty for a job
    std::vector<ProsodyStep> steps;           // per chunk with a prosody stream
    std::vector<FormantStep> fsteps;          // per chunk whose stream runs the formant stage
    std::vector<int> warped, formed, warp_of; // the chunks of pp's and fp's segments; warp_of[k]: chunk k's segment of pp
    std::vector<long long> n_res;             // per chunk: the samples the resample launch takes
    std::vector<float> out_gain;              // per chunk (or empty): the gain of its resampled output's PcmPost
    std::vector<int> fixed_scale;             // per chunk (or empty): that PcmPost's fixed_scale
    bool streams() const { return !chunks.empty(); }
};
// The output stage of job j's utterances on the frame layout j.frames with `hop` samples per frame, and what the job
// hands out (osegs, out_hop, out_total, osr).  With a contour (cum: the batch's cum rows on the host) every utterance is
// planned from its ids' ends, and bounds receives each id's delivered end, packed like the ids.  A volume contour's
// pieces and the breaks' tables are planned over the same ends (cum is then on the host too); with breaks, bounds
// receives every utterance's ends after its pauses.
OutputPlan plan_job_output(Job& j, int hop, const std::vector<int>& cum, std::vector<long long>& bounds);
// The output stage of chunk pass chunks, chunk k bringing n_in[k] samples after its trims: each chunk's prosody stream,
// its formant, volume and break stages, with `resample` the resample launch (a chunk without a resampler is copied), and its meter, which
// reads what the resample launch delivers (without it: the chunk's stage output).
OutputPlan plan_chunk_output(const std::vector<ChunkSpec>& chunks, const std::vector<long long>& n_in, bool resample);

// The device buffers and tables of plan p and their pinned mirrors.  `in` is where the stage's input goes (the decoder's
// waveforms, in_total samples): a buffer of the pass's own, followed by the prosody output `py`, the formant output
// `fy`, a chunk pass's volume output `vy` and the break output `by`, or the caller's d_out when no stage writes a result of its own.  With d_out the last stage that writes writes
// there; the resample output `ry` is otherwise the pass's own.  offsets, ps (the stretched signal) and py stay
// reachable after the pass.
struct OutputBufs {
    Staged<ProsodySeg> psegs; Staged<FrameSeg> posegs; Staged<ProsodyCarry> pcarry;
    Staged<ContourPiece> pieces;              // the contours' piece tables (only when a segment has one)
    long long* apos = nullptr;                // and their analysis positions, indexed like the offsets
    int* offsets = nullptr; float *px = nullptr, *ps = nullptr, *py = nullptr;
    Staged<FormantSeg> fsegs; Staged<FormantCarry> fcarry; float *fwin = nullptr, *fy = nullptr;
    Staged<VolumeSeg> vsegs; Staged<VolumePiece> vpieces; float* vy = nullptr;
    Staged<BreakSeg> bsegs; Staged<BreakPiece> bpieces; Staged<FrameSeg> bosegs; float* by = nullptr;
    Staged<FrameSeg> rin; Staged<PcmPost> rpost;  // chunk passes: what the resample launch reads after the stages
    Staged<ResampleSeg> rsegs; Staged<PcmPost> rposts; Staged<FrameSeg> rosegs; float* ry = nullptr;
    Staged<WatermarkSeg> wsegs; Staged<FrameSeg> wosegs; Staged<PcmPost> wposts; float* wy = nullptr;
    Staged<LoudSeg> lsegs; double* lscratch = nullptr; Staged<double> lufs; Staged<float> gain;
    Staged<LoudStreamSeg> msegs; float* mwin = nullptr; double* me = nullptr;
    Staged<double> mlufs; Staged<float> mgains; Staged<unsigned long long> mclip;
    float* in = nullptr;
    void carve(Arena& dev, Arena& pin, const OutputPlan& p, long long in_total, float* d_out);
    // Fills and uploads every table.  A chunk pass's input is read at `hop` samples per frame through the host mirrors
    // of its segment and post tables (in_segs, in_posts; null posts: read plainly); a job's needs neither.
    void upload(const OutputPlan& p, int hop, const FrameSeg* in_segs, const PcmPost* in_posts, cudaStream_t st);
};

// The launches of plan p from the input wave `in` (in.buf == b.in) on st: profile regions "stretch", "pitch",
// "formant", "volume", "break", "resample", "watermark" (a job of a marked voice: into wy, at the same offsets) and
// "loudness", each only when its stage runs.  A job's volume stage scales
// its utterances in place; a chunk pass's writes each chunk to vy (after fy).  The break stage writes every segment to
// by, longer by its pauses.  Returns what the stage delivers: the last
// output's wave (a job's: its segments at hop 1 once a stage has changed their lengths).  The loudness results are
// downloaded to their pinned mirrors.
Wave run_output_stage(Profile& prof, const OutputPlan& p, const OutputBufs& b, Wave in, cudaStream_t st);
// After a chunk pass's plan p has run and synchronised: its resamplers, prosody and formant stages and meters take their
// new counts, and each stream the region times of the pass in prof.
void advance_streams(const OutputPlan& p, const OutputBufs& b, const Profile& prof);

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
