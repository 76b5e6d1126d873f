// Shared declarations for libsonata_b200 (sm_90a only).
//
// Activation layout everywhere: TIME-MAJOR fp32 matrices  A[row][channel]  (channel contiguous).
// A "row" is one time step (phoneme id at the X level, frame at the Y level, sample-group at the
// decoder levels).  Utterances of a batch are concatenated along rows as SEGMENTS; segment b
// occupies rows [off_b, off_b + T_b) and is followed by >= HALO all-zero gap rows, so a
// convolution that reads across a segment edge sees the zero padding the reference's B=1
// onnxruntime run would see (piper/src/lib.rs:433-435 runs every utterance alone).
// Every kernel that produces an activation writes ZERO into gap rows (or leaves accumulated
// buffers untouched there), which keeps that invariant without memsets.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <mutex>

#define SB_MAX_TAPS 16

namespace sb200 {

// Row validity: row q is a real time step iff  q < seg_end[q / gran] * seg_mul.
// seg_end is indexed by "granule" (64 ids at the X level, 128 frames at the Y level; a granule
// never straddles two segments) and holds off_b + T_b in granule-level rows; decoder levels
// that run at U x the frame rate pass gran = 128*U, seg_mul = U.
struct RowMap {
    const int* seg_end;
    int gran;
    int seg_mul;
    int rows;   // total rows at this level
};

__device__ __forceinline__ bool row_valid(const RowMap& m, int q) {
    if (q < 0 || q >= m.rows) return false;
    return q < m.seg_end[q / m.gran] * m.seg_mul;
}

enum ConvAct { ACT_NONE = 0, ACT_RELU = 1, ACT_GATE = 2 };

// One implicit-GEMM convolution:  for GEMM row q, output column n
//   acc = bias[n] + sum_t sum_c  f(x[q + tap_off[t]][c]) * w[t][c][n],   f = leaky_relu(in_slope)
//   v   = act(acc) (+ res[orow][n]) ; v *= scale ; y[orow][n] (=|+=) v,   orow = q*orow_mul + orow_add
struct ConvArgs {
    const float* x; int ldx; int rows_in; int cin; float in_slope;
    const float* w; const float* bias; int ldw; int cout;
    const float* wtc; int tc_nt;                                  // bf16 hi/lo weight images (conv_tc.cu) or null
    const float* wtf;                                             // tf32 hi/lo images (conv_tf.cu) or null
    int ntaps; int tap_off[SB_MAX_TAPS]; int min_off; int span;   // span = max_off - min_off
    int rows_q; int orow_mul; int orow_add;
    RowMap map;                                                   // validity of q
    int act; float scale;
    const float* res; int ldres;
    float* y0; int ldy0; int acc0; int split;                     // columns [0, split)
    float* y1; int ldy1; int acc1;                                // columns [split, cout)
    float* yt; int yt_col0; int ldyt;                             // conv_tf.cu: column tiles >= yt_col0 are stored TRANSPOSED,
                                                                  // yt[(n - yt_col0) * ldyt + q] (row index contiguous)
    const int* bias_slot; int ldbias;                             // per-row bias: row q adds bias[bias_slot[q / map.gran] * ldbias + n]
                                                                  // (speaker-conditioned convs of a batch with several speakers)
};

// Epilogue view of GEMM row q >= 0: its validity (row_valid) and its bias row (the conv's own, or with a slot table the
// one of q's slot), sharing one granule division.
__device__ __forceinline__ const float* conv_row(const ConvArgs& a, int q, bool& valid) {
    const int g = q / a.map.gran;
    valid = q < a.map.rows && q < a.map.seg_end[g] * a.map.seg_mul;
    return a.bias_slot ? a.bias + (size_t)a.bias_slot[g] * a.ldbias : a.bias;
}

// One tile of a grouped GEMM on conv_tf.cu's kernel (the attention contractions): two 128-row m-tiles of A against
// one block of nth B rows over `nkb` 32-column K-blocks;  C = scale * A . B^T (+ res).
struct TfTile {
    int a_row0[2];        // first row of m-tile h in A (rows outside the array read as zeros)
    int a_col0;           // first K column in A
    int b_row0;           // first row of the B block
    int b_col0;           // first K column in B
    int nkb;              // 32-column K-blocks
    int kcols;            // K columns that hold data (from a_col0 / b_col0); the rest of the last K-block reads as zeros
    int rows_valid[2];    // rows of m-tile h that are stored
    long long out_off[2]; // element offset of (row 0, column 0) of m-tile h's output block in y (and res)
};
struct TfGemm {
    const float* a; int a_rows, a_cols, lda;      // A [a_rows][a_cols], K along the columns
    const float* b; int b_rows, b_cols, ldb;      // B [b_rows][b_cols], rows = output columns
    int nth;                                      // B rows (= output columns) per tile: 96 / 64 / 48 / 32
    float* y; int ldy; const float* res; float scale;
    const TfTile* tiles; int ntiles;              // device table
};

// Function attributes (opt-in shared-memory size) are per DEVICE: `run` executes `f` the first time the calling site
// runs on the current device (a process driving several GPUs through the C ABI configures each of them).  The device
// bit is published only AFTER `f` returned, under a mutex, so a second host thread on the same device can never
// launch with more than 48 KB of dynamic shared memory before the opt-in has been applied.
struct PerDeviceOnce {
    std::mutex mu;
    unsigned long long done = 0;
    template <typename F> void run(F&& f) {
        int dev = 0;
        cudaGetDevice(&dev);
        const unsigned long long bit = 1ull << (dev & 63);
        if (__atomic_load_n(&done, __ATOMIC_ACQUIRE) & bit) return;
        std::lock_guard<std::mutex> g(mu);
        if (done & bit) return;
        f();
        __atomic_fetch_or(&done, bit, __ATOMIC_RELEASE);
    }
};

// Programmatic dependent launch.  The step is a chain of ~170-200 dependent kernels; at single-utterance sizes most of
// them run for 5-30 us, so the launch gap and each kernel's prologue (mbarrier init, weight fetch)
// are a visible part of the step.  Every kernel of the library is launched with the programmatic-stream-serialization
// attribute and starts with pdl_wait() BEFORE its first access to global memory (wgmma kernels: after their weight fetch is issued),
// after a pdl_trigger() at its very top: the following kernels' CTAs may become resident and run their own prologues (and
// fetch their weights, which no kernel writes) while this kernel is still working; their pdl_wait() returns only when the
// preceding grid has completed and its writes are visible.  Nothing before a pdl_wait() touches memory another kernel
// writes, and a kernel whose CTAs are all resident can always finish, so running ahead cannot deadlock.
// SB200_NO_PDL=1 launches without the attribute (the two instructions are then no-ops).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    static const int allowed = getenv("SB200_NO_PDL") ? 0 : 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = allowed;
    cfg.attrs = at; cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

// Experiment knobs of the launch planners come from the environment.  getenv() scans the whole environment block
// (~1 us), and a planner runs twice per launch with up to seven knobs: 170 launches of a single-utterance call spent
// more host time there than the GPU needed for the kernels.  Each knob is read ONCE per process.
#define SB_ENV_ONCE(name) ([]() -> const char* { static const char* v = getenv(name); return v; }())

void launch_conv_simt(const ConvArgs& a, cudaStream_t st);
int conv_simt_bn_for(int cout);
// planning only, see sb200_debug_plan; *staging_bytes: the staged epilogue operands' shared memory (0: not staged)
bool conv_tc_plan_info(const ConvArgs& a, int* out16, int* staging_bytes = nullptr);
// try_launch_conv_tc / _tf plan once and launch; false (nothing launched) when the kernel does not take the shape
bool try_launch_conv_tc(const ConvArgs& a, cudaStream_t st);
extern int g_conv_tc_grid_cap;     // at most this many CTAs per conv_tc launch (0: no cap); see sb200_debug_conv_grid_cap
size_t conv_tc_weight_floats(int cin, int cout, int ntaps, int nt);
void conv_tc_build_weights(const float* wt, int ldw, int cin, int cout, int ntaps, int nt, float* out);
bool conv_tf_plan_info(const ConvArgs& a, int* out16);
bool try_launch_conv_tf(const ConvArgs& a, cudaStream_t st);
size_t conv_tf_weight_floats(int cin, int cout, int ntaps);
void conv_tf_build_weights(const float* wt, int ldw, int cin, int cout, int ntaps, float* out);
bool gemm_tf_supported(const TfGemm& g);
void launch_gemm_tf(const TfGemm& g, cudaStream_t st);
void throw_launch_error(const char* what);

struct SegInfo { int off; int len; };   // rows

// ---- misc kernels (kernels_misc.cu) ----
void launch_embed(const int* ids_rows, const float* emb, float scale, float* x, int rows, int H, cudaStream_t st);
// out = (res2 ? res2 : 0) + act( LN(x + (res1 ? res1 : 0)) * gamma + beta ),  act: 0 none, 1 exact GELU
void launch_ln(const float* x, const float* res1, const float* res2, const float* gamma, const float* beta,
               float* out, int C, int act, RowMap map, cudaStream_t st);
// out = GELU(LN(depthwise_conv_k(x, dilation)))   (DDSConv first half)
void launch_dw_ln_gelu(const float* x, const float* wdw /*[k][C]*/, const float* bdw, int k, int dil,
                       const float* gamma, const float* beta, float* out, int C, RowMap map, cudaStream_t st);
// Relative-position softmax between the two attention GEMMs (in place on the score rows): see kernels_misc.cu
void launch_attn_softmax(float* S, int Tp, const float* qkv, int ldq, const float* relk, const float* relv, int window,
                         float* orel, int ldo, int H, int heads, int RX, const SegInfo* segs, const int* seg_of_gran,
                         int gran, int max_len, cudaStream_t st);
void launch_attention(const float* qkv, int ldq, const float* relk, const float* relv, int window,
                      float* out, int ldo, int H, int heads, const SegInfo* segs, int nseg, int max_len,
                      cudaStream_t st);
size_t attention_smem_bytes(int max_len, int D);
// h[r][c] = w[c]*z[r][zcol] + b[c] + g[r][c]
void launch_flow_pre(const float* z, int zcol, const float* w, const float* b, const float* g, float* h,
                     int C, RowMap map, cudaStream_t st);
// z[r][tcol] = RQS^-1(z[r][tcol]; params h29[r][0..3*bins-1))
void launch_spline(const float* h29, int ldh, float* z, int tcol, int bins, float inv_sqrt_filter,
                   RowMap map, cudaStream_t st);
// logw = (z[:,0]-m0)*exp(-logs0); w = exp(logw)*length_scale[b]; w_ceil; per-segment inclusive scan.  Optional per-id
// controls at the id level (null: none): w_ceil = ceil(w * dur_scale[r]), and dur_frames[r] >= 0 replaces w_ceil.
void launch_durations(const float* z, float m0, float logs0, const float* length_scale, const SegInfo* segs, int nseg,
                      float* logw, int* cum, int* y_len, cudaStream_t st, const float* dur_scale = nullptr,
                      const int* dur_frames = nullptr);
struct FrameSeg { int off; int len; int xoff; int xlen; long long out_off; };
// z_p rows: gather m_p/logs_p of the token whose cumulative duration covers the frame, add noise scaled by the noise_scale
// of the frame's segment (ftile_seg)
void launch_expand(const float* stats, int ldst, int I, const int* cum, const float* eps, const float* noise_scale,
                   float* zp, const FrameSeg* fsegs, const int* ftile_seg, RowMap ymap, cudaStream_t st);
// wav = tanh(conv_k7(lrelu_{0.01}(x)))  ->  compact per-segment output
void launch_conv_post(const float* x, int C, const float* w /*[7][C]*/, float* wav, const FrameSeg* fsegs,
                      const int* ftile_seg, int U, RowMap map, cudaStream_t st);
// per-utterance peak-normalised f32 -> i16 (audio-ops `to_i16_vec`), out indexed like wav
// what the reference applies to a chunk before the 16-bit conversion (see kernels_misc.cu): overlap trim (samples),
// crossfade table of fade_n <= 48 entries, linear gain.  Default = plain to_i16_vec.  fixed_scale = 1 converts at the
// fixed scale 32767 instead of the segment's peak (loudness-normalised utterances).
struct PcmPost { float gain = 1.f; int fade_n = 0; long long trim_lo = 0, trim_hi = 0; float tab[48] = {0}; int fixed_scale = 0; };
// One segment's PcmPost with its scalars in registers, and sample i of the segment after it (kernels_misc.cu).
struct PcmSeg {
    const float* x; long long n; float gain; int fade_n; const float* tab;
};
__device__ __forceinline__ PcmSeg pcm_seg(const float* wav, const FrameSeg& fs, const PcmPost* p, int hop) {
    const long long trim_lo = p->trim_lo;
    return {wav + fs.out_off + trim_lo, (long long)fs.len * hop - trim_lo - p->trim_hi, p->gain, p->fade_n, p->tab};
}
__device__ __forceinline__ float pcm_value(const PcmSeg& s, long long i) {
    float v = s.x[i];
    if (s.fade_n > 0) {
        if (i < s.fade_n) v = __fmul_rn(v, s.tab[i]);
        else if (i >= s.n - s.fade_n) v = __fmul_rn(v, s.tab[s.n - 1 - i]);
    }
    return s.gain == 1.f ? v : __fmul_rn(v, s.gain);
}
// Output formats of a result: 0 f32, 1 i16 PCM, 2 G.711 mu-law, 3 G.711 A-law (one byte per sample).
enum PcmFormat { PCM_F32 = 0, PCM_I16 = 1, PCM_MULAW = 2, PCM_ALAW = 3 };
inline size_t pcm_bytes(int fmt) { return fmt == PCM_F32 ? 4 : fmt == PCM_I16 ? 2 : 1; }
// G.711 of one 16-bit sample, as CPython's audioop.lin2ulaw / lin2alaw (the Sun g711.c lineage) compute it.
// mu-law: the sample >> 2 (14 bits), clipped to +-8159, biased by 33, segment from its leading bit, one's complement.
__host__ __device__ inline uint8_t g711_ulaw(int16_t x) {
    int v = x >> 2;                             // arithmetic shift
    int mask = 0xFF;
    if (v < 0) { v = -v; mask = 0x7F; }
    if (v > 8159) v = 8159;
    v += 33;                                    // 33 <= v <= 8192
    int seg = 0;
    while (seg < 8 && v >= (0x40 << seg)) seg++; // segment ends 0x3F, 0x7F, .., 0x1FFF
    if (seg >= 8) return (uint8_t)(0x7F ^ mask);
    return (uint8_t)((((seg << 4) | ((v >> (seg + 1)) & 0xF))) ^ mask);
}
// A-law: the sample >> 3 (13 bits), segment and mantissa, even bits inverted (XOR 0x55; 0xD5 also sets the sign bit).
__host__ __device__ inline uint8_t g711_alaw(int16_t x) {
    int v = x >> 3;
    int mask = 0xD5;
    if (v < 0) { v = -v - 1; mask = 0x55; }    // 0 <= v <= 4095
    int seg = 0;
    while (seg < 8 && v >= (0x20 << seg)) seg++; // segment ends 0x1F, 0x3F, .., 0xFFF
    if (seg >= 8) return (uint8_t)(0x7F ^ mask);
    const int aval = (seg << 4) | ((seg < 2 ? v >> 1 : v >> seg) & 0xF);
    return (uint8_t)(aval ^ mask);
}
// posts: device array, one entry per segment; max_samples: the longest segment (before trimming), sizes the grid.
// fmt: PCM_I16 writes short, PCM_MULAW / PCM_ALAW write the G.711 byte of that same short (out is uint8_t).
void launch_pcm(const float* wav, const FrameSeg* fsegs, const PcmPost* posts, int nseg, int hop, long long max_samples,
                unsigned* maxbits, int fmt, void* out, cudaStream_t st);
// out[i] = the G.711 byte (fmt PCM_MULAW / PCM_ALAW) of x[i], i < n: the encoders on the device over a plain buffer.
void launch_g711(const short* x, long long n, int fmt, uint8_t* out, cudaStream_t st);
// Polyphase resampling of one segment (resample_poly's sum, kernels_misc.cu resample_kernel): n_out outputs at
// out[out_off ..), from the segment's samples as pcm_value reads them.  taps: phase-major [up][K], taps[p][k] =
// h[p + k*up] (0 past 2H).  up == 0: the segment is copied unchanged.  A stream's chunk continues its stream: the
// segment's samples are inputs c .. c + n, hist holds the h inputs before them, the outputs written are j0 .. j0 + n_out,
// and hist_out (null: none) receives the last h_out inputs for the next chunk.  A whole utterance is c = h = j0 = 0.
struct ResampleSeg {
    const float* taps; long long out_off, n_out; int up, down, H, K;
    const float* hist; float* hist_out; long long c, j0; int h, h_out;
};
constexpr int RS_OUTS = 1024;     // consecutive outputs per block iteration
// Shared-memory floats a block needs for one run of RS_OUTS outputs of a segment with this ratio.
inline int resample_span(int up, int down, int K) {
    return up > 0 ? (int)(((long long)(RS_OUTS - 1) * down) / up) + K + 1 : 0;
}
// One launch over nseg segments (blockIdx.y = segment), each segment with its own ratio; max_out: the most outputs of
// any segment, smem_floats: the largest resample_span of the segments.
void launch_resample(const float* wav, const FrameSeg* fsegs, const PcmPost* posts, int hop, const ResampleSeg* segs,
                     int nseg, long long max_out, int smem_floats, float* out, cudaStream_t st);
// Integrated loudness (BS.1770-4, one channel) of one segment, wav[off, off + n) at one rate, and its normalisation in
// place (kernels_misc.cu loudness_kernel; the filter design is loudness.cu's).  The segment is cut into chunks of S
// samples, chunk c at scratch[LD_SCRATCH * (c0 + c) ..).  k: the K-weighting cascade, shelf then high-pass, each
// {b0, b1, b2, a1, a2} (a0 = 1); AS: A^S, row-major, of its state recurrence s' = A s + B x with s = the two biquads'
// transposed-direct-form-II states {s1, s2, t1, t2}.  target: LUFS, NaN = measured only.
struct LoudSeg {
    long long off, n, c0;
    int S; float target;
    double k[10], AS[16];
};
constexpr int LD_SCRATCH = 6;     // doubles per chunk: its 4 states, its sum of y^2, its peak
// One launch over nseg segments (blockIdx.x = segment): lufs[b] = the integrated loudness (-inf when no block passes the
// gates), gain[b] = the gain applied to the segment (1 without a target).
void launch_loudness(float* wav, const LoudSeg* segs, int nseg, double* scratch, double* lufs, float* gain, cudaStream_t st);
// Pitch and tempo of one segment (prosody.cu): x = wav[in_off, in_off + n) is time-stretched by alpha = pitch / tempo
// (WSOLA: synthesis hop Hs, frame 2 Hs, search radius D, F frames whose offsets go to offsets[d_off ..)) into n1 samples
// when `stretch`, then resampled by p into n2 samples when `pitch`.  The delivered signal is y[y_off, y_off + n2); with
// both stages the stretched signal passes through s[s_off, s_off + n1).  With neither, x is copied to y.
// A segment is a window of its signal, at absolute positions: wav[in_off] is input x0 (inputs at n and past it read as
// zeros), offsets[d_off] is frame d0's delta, s[s_off] is stretched sample s0 (n1: the stretched samples known; the
// pitch stage reads none past it).  The launches compute the offsets of frames [k0, k1), stretched samples [m0, m1)
// and outputs [j0, j1), written from y[y_off] (the stretched samples too when there is no pitch stage, j0 = m0).  A
// whole utterance is x0 = s0 = d0 = m0 = j0 = k0 = 0, k1 = F, m1 = n1, j1 = n2; a stream's chunk pass is a later window
// of its stream (ProsodyStream), the frames before k0 known from earlier passes and staged at offsets[d_off].
struct ProsodySeg {
    long long in_off, n, s_off, n1, y_off, n2, d_off;
    int F, Hs, D, stretch, pitch;
    double alpha, p;
    long long x0, s0, m0, m1, j0, j1;
    int k0, k1, d0;
};
// What a stream's chunk pass stages before the prosody launches and carries after them (prosody.cu): the chunk's
// samples after the post-path (fsegs / posts entry `chunk`) follow h_in history inputs in the segment's input window,
// h_s stretched samples of history start its stretched window and the deltas of frames d0, d0 + 1 start its offsets.
// Afterwards in_keep inputs from window position in_from, s_keep stretched samples from s_from and the two deltas from
// d_from go to the stream's other buffers.
struct ProsodyCarry {
    int chunk, h_in, h_s, in_keep, s_keep;
    long long in_from, s_from, d_from;
    const float *in_hist, *s_hist; const int* d_hist;
    float *in_next, *s_next; int* d_next;
};
// Analysis position of WSOLA frame k: floor(k Hs / alpha + 0.5), every operation exactly rounded in double, so the host
// plan and the kernels agree; the virtual frame -1 sits at -Hs.
__host__ __device__ inline long long prosody_analysis(int Hs, double alpha, long long k) {
    return k < 0 ? -(long long)Hs : (long long)floor((double)(k * Hs) / alpha + 0.5);
}
constexpr int PP_OUTS = 256;      // consecutive outputs of the pitch resampler per block iteration
constexpr int PP_SPAN = 640;      // shared-memory floats of their input span: 255 p + 2 W + 3 at p = 2, W = 32
// The offset chain (blockIdx.x = segment, one persistent block each; smem_ints: the largest 4 Hs + 2 D of the segments),
// the overlap-add or copy (max_out: the most samples any segment writes) and the pitch resampler, one launch each.
void launch_prosody_offsets(const float* wav, const ProsodySeg* segs, int nseg, int smem_ints, int* offsets,
                            cudaStream_t st);
void launch_prosody_ola(const float* wav, const ProsodySeg* segs, int nseg, long long max_out, const int* offsets,
                        float* s, float* y, cudaStream_t st);
void launch_prosody_pitch(const float* wav, const float* s, const ProsodySeg* segs, int nseg, long long max_out, float* y,
                          cudaStream_t st);
// A stream pass's staging (before the launches above; chunks read from src through fsegs / posts, max_in: the longest
// window) and carry (after the overlap-add; max_keep: the longest tail), one launch each over the nseg segments.
void launch_prosody_stage(const float* src, const FrameSeg* fsegs, const PcmPost* posts, int hop, const ProsodySeg* segs,
                          const ProsodyCarry* cs, int nseg, long long max_in, float* wav, float* s, int* offsets,
                          cudaStream_t st);
void launch_prosody_carry(const float* wav, const float* s, const int* offsets, const ProsodySeg* segs,
                          const ProsodyCarry* cs, int nseg, long long max_keep, cudaStream_t st);
// One row range of a frame level taken from a latent: rows [off, off + len) of the level are rows [lo, lo + len) of src.
struct GatherSeg { const float* src; long long lo; int off; int len; };
// s[r] = the source row of r's segment (tile_seg: segment of every gran-row tile), or exact zeros past its end.
// cols is a multiple of 4 and every src is 16-byte aligned.
void launch_gather_rows(const GatherSeg* segs, const int* tile_seg, int gran, int rows, int cols, float* s, cudaStream_t st);
void launch_randn(float* out, long long n, unsigned long long seed, unsigned long long stream_id, cudaStream_t st);
// One utterance's noise seed (seeded = 0: positional noise).
struct NoiseSeed { unsigned long long seed; int seeded; int pad; };
// launch_randn's buffer of map.rows x cols values, except that the valid rows of seeded segments (segment of a row:
// seg_of_gran, its first row: segs[].off) get the keyed draws of their segment's seed and tensor `tag` (0: eps_w,
// 1: eps_z), a function of the row within the utterance and the column only (kernels_misc.cu).
void launch_randn_seeded(float* out, int cols, unsigned tag, unsigned long long seed, unsigned long long stream_id,
                         const NoiseSeed* seeds, const SegInfo* segs, const int* seg_of_gran, RowMap map, cudaStream_t st);
void launch_randn_seeded(float* out, int cols, unsigned tag, unsigned long long seed, unsigned long long stream_id,
                         const NoiseSeed* seeds, const FrameSeg* segs, const int* seg_of_gran, RowMap map, cudaStream_t st);
// z[r][0..1] = eps * s[seg_of_gran[r / map.gran]]
void launch_scale_copy2(const float* eps, const float* s, const int* seg_of_gran, float* z, RowMap map, cudaStream_t st);
// out[s][r] = base[r] + sum_k w[r][k] * emb_g[sid[s]][k]  for every slot s < nslots   (speaker conditioning: effective
// biases of the conditioned convs, one set per distinct speaker of a batch)
void launch_cond_bias(const float* w, const float* base, const float* emb_g, const int* sid, int nslots, int rows, int gin,
                      float* out, cudaStream_t st);

// launch-configuration errors are not sticky and would otherwise be lost: throw immediately
void check_launch(const char* what);

extern unsigned long long g_launch_count;   // kernels launched by this library (host-side counter)

}  // namespace sb200
