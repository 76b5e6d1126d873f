// The batched phoneme-id -> waveform pass: packs B utterances into row segments, launches the
// kernel sequence of the Piper graph (SURVEY Appendix A; oracle/vits_oracle.py is the op-by-op
// restatement) and returns per-utterance waveforms.  Replaces VitsModel::infer_with_values +
// the `session.run` it wraps (piper/src/lib.rs:342-399); `speak_batch`'s sequential B=1 loop
// (:433-435) becomes ONE pass whose per-utterance results equal the B=1 results.
#include "engine.h"
#include <algorithm>
#include <array>
#include <cmath>
#include <cstring>
#include <cstdlib>

namespace sb200 {

void throw_launch_error(const char* what) { throw Error(19, std::string("internal: ") + what); }

void check_launch(const char* what) {
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw Error(19, std::string("CUDA launch failed (") + what + "): " + cudaGetErrorString(e));
}

ConvArgs conv_args(const ConvW& w, const float* x, int ldx, const RowMap& map, const ConvCall& c) {
    ConvArgs p{};
    p.x = x; p.ldx = ldx; p.rows_in = map.rows; p.cin = w.cin; p.in_slope = c.in_slope;
    p.w = w.w; p.bias = w.bias; p.ldw = w.ldw; p.cout = w.cout; p.wtc = w.wtc; p.tc_nt = w.tc_nt; p.wtf = w.wtf;
    p.ntaps = w.ntaps; memcpy(p.tap_off, w.tap_off, sizeof(p.tap_off)); p.min_off = w.min_off; p.span = w.span;
    p.rows_q = map.rows; p.orow_mul = c.orow_mul; p.orow_add = c.orow_add;
    p.map = map;
    p.act = c.act; p.scale = c.scale; p.res = c.res; p.ldres = c.ldres;
    p.y0 = c.y0; p.ldy0 = c.ldy0; p.acc0 = c.acc0; p.split = c.split < 0 ? w.cout : c.split;
    p.y1 = c.y1; p.ldy1 = c.ldy1; p.acc1 = c.acc1;
    p.yt = c.yt; p.yt_col0 = c.yt_col0; p.ldyt = c.ldyt;
    return p;
}

namespace {
constexpr int GX = 64;     // X-level granule (ids)
constexpr int HX = 16;     // min zero rows between X segments (DDSConv dilation 9 + margin)
constexpr int GY = 128;    // Y-level granule (frames)
constexpr int HY = 8;      // min zero frames between Y segments (>= decoder halo / 8)
inline int round_up(int x, int m) { return (x + m - 1) / m * m; }
}  // namespace

// ------------------------------------------------------------------ Context
// Arenas grow with headroom, so a warmed-up context allocates nothing in steady state.
void Arena::reserve(size_t bytes) {
    used = 0;
    if (bytes <= cap) return;
    release();
    const size_t want = pinned ? bytes * 2 : bytes + bytes / 8 + (64u << 20);
    void* p = nullptr;
    SB_CUDA(pinned ? cudaMallocHost(&p, want) : cudaMalloc(&p, want));
    base = (char*)p; cap = want;
}
void Arena::release() {
    if (base) pinned ? cudaFreeHost(base) : cudaFree(base);
    base = nullptr; cap = 0; used = 0;
}
cudaEvent_t Context::next_event() {
    if (events_used == events.size()) {
        cudaEvent_t e;
        SB_CUDA(cudaEventCreate(&e));
        events.push_back(e);
    }
    return events[events_used++];
}
Context::~Context() {
    dev_id.release();
    dev_frame.release();
    pin.release();
    for (auto e : events) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
}

Context* Voice::acquire() {
    {
        std::lock_guard<std::mutex> g(pool_mu);
        if (!pool.empty()) { Context* c = pool.back(); pool.pop_back(); return c; }
    }
    SB_CUDA(cudaSetDevice(device));
    std::unique_ptr<Context> c(new Context());
    c->device = device;
    SB_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    return c.release();
}
void Voice::release(Context* c) {
    std::lock_guard<std::mutex> g(pool_mu);
    pool.push_back(c);
}

// ------------------------------------------------------------------ Job
Job::~Job() {
    if (ctx && v) v->release(ctx);
}

Job* create_job(Voice* v, const long long* ids, const size_t* offs, size_t B, const float* const* eps_w,
                const float* const* eps_z, const size_t* eps_z_frames, bool debug) {
    if (B == 0) throw Error(19, "empty batch");
    if (v->device < 0 || !v->emb)
        throw Error(19, "Failed to run model inference. Error: voice was loaded config-only (device -1); libsonata_b200 has no CPU path");
    std::unique_ptr<Job> j(new Job());
    j->v = v; j->B = B; j->debug = debug;
    set_job_configs(*j, nullptr);
    j->offs.assign(offs, offs + B + 1);
    j->ids.assign(ids + offs[0], ids + offs[B]);
    const size_t base = offs[0];
    for (auto& o : j->offs) o -= base;
    for (size_t b = 0; b < B; b++) {
        const size_t n = j->offs[b + 1] - j->offs[b];
        if (n == 0) throw Error(19, "Failed to run model inference. Error: empty input sequence");
        for (size_t i = j->offs[b]; i < j->offs[b + 1]; i++)
            if (j->ids[i] < 0 || j->ids[i] >= v->a.n_vocab)
                throw Error(19, "Failed to run model inference. Error: phoneme id out of range for the embedding table");
    }
    if (eps_w) { j->eps_w.resize(B); for (size_t b = 0; b < B; b++) if (eps_w[b]) j->eps_w[b].assign(eps_w[b], eps_w[b] + 2 * (j->offs[b + 1] - j->offs[b])); }
    if (eps_z) {
        j->eps_z.resize(B); j->eps_z_frames.assign(eps_z_frames, eps_z_frames + B);
        for (size_t b = 0; b < B; b++) if (eps_z[b]) j->eps_z[b].assign(eps_z[b], eps_z[b] + eps_z_frames[b] * (size_t)v->a.inter);
    }
    // X layout
    int cur = 0;
    for (size_t b = 0; b < B; b++) {
        const int n = (int)(j->offs[b + 1] - j->offs[b]);
        j->xsegs.push_back({cur, n});
        j->max_tx = std::max(j->max_tx, n);
        cur += round_up(n + HX, GX);
    }
    j->RX = round_up(cur, 256);
    {
        // Tile tables of the two attention GEMMs (conv_tf.cu, grouped mode).  S[head][row][key] = Q.K^T / sqrt(D):
        // A = Q rows, B = K rows of the fused q/k/v activation [RX][3H]; O = P.V: A = P rows of S viewed as
        // [heads*RX][Tp], B = V^T [H][RX] (the q/k/v projection stores V transposed).
        const int H = v->a.hidden, heads = v->a.heads, D = H / heads;
        j->att_tp = round_up(std::max(j->max_tx, 1), 64);      // key tile of the Q.K^T GEMM (64: see conv_tf.cu tf_nth_for)
        // Small jobs (a single utterance): narrower column tiles put the same MMAs on more SMs (conv_tf.cu plan()); tile
        // width changes no summation order, so results do not depend on it.
        {
            int sms = 132, dev = 0;
            if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
            long long wide_s = 0, wide_o = 0;
            for (size_t b = 0; b < B; b++) {
                const int T = j->xsegs[b].len;
                wide_s += (long long)heads * ((T + 255) / 256) * ((T + 63) / 64);
                wide_o += (long long)heads * ((T + 255) / 256);
            }
            j->att_nth_s = wide_s * 2 <= sms ? 32 : 64;
            j->att_nth_o = (D % 32 == 0 && wide_o * (D / 32) <= sms) ? 32 : D;
        }
        const int ks = j->att_nth_s, ko = j->att_nth_o;
        for (size_t b = 0; b < B; b++) {
            const int off = j->xsegs[b].off, T = j->xsegs[b].len;
            const int nmp = (T + 255) / 256, nnt = (T + ks - 1) / ks;
            for (int h = 0; h < heads; h++)
                for (int mp = 0; mp < nmp; mp++) {
                    TfTile t{};
                    for (int m = 0; m < 2; m++) {
                        const int r0 = (mp * 2 + m) * 128;
                        t.rows_valid[m] = std::max(0, std::min(128, T - r0));
                    }
                    // Q.K^T: one tile per block of ks keys
                    for (int nt = 0; nt < nnt; nt++) {
                        TfTile s = t;
                        for (int m = 0; m < 2; m++) {
                            s.a_row0[m] = off + (mp * 2 + m) * 128;
                            s.out_off[m] = ((long long)h * j->RX + s.a_row0[m]) * j->att_tp + (long long)nt * ks;
                        }
                        // 48-wide heads: the second K-block is half used and zero-filled past the head
                        s.a_col0 = h * D; s.b_row0 = off + nt * ks; s.b_col0 = H + h * D; s.nkb = (D + 31) / 32; s.kcols = D;
                        j->tiles_s.push_back(s);
                    }
                    // P.V: K runs over the utterance's keys in blocks of 32 (the softmax zero-fills up to the block end)
                    for (int c0 = 0; c0 < D; c0 += ko) {               // one tile per ko head-dim columns
                        TfTile o = t;
                        for (int m = 0; m < 2; m++) {
                            o.a_row0[m] = h * j->RX + off + (mp * 2 + m) * 128;
                            o.out_off[m] = (long long)(off + (mp * 2 + m) * 128) * H + (long long)h * D + c0;
                        }
                        o.a_col0 = 0; o.b_row0 = h * D + c0; o.b_col0 = off; o.nkb = (T + 31) / 32; o.kcols = o.nkb * 32;
                        j->tiles_o.push_back(o);
                    }
                }
        }
    }
    if (attention_smem_bytes(j->max_tx, v->a.hidden / v->a.heads) > 220 * 1024)
        throw Error(19, "Failed to run model inference. Error: sentence too long for one pass (" + std::to_string(j->max_tx) + " ids)");
    j->noise_call = ++v->call_counter;
    j->ctx = v->acquire();
    return j.release();
}

void check_config(const Voice& v, const SynthConfig& c, const std::string& who) {
    if (!c.has_speaker) return;
    for (auto& kv : v.speaker_id_map)
        if (kv.second == c.speaker) return;
    throw Error(19, who + "No speaker was found with the given id `" + std::to_string(c.speaker) + "`");
}

void set_job_configs(Job& j, const SynthConfig* cfgs) {
    if (!cfgs) {
        std::shared_lock<std::shared_mutex> g(j.v->cfg_mu);   // read lock, like piper/src/lib.rs:343
        j.cfgs.assign(j.B, j.v->cfg);
        return;
    }
    for (size_t b = 0; b < j.B; b++) check_config(*j.v, cfgs[b], "utterance " + std::to_string(b) + ": ");
    j.cfgs.assign(cfgs, cfgs + j.B);
}

void set_job_durations(Job& j, const float* scale, const int* frames) {
    for (size_t b = 0; b < j.B; b++)
        for (size_t i = j.offs[b]; i < j.offs[b + 1]; i++) {
            auto fail = [&](const std::string& what) {
                throw Error(19, "utterance " + std::to_string(b) + ", id " + std::to_string(i - j.offs[b]) + ": " + what);
            };
            if (scale && !(std::isfinite(scale[i]) && scale[i] >= 0.f))
                fail("duration scale " + std::to_string(scale[i]) + " is not a finite value >= 0");
            if (frames && frames[i] < -1)
                fail("fixed duration " + std::to_string(frames[i]) + " is neither -1 (predicted) nor a frame count >= 0");
        }
    const size_t n = j.ids.size();
    if (scale) j.dur_scale.assign(scale, scale + n); else j.dur_scale.clear();
    if (frames) j.dur_frames.assign(frames, frames + n); else j.dur_frames.clear();
}

void set_job_seeds(Job& j, const unsigned long long* seeds, const int* seeded) {
    if (!seeds) { j.seeds.clear(); return; }
    std::vector<NoiseSeed> s(j.B);
    bool any = false;
    for (size_t b = 0; b < j.B; b++) {
        const int f = seeded ? seeded[b] : 1;
        if (f != 0 && f != 1) throw Error(19, "utterance " + std::to_string(b) + ": seeded flag " + std::to_string(f) + " is neither 0 nor 1");
        if (f && (!j.eps_w.empty() || !j.eps_z.empty()))     // injection zero-fills the utterances it leaves out
            throw Error(19, "utterance " + std::to_string(b) + ": a noise seed on a job with injected eps_w / eps_z");
        s[b] = NoiseSeed{f ? seeds[b] : 0ull, f, 0};
        any |= f != 0;
    }
    if (any) j.seeds.swap(s); else j.seeds.clear();
}

void set_job_output_rates(Job& j, const unsigned* rates) {
    if (!rates) { j.out_rates.clear(); return; }
    std::vector<int> r(j.B, 0);
    bool any = false;
    for (size_t b = 0; b < j.B; b++) {
        if (rates[b] == 0 || rates[b] == (unsigned)j.v->sample_rate) continue;
        resample_ratio(j.v->sample_rate, rates[b], "utterance " + std::to_string(b) + ": ");
        r[b] = (int)rates[b];
        any = true;
    }
    if (any) j.out_rates.swap(r); else j.out_rates.clear();
}

void set_job_loudness(Job& j, const float* targets) {
    if (check_loudness_targets(targets, j.B)) j.loud_target.assign(targets, targets + j.B);
    else j.loud_target.clear();
}

void set_job_prosody(Job& j, const float* pitch, const float* tempo) {
    if (!check_prosody(pitch, tempo, j.B)) { j.pitch.clear(); j.tempo.clear(); return; }
    const std::vector<float> none(j.B, NAN);
    j.pitch.assign(pitch ? pitch : none.data(), (pitch ? pitch : none.data()) + j.B);
    j.tempo.assign(tempo ? tempo : none.data(), (tempo ? tempo : none.data()) + j.B);
}

namespace {

// Launches of one pass on context c's stream, each counted in the profile region of `regions` open at the time.  cond:
// the effective biases of the speaker-conditioned convs, [slot][cond_rows] (null on a single-speaker voice).
struct Runner {
    Voice& v; Context& c; std::vector<Region>& regions; const float* cond; const Arch& a; cudaStream_t st;
    Region* cur = nullptr;
    Runner(Voice& voice, Context& ctx, std::vector<Region>& regs, const float* cond_bias)
        : v(voice), c(ctx), regions(regs), cond(cond_bias), a(voice.a), st(ctx.stream) {}

    void begin(const std::string& name) {
        regions.emplace_back();
        cur = &regions.back();
        cur->name = name;
        cur->e0 = c.next_event(); cur->e1 = c.next_event();
        cudaEventRecord(cur->e0, st);
    }
    void end() { cudaEventRecord(cur->e1, st); cur = nullptr; }
    void count(double flops, double bytes, int launches = 1) {
        if (cur) { cur->flops += flops; cur->bytes += bytes; cur->launches += launches; }
    }

    void conv(const ConvW& w, const float* x, int ldx, const Level& lin, const ConvCall& o) {
        ConvArgs p = conv_args(w, x, ldx, lin.map, o);
        // on a multi-speaker voice, the speaker-conditioned bias of each row's slot
        if (cond && w.cond_off >= 0) {
            if (!lin.bias_slot) throw Error(19, "internal: a speaker-conditioned conv on a level without a slot table");
            p.bias = cond + w.cond_off; p.bias_slot = lin.bias_slot; p.ldbias = v.cond_rows;
        }
        // The layer's images name the kernels that can run it.  Backend 1 (default): conv_tf, else conv_tc; 2: conv_tc
        // (the text encoder and the duration predictor on fp32 CUDA cores, kept for A/B runs); 0: fp32 CUDA cores
        // everywhere.  Each try_launch plans once and returns false without launching when the shape is not supported.
        if (v.backend == 1 && w.wtf && try_launch_conv_tf(p, st)) {}
        else if (o.yt) throw Error(19, "internal: a transposed conv output needs the conv_tf kernel");
        else if (v.backend >= 1 && w.wtc && try_launch_conv_tc(p, st)) {}
        else if (!w.w) throw Error(19, "internal: no kernel for a conv without fp32 weights");
        else launch_conv_simt(p, st);
        const double vr = (double)lin.valid_rows;
        const int cout_w = (o.act == ACT_GATE) ? w.cout / 2 : w.cout;
        count(2.0 * vr * w.macs,
              4.0 * (vr * (w.cin + cout_w + ((o.res && o.res != x) ? w.cout : 0) + ((o.acc0 | o.acc1) ? w.cout : 0)) +
                     (double)w.macs));
    }

    void dds(const DDSW& d, float* x, float* t1, float* t2, const Level& L) {
        const int C = a.hidden;
        int dil = 1;
        for (int i = 0; i < 3; i++) {
            launch_dw_ln_gelu(x, d.wdw[i], d.bdw[i], a.dp_kernel, dil, d.g1[i], d.b1[i], t1, C, L.map, st);
            count(2.0 * L.valid_rows * C * a.dp_kernel, 8.0 * L.valid_rows * C);
            ConvCall o; o.y0 = t2; o.ldy0 = C;
            conv(d.c1x1[i], t1, C, L, o);
            launch_ln(t2, nullptr, x, d.g2[i], d.b2[i], x, C, 1, L.map, st);
            count(0, 12.0 * L.valid_rows * C);
            dil *= a.dp_kernel;
        }
    }
};

void d2d(float* dst, const float* src, size_t n, cudaStream_t st) {
    SB_CUDA(cudaMemcpyAsync(dst, src, n * 4, cudaMemcpyDeviceToDevice, st));
}

void expose(Job& j, const std::string& name, float* p, int cols, int level) {
    j.dbg[name] = {p, cols};
    j.dbg_level[name] = level;
}

// Each workspace below hands out its buffers in one carve(dev, pin).  plan() runs it on dry arenas to learn the sizes,
// makes room in the context's arenas and carves again for real, so no size is written down twice.
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

// Gives the next segment of a pass the slot of speaker `sid`, a new one for a speaker not seen before; false when sid
// is not a speaker of the voice.  On a single-speaker voice every segment has slot 0 and the pass has no slots.
bool assign_slot(FrameLayout& l, const Voice& v, long long sid) {
    if (v.num_speakers <= 1) { l.slot_of.push_back(0); return true; }
    if (sid < 0 || sid >= v.emb_rows) return false;
    const auto it = std::find(l.slot_sid.begin(), l.slot_sid.end(), (int)sid);
    l.slot_of.push_back((int)(it - l.slot_sid.begin()));
    if (it == l.slot_sid.end()) l.slot_sid.push_back((int)sid);
    return true;
}

// Speaker conditioning of a pass with speaker slots: the speaker of every slot and the effective biases of the
// speaker-conditioned convs, [slot][cond_rows].  Unset without slots.
struct SpeakerBias {
    Staged<int> sid; float* cond = nullptr;
    void carve(Arena& dev, Arena& pin, const Voice& v, const FrameLayout& l) {
        if (l.slot_sid.empty()) return;
        cond = dev.get<float>(l.slot_sid.size() * v.cond_rows);
        sid.carve(dev, pin, l.slot_sid.size());
    }
    // Fills the speaker table and launches the computation of the biases.
    void run(const Voice& v, const FrameLayout& l, cudaStream_t st) const {
        if (!cond) return;
        std::copy(l.slot_sid.begin(), l.slot_sid.end(), sid.h);
        sid.upload(st);
        launch_cond_bias(v.cond_w, v.cond_base, v.emb_g, sid.d, (int)sid.n, v.cond_rows, v.gin, cond, st);
    }
};

// The start of a pass on context c: its events are taken again from the first, and ev_begin is recorded.
void begin_pass(Context& c) {
    c.events_used = 0;
    if (!c.ev_begin) { SB_CUDA(cudaEventCreate(&c.ev_begin)); SB_CUDA(cudaEventCreate(&c.ev_end)); }
    SB_CUDA(cudaEventRecord(c.ev_begin, c.stream));
}

// Id level (phase 1): X tables, encoder and duration-predictor activations, and with debug the captures.
struct IdBufs {
    Staged<int> ids_rows, xend, xseg_of_gran, ylen; Staged<SegInfo> xsegs; Staged<TfTile> tiles;
    Staged<float> scales;                      // per utterance: noise_w [B], length_scale [B], noise_scale [B]
    Staged<int> xslot;                         // multi-speaker voices: speaker slot of every X granule
    SpeakerBias spk;
    int* cum;
    float *xa, *xb, *qkv, *att, *ffn, *stats, *d0, *t1, *t2, *g, *h29, *zz, *logw;
    float *att_s, *att_vt, *att_orel;          // tensor-core attention: scores of every head, V^T, relative-value term
    float* epsw;
    Staged<float> dscale; Staged<int> dframes; // per-id duration controls (only when the job has them)
    Staged<NoiseSeed> seeds;                   // per utterance (only when the job has seeds; read at both levels)
    float *qkv0, *att0, *p0, *vt0;             // debug: layer 0's attention operands and result
    std::vector<std::array<float*, 4>> dpf;    // debug: each duration flow's input, DDSConv output, spline parameters, output
    float* emb0;                               // debug: the scaled embedding, before layer 0
    // debug: each encoder layer's stages, ENC_* order (vt only with the tensor-core attention, stored [H][RX])
    enum { ENC_QKV, ENC_VT, ENC_ATT, ENC_O, ENC_LN1, ENC_FFN1, ENC_FFN2, ENC_LN2, ENC_NCAP };
    std::vector<std::array<float*, ENC_NCAP>> encl;

    void carve(Arena& dev, Arena& pin, const Job& j, bool tc_att) {
        const Voice& v = *j.v; const Arch& a = v.a;
        const int RX = j.RX, nxg = RX / GX, H = a.hidden;
        const size_t B = j.B, ntiles = j.tiles_s.size() + j.tiles_o.size();
        auto rows = [&](int cols) { return dev.get<float>((size_t)RX * cols); };
        ids_rows.carve(dev, pin, RX); xend.carve(dev, pin, nxg); xseg_of_gran.carve(dev, pin, nxg);
        xsegs.carve(dev, pin, B); ylen.carve(dev, pin, B);
        if (tc_att) tiles.carve(dev, pin, ntiles);
        scales.carve(dev, pin, 3 * B);
        if (!j.frames.slot_sid.empty()) xslot.carve(dev, pin, nxg);
        spk.carve(dev, pin, v, j.frames);
        cum = dev.get<int>(RX);
        xa = rows(H); xb = rows(H); qkv = rows(3 * H); att = rows(H); ffn = rows(a.filter); stats = rows(2 * a.inter);
        d0 = rows(H); t1 = rows(H); t2 = rows(H); g = rows(H); h29 = rows(32); zz = rows(2); logw = rows(1);
        att_s = att_vt = att_orel = nullptr;
        if (tc_att) { att_s = dev.get<float>((size_t)a.heads * RX * j.att_tp); att_vt = rows(H); att_orel = rows(H); }
        bool any_noise_w = false;
        for (const SynthConfig& c : j.cfgs) any_noise_w |= c.noise_w != 0.f;
        epsw = any_noise_w ? rows(2) : nullptr;
        if (!j.dur_scale.empty()) dscale.carve(dev, pin, RX);
        if (!j.dur_frames.empty()) dframes.carve(dev, pin, RX);
        if (!j.seeds.empty()) seeds.carve(dev, pin, B);
        qkv0 =att0 = p0 = vt0 = nullptr;
        emb0 = nullptr;
        dpf.clear();
        encl.clear();
        if (j.debug) {
            qkv0 = rows(3 * H); att0 = rows(H);
            if (tc_att) { p0 = rows(j.att_tp); vt0 = rows(H); }
            dpf.resize(v.dp_flows.size());
            for (auto& f : dpf) f = {rows(2), rows(H), rows(32), rows(2)};
            emb0 = rows(H);
            encl.resize(a.layers);
            for (auto& e : encl)
                e = {rows(3 * H), tc_att ? rows(H) : nullptr, rows(H), rows(H), rows(H), rows(a.filter), rows(H), rows(H)};
        }
    }
};

// Frame-level tables (segment end, owner and on multi-speaker voices speaker slot of every GY-frame tile, the segment
// list) of layout l.
struct FrameTables {
    Staged<int> yend, ftile, yslot; Staged<FrameSeg> fsegs;
    void carve(Arena& dev, Arena& pin, const FrameLayout& l) {
        const int ntile = l.RY / GY;
        yend.carve(dev, pin, ntile); ftile.carve(dev, pin, ntile); fsegs.carve(dev, pin, l.fsegs.size());
        if (!l.slot_sid.empty()) yslot.carve(dev, pin, ntile);
    }
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
    void add(const ResampleFilter* f, long long n_in, const Resampler* r = nullptr, bool last = false) {
        ResampleSeg s{};
        s.out_off = total; s.n_out = n_in; s.down = 1;
        if (f) {
            const long long N = (r ? r->consumed : 0) + n_in;
            s.taps = f->taps; s.up = f->up; s.down = f->down; s.H = f->H; s.K = f->K;
            s.n_out = resample_emit_end(*f, N, !r || last) - (r ? r->emitted : 0);
            if (r) {
                s.hist = r->hist[r->cur]; s.hist_out = r->hist[1 - r->cur];
                s.c = r->consumed; s.j0 = r->emitted; s.h = r->h; s.h_out = (int)std::min<long long>(N, f->K - 1);
            }
        }
        bytes += 4.0 * ((double)n_in + s.n_out);
        if (f) {
            smem = std::max(smem, resample_span(f->up, f->down, f->K));
            flops += 2.0 * (double)s.n_out * (2.0 * f->H + 1.0) / f->up;
            bytes += 4.0 * (double)f->up * f->K;
        }
        max_out = std::max(max_out, s.n_out);
        total += s.n_out;
        segs.push_back(s);
    }
};

// Device tables of a resample launch and their pinned mirrors: the segments, identity posts (for a launch whose input
// has no post-path, or for the i16 conversion of its output; out_gain[k], when given, is output k's gain there) and the
// output segments, n_out samples at out_off.
struct ResampleTables {
    Staged<ResampleSeg> segs; Staged<PcmPost> posts; Staged<FrameSeg> osegs;
    void carve(Arena& dev, Arena& pin, size_t n) {
        segs.carve(dev, pin, n); posts.carve(dev, pin, n); osegs.carve(dev, pin, n);
    }
    void upload(const ResamplePlan& p, cudaStream_t st, const std::vector<float>* out_gain = nullptr) {
        for (size_t k = 0; k < p.segs.size(); k++) {
            segs.h[k] = p.segs[k];
            posts.h[k] = PcmPost();
            if (out_gain) posts.h[k].gain = (*out_gain)[k];
            osegs.h[k] = FrameSeg{0, (int)p.segs[k].n_out, 0, 0, p.segs[k].out_off};
        }
        segs.upload(st); posts.upload(st); osegs.upload(st);
    }
};

// Device buffers of the prosody launches of plan p and the pinned mirrors of their tables: the segments, every frame's
// offset, the stretched signals of the segments that run both stages, and the output unless it goes elsewhere.  A plan
// of whole signals adds the output segments (n2 samples at y_off, for the launches that read the prosody output); a
// plan of stream windows the carry entry of every window and the staged input windows.
struct ProsodyBufs {
    Staged<ProsodySeg> segs; Staged<FrameSeg> osegs; Staged<ProsodyCarry> carry;
    int* offsets = nullptr; float *x = nullptr, *s = nullptr, *y = nullptr;
    void carve(Arena& dev, Arena& pin, const ProsodyPlan& p, bool own_y) {
        const size_t n = p.segs.size();
        y = nullptr;
        if (n == 0) return;
        segs.carve(dev, pin, n);
        if (p.in_total) {
            carry.carve(dev, pin, n);
            x = dev.get<float>((size_t)p.in_total + 4);
        } else {
            osegs.carve(dev, pin, n);
        }
        offsets = p.d_total ? dev.get<int>((size_t)p.d_total) : nullptr;
        s = p.s_total ? dev.get<float>((size_t)p.s_total + 4) : nullptr;
        if (own_y) y = dev.get<float>((size_t)p.y_total + 4);
    }
    // Fills and uploads the segments and, for whole signals, the output segments; a stream pass fills the carry.
    void upload(const ProsodyPlan& p, cudaStream_t st) const {
        for (size_t k = 0; k < p.segs.size(); k++) {
            segs.h[k] = p.segs[k];
            if (osegs.d) osegs.h[k] = FrameSeg{0, (int)p.segs[k].n2, 0, 0, p.segs[k].y_off};
        }
        segs.upload(st);
        if (osegs.d) osegs.upload(st);
    }
};

// The loudness launch over what a job hands out: one segment per utterance at its delivered rate, chunk scratch laid out
// back to back.
struct LoudnessPlan {
    std::vector<LoudSeg> segs;
    long long chunks = 0;
};

// Device tables of the loudness launch and their pinned mirrors: the segments, the chunk scratch and the results.
struct LoudnessBufs {
    Staged<LoudSeg> segs;
    double* scratch = nullptr;
    Staged<double> lufs; Staged<float> gain;
    void carve(Arena& dev, Arena& pin, const LoudnessPlan& p) {
        const size_t n = p.segs.size();
        if (n == 0) return;
        segs.carve(dev, pin, n);
        scratch = dev.get<double>((size_t)LD_SCRATCH * std::max<long long>(p.chunks, 1));
        lufs.carve(dev, pin, n); gain.carve(dev, pin, n);
    }
};

// Decoder over RY frames: conv_pre's output, then ping-pong stage buffers sized for the widest stage, or with debug one
// set per stage so every stage can be fetched.
struct DecoderBufs {
    float* p0;
    std::vector<std::array<float*, 5>> stage;    // per upsampling stage: up, ys, tmp[3]
    void carve(Arena& dev, const Voice& v, int RY, bool debug) {
        p0 = dev.get<float>((size_t)RY * v.a.up_init);
        stage.assign(v.ups.size(), {});
        int U = 1;
        if (debug) {
            for (size_t i = 0; i < v.ups.size(); i++) {
                U *= v.ups[i].u;
                for (auto& b : stage[i]) b = dev.get<float>((size_t)RY * U * v.ups[i].cout);
            }
            return;
        }
        size_t max_elems = 0;
        for (auto& st : v.ups) { U *= st.u; max_elems = std::max(max_elems, (size_t)RY * U * st.cout); }
        const int ntmp = (v.a.resblock == 2) ? 2 : 4;
        float* pool[6] = {nullptr};
        for (int i = 0; i < 2 + ntmp; i++) pool[i] = dev.get<float>(max_elems);
        for (size_t i = 0; i < v.ups.size(); i++)
            stage[i] = {pool[2], pool[i & 1], pool[3], ntmp > 2 ? pool[4] : nullptr, ntmp > 2 ? pool[5] : nullptr};
    }
    void expose_to(Job& j) const {
        const Voice& v = *j.v;
        expose(j, "dec.pre", p0, v.a.up_init, 1);
        int U = 1;
        for (size_t i = 0; i < v.ups.size(); i++) {
            U *= v.ups[i].u;
            expose(j, "dec.up" + std::to_string(i), stage[i][0], v.ups[i].cout, U);
            expose(j, "dec.mrf" + std::to_string(i), stage[i][1], v.ups[i].cout, U);
        }
    }
};

// Frame level of a synthesis pass (phase 2): tables, the latent, the flow's scratch, and unless the pass stops after
// the flow the decoder and (when the caller passed no buffer) the waveforms.  With prosody or output rates the decoder's
// waveforms are always the pass's own.  The prosody output (plan `pp`) is the pass's own too unless it is the result
// and the caller passed a buffer; the resampled waveforms go to the caller's buffer or to `rs`, with the tables of the
// resampling launch `rp`.
struct FrameBufs {
    FrameTables y;
    float *s, *epsz, *zp, *h, *acts, *outb, *wav;
    std::vector<float*> flow;                  // debug: z after each coupling layer, in the engine's channel order
    DecoderBufs dec;
    ResampleTables rt; float* rs;
    LoudnessBufs ld;
    ProsodyBufs pr;
    void carve(Arena& dev, Arena& pin, const Job& j, const ProsodyPlan& pp, const ResamplePlan& rp, const LoudnessPlan& lp,
               bool own_wav) {
        rt.carve(dev, pin, rp.segs.size());
        ld.carve(dev, pin, lp);
        pr.carve(dev, pin, pp, own_wav || !rp.segs.empty());
        rs = nullptr;
        if (!rp.segs.empty()) {
            if (own_wav) rs = dev.get<float>((size_t)rp.total + 4);
            own_wav = true;
        }
        if (!pp.segs.empty()) own_wav = true;
        const Arch& a = j.v->a;
        const size_t RY = (size_t)j.frames.RY;
        y.carve(dev, pin, j.frames);
        s = dev.get<float>(RY * a.inter);
        bool any_noise = false;
        for (const SynthConfig& c : j.cfgs) any_noise |= c.noise_scale != 0.f;
        epsz = any_noise ? dev.get<float>(RY * a.inter) : nullptr;
        zp = j.debug ? dev.get<float>(RY * a.inter) : nullptr;
        flow.assign(j.debug ? j.v->flows.size() : 0, nullptr);
        for (auto& p : flow) p = dev.get<float>(RY * a.inter);
        h = dev.get<float>(RY * a.hidden); acts = dev.get<float>(RY * a.hidden); outb = dev.get<float>(RY * a.hidden);
        wav = nullptr;
        if (j.encode_only) return;
        if (own_wav) wav = dev.get<float>((size_t)j.frames.total_samples + 4);
        dec.carve(dev, *j.v, j.frames.RY, j.debug);
    }
};

// One pass of streaming decoder chunks (layout l): speaker biases of every slot, tables, the gather table and the
// latent slices, the decoder and the waveforms; the post-path table when an output stage runs, the resample launch's
// tables and output, the i16 or G.711 scratch; and the pinned block the packed result (`total` values) is copied to.
struct ChunkBufs {
    SpeakerBias spk;
    FrameTables y;
    Staged<GatherSeg> src;
    float *s, *wav;
    DecoderBufs dec;
    Staged<PcmPost> post;
    ResampleTables rt; float* rs;
    void* pcm; unsigned* max;
    void* out_h;
    // warped chunks (plan `pp`): the prosody buffers, the output after the waveforms in `wav`, and the resample
    // launch's input table (the prosody output for a warped chunk, the post-path's chunk for the others)
    ProsodyBufs pr;
    Staged<FrameSeg> rin; Staged<PcmPost> rpost;
    void carve(Arena& dev, Arena& pin, const Voice& v, const FrameLayout& l, const ChunkPass& p, const ResamplePlan& rp,
               const ProsodyPlan& pp, size_t total) {
        const bool i16_out = p.format != PCM_F32;
        const size_t n = l.fsegs.size();
        spk.carve(dev, pin, v, l);
        y.carve(dev, pin, l);
        src.carve(dev, pin, n);
        s = dev.get<float>((size_t)l.RY * v.a.inter);
        wav = dev.get<float>((size_t)l.total_samples + (size_t)pp.y_total + 4);
        pr.carve(dev, pin, pp, false);
        if (!pp.segs.empty()) { rin.carve(dev, pin, n); rpost.carve(dev, pin, n); }
        dec.carve(dev, v, l.RY, false);
        if (p.resample || i16_out) post.carve(dev, pin, n);
        rt.carve(dev, pin, rp.segs.size());
        rs = p.resample ? dev.get<float>(total + 4) : nullptr;
        pcm = i16_out ? dev.alloc((total + 8) * pcm_bytes(p.format)) : nullptr;
        max = i16_out ? dev.get<unsigned>(n) : nullptr;
        out_h = pin.alloc(total * pcm_bytes(p.format));
    }
};

// decoder over an already-laid-out Y level: s [RY][inter] (gap rows zero) -> wav
void run_decoder(Runner& R, const Level& LY, const FrameTables& y, const DecoderBufs& d, const float* s, float* d_wav) {
    Voice& v = R.v; const Arch& a = R.a;
    const int RY = LY.map.rows;
    R.begin("dec.pre");
    { ConvCall o; o.y0 = d.p0; o.ldy0 = a.up_init; R.conv(v.conv_pre, s, a.inter, LY, o); }
    R.end();

    const float* cur = d.p0; Level Lin = LY; int U = 1;
    for (size_t i = 0; i < v.ups.size(); i++) {
        const UpStageW& st = v.ups[i];
        const int Uo = U * st.u;
        Level Lo; Lo.map = {y.yend.d, GY * Uo, Uo, RY * Uo}; Lo.valid_rows = LY.valid_rows * Uo;
        float *up = d.stage[i][0], *ys = d.stage[i][1];
        float* const* tmp = &d.stage[i][2];
        R.begin("dec.up" + std::to_string(i));
        if (v.backend >= 1 && st.fused.wtc) {
            // all u phases in one launch (input read once, N = u*cout columns).  Column block p of GEMM row q is output
            // row q*u + p, column n % cout, so with ldy0 = u*cout the output is the GEMM's own row-major matrix.
            ConvCall o; o.in_slope = 0.1f; o.y0 = up; o.ldy0 = st.fused.cout;
            R.conv(st.fused, cur, st.cin, Lin, o);
        } else {
            for (int p = 0; p < st.u; p++) {
                ConvCall o; o.in_slope = 0.1f; o.y0 = up; o.ldy0 = st.cout; o.orow_mul = st.u; o.orow_add = p;
                R.conv(st.phase[p], cur, st.cin, Lin, o);
            }
        }
        R.end();
        R.begin("dec.mrf" + std::to_string(i));
        // A 64-channel ResBlock2 stage is one fused launch: it reads its input once and writes the mean once, where the
        // six layer-wise convs each read and write a full activation.  The 32- and 128-channel stages stay layer-wise
        // (DESIGN.md section 3).
        if (v.backend >= 1 && a.resblock == 2 && st.cout == 64 && resblock2_tc_plan(st.res, Lo.map.rows, nullptr)) {
            launch_resblock2_tc(st.res, up, ys, Lo.map, R.st);
            const double vr = (double)Lo.valid_rows;
            double macs = 0;
            for (const ResBW& rb : st.res)
                for (const ConvW& w : rb.c1) macs += w.macs;
            R.count(2.0 * vr * macs, 4.0 * (vr * 2 * st.cout + macs));
            R.end();
            cur = ys; Lin = Lo; U = Uo;
            continue;
        }
        const float third = 1.0f / (float)st.res.size();
        for (size_t jb = 0; jb < st.res.size(); jb++) {
            const ResBW& rb = st.res[jb];
            const float* xb = up;
            const size_t nd = rb.dils.size();
            for (size_t m = 0; m < nd; m++) {
                const bool last = (m + 1 == nd);
                const float* cin_ptr = xb;
                if (a.resblock != 2) {
                    ConvCall o1; o1.in_slope = 0.1f; o1.y0 = tmp[0]; o1.ldy0 = st.cout;
                    R.conv(rb.c1[m], xb, st.cout, Lo, o1);
                    cin_ptr = tmp[0];
                }
                ConvCall o; o.in_slope = 0.1f; o.res = xb; o.ldres = st.cout;
                float* dst;
                if (last) { dst = ys; o.scale = third; o.acc0 = jb > 0 ? 1 : 0; }
                else dst = (a.resblock == 2) ? tmp[0] : tmp[1 + (m & 1)];
                o.y0 = dst; o.ldy0 = st.cout;
                R.conv(a.resblock == 2 ? rb.c1[m] : rb.c2[m], cin_ptr, st.cout, Lo, o);
                xb = dst;
            }
        }
        R.end();
        cur = ys; Lin = Lo; U = Uo;
    }
    R.begin("dec.post");
    launch_conv_post(cur, v.c_last, v.conv_post_w, d_wav, y.fsegs.d, y.ftile.d, U, Lin.map, R.st);
    R.count(2.0 * Lin.valid_rows * v.c_last * 7, 4.0 * Lin.valid_rows * (v.c_last + 1));
    R.end();
}

// Lays out the frame level for given per-segment frame counts (host side: segments, rows, output offsets).  xsegs: the
// X segments the frames come from (a job's utterances), or none (a chunk pass).
void lay_out_frames(FrameLayout& l, const std::vector<int>& y_len, int hop, const std::vector<SegInfo>& xsegs) {
    const size_t B = y_len.size();
    l.fsegs.resize(B);
    int cur = 0; long long out = 0;
    for (size_t b = 0; b < B; b++) {
        FrameSeg& f = l.fsegs[b];
        f.off = cur; f.len = y_len[b];
        f.xoff = b < xsegs.size() ? xsegs[b].off : 0;
        f.xlen = b < xsegs.size() ? xsegs[b].len : 0;
        f.out_off = out;
        out += (long long)y_len[b] * hop;
        cur += round_up(y_len[b] + HY, GY);
    }
    l.RY = cur; l.total_samples = out;
}

// The prosody launches of a job whose utterances ask for a pitch or a tempo (an empty plan when none does): every
// utterance's decoder waveform, with its ratios or NaN.
ProsodyPlan lay_out_prosody(const Job& j, int hop) {
    ProsodyPlan p;
    if (j.pitch.empty() || j.encode_only) return p;
    for (size_t b = 0; b < j.B; b++) {
        const FrameSeg& f = j.frames.fsegs[b];
        const long long n = (long long)f.len * hop;
        p.add(prosody_shape(j.v->sample_rate, n, j.pitch[b], j.tempo[b]), f.out_off, n);
    }
    return p;
}

// What the job hands out (osegs, out_hop, out_total): the frame layout itself without prosody and output rates (an empty
// plan), the prosody output without output rates (an empty plan too), else the segments of the returned plan, one
// utterance each at its rate, back to back, resampled from the prosody output when there is one.
ResamplePlan lay_out_output(Job& j, int hop, const ProsodyPlan& pp) {
    ResamplePlan p;
    j.osr.assign(j.B, j.v->sample_rate);
    if (j.out_rates.empty() || j.encode_only) {
        j.osegs = j.frames.fsegs; j.out_hop = hop; j.out_total = j.frames.total_samples;
        if (!pp.segs.empty()) {
            for (size_t b = 0; b < j.B; b++) j.osegs[b] = FrameSeg{0, (int)pp.segs[b].n2, 0, 0, pp.segs[b].y_off};
            j.out_hop = 1; j.out_total = pp.y_total;
        }
        return p;
    }
    j.osegs.assign(j.B, FrameSeg{});
    for (size_t b = 0; b < j.B; b++) {
        const ResampleFilter* f = nullptr;
        if (j.out_rates[b]) {
            j.osr[b] = j.out_rates[b];
            f = &voice_resampler(*j.v, j.out_rates[b], "utterance " + std::to_string(b) + ": ");
        }
        p.add(f, pp.segs.empty() ? (long long)j.frames.fsegs[b].len * hop : pp.segs[b].n2);
        j.osegs[b] = FrameSeg{0, (int)p.segs[b].n_out, 0, 0, p.segs[b].out_off};
    }
    j.out_hop = 1; j.out_total = p.total;
    return p;
}

// The resample launch of plan `p` (tables `t`) over the segments of wav, read through `posts`, into out: profile region
// "resample".
void run_resample(Runner& R, const ResamplePlan& p, const ResampleTables& t, const float* wav, const FrameSeg* fsegs,
                  const PcmPost* posts, int hop, float* out) {
    R.begin("resample");
    launch_resample(wav, fsegs, posts, hop, t.segs.d, (int)p.segs.size(), p.max_out, p.smem, out, R.st);
    R.count(p.flops, p.bytes);
    R.end();
}

// The prosody launches of plan `p` (buffers `t`) over the segments of wav into y: profile regions "stretch" (the offset
// chain and the overlap-add, which also copies the segments without a ratio) and "pitch".
void run_prosody(Runner& R, const ProsodyPlan& p, const ProsodyBufs& t, const float* wav, float* y) {
    const int n = (int)p.segs.size();
    R.begin("stretch");
    if (p.smem_ints) launch_prosody_offsets(wav, t.segs.d, n, p.smem_ints, t.offsets, R.st);
    launch_prosody_ola(wav, t.segs.d, n, p.max_ola, t.offsets, t.s, y, R.st);
    R.count(p.stretch_flops, p.stretch_bytes, p.smem_ints ? 2 : 1);
    R.end();
    if (p.max_pitch == 0) return;
    R.begin("pitch");
    launch_prosody_pitch(wav, t.s, t.segs.d, n, p.max_pitch, y, R.st);
    R.count(p.pitch_flops, p.pitch_bytes);
    R.end();
}

// The loudness launch of a job with targets (an empty plan without): every utterance as the job hands it out, at its
// rate, with its target or NaN.
LoudnessPlan lay_out_loudness(const Job& j) {
    LoudnessPlan p;
    if (j.loud_target.empty() || j.encode_only) return p;
    p.segs.resize(j.B);
    for (size_t b = 0; b < j.B; b++) {
        LoudSeg& s = p.segs[b];
        loudness_design(j.osr[b], s);
        s.off = j.osegs[b].out_off;
        s.n = (long long)j.osegs[b].len * j.out_hop;
        s.c0 = p.chunks;
        s.target = j.loud_target[b];
        p.chunks += (s.n + s.S - 1) / s.S;
    }
    return p;
}

// The loudness launch of plan `p` over wav in place, and the copy of its results to the pinned mirrors: profile region
// "loudness".  Its bytes are the samples read and, where a target scales them, written.
void run_loudness(Runner& R, const LoudnessPlan& p, const LoudnessBufs& t, float* wav) {
    const size_t n = p.segs.size();
    double samples = 0, scaled = 0;
    for (const LoudSeg& s : p.segs) {
        samples += (double)s.n;
        if (!std::isnan(s.target)) scaled += (double)s.n;
    }
    R.begin("loudness");
    launch_loudness(wav, t.segs.d, (int)n, t.scratch, t.lufs.d, t.gain.d, R.st);
    R.count(2.0 * 22.0 * samples, 4.0 * (samples + scaled));
    R.end();
    t.lufs.download(R.st);
    t.gain.download(R.st);
}

// Fills the frame-level tables of layout l through their pinned mirrors; returns the level.
Level upload_frames(const FrameLayout& l, const FrameTables& t, cudaStream_t st) {
    const size_t B = l.fsegs.size();
    Level L; L.map = {t.yend.d, GY, 1, l.RY}; L.valid_rows = 0; L.bias_slot = t.yslot.d;
    for (size_t b = 0; b < B; b++) {
        const int t0 = l.fsegs[b].off / GY;
        const int t1 = (b + 1 < B ? l.fsegs[b + 1].off : l.RY) / GY;
        for (int k = t0; k < t1; k++) {
            t.yend.h[k] = l.fsegs[b].off + l.fsegs[b].len; t.ftile.h[k] = (int)b;
            if (t.yslot.d) t.yslot.h[k] = l.slot_of[b];
        }
        L.valid_rows += l.fsegs[b].len;
    }
    std::copy(l.fsegs.begin(), l.fsegs.end(), t.fsegs.h);
    t.yend.upload(st);
    t.ftile.upload(st);
    t.fsegs.upload(st);
    if (t.yslot.d) t.yslot.upload(st);
    return L;
}

// Starts the copy of the batch's cum rows (up to the end of the last utterance: one copy, gap rows included) into the
// context's page-locked staging, on the job's stream; the caller synchronises.  The pass is over, so the staging of its
// tables is free.
const int* stage_cum(Job& j) {
    const SegInfo& last = j.xsegs[j.B - 1];
    const size_t n = (size_t)last.off + (size_t)last.len;
    Context& C = *j.ctx;
    C.pin.reserve(n * sizeof(int));
    int* h = C.pin.get<int>(n);
    SB_CUDA(cudaMemcpyAsync(h, j.d_cum, n * sizeof(int), cudaMemcpyDeviceToHost, C.stream));
    return h;
}

// Frames per id of utterance b, from the staged cum rows.
void cum_to_frames(const Job& j, const int* cum, size_t b, int* out) {
    const int* c = cum + j.xsegs[b].off;
    int prev = 0;
    for (int i = 0; i < j.xsegs[b].len; i++) { out[i] = c[i] - prev; prev = c[i]; }
}

}  // namespace

const std::vector<int>& job_id_frames(Job& j) {
    if (!j.ran) throw Error(19, "job has not run: no per-id frame counts yet");
    if (!j.id_frames.empty()) return j.id_frames;
    SB_CUDA(cudaSetDevice(j.v->device));
    const int* h = stage_cum(j);
    SB_CUDA(cudaStreamSynchronize(j.ctx->stream));
    j.id_frames.resize(j.ids.size());
    for (size_t b = 0; b < j.B; b++) cum_to_frames(j, h, b, j.id_frames.data() + j.offs[b]);
    return j.id_frames;
}

void Job::run(float* d_out, size_t d_out_cap) {
    Voice& V = *v; Context& C = *ctx; const Arch& a = V.a;
    SB_CUDA(cudaSetDevice(V.device));
    cudaStream_t st = C.stream;
    const int H = a.hidden, I = a.inter, F = a.filter;
    regions.clear(); dbg.clear(); dbg_level.clear(); id_frames.clear();

    // ---------------- id level (phase 1) workspace ----------------
    // tensor-core attention (two grouped GEMMs around a softmax): default backend, 96- or 48-wide heads, rows that fit
    // the softmax kernel's registers; otherwise the fp32 CUDA-core attention kernel
    const int D = H / a.heads;
    const bool tc_att = V.backend == 1 && (D == 96 || D == 48) && max_tx <= 1280 && getenv("SB200_ATT_SIMT") == nullptr;
    frames.slot_of.clear(); frames.slot_sid.clear();
    for (size_t b = 0; b < B; b++)      // piper/src/lib.rs:353-358: speaker.unwrap_or(0)
        if (!assign_slot(frames, V, cfgs[b].has_speaker ? cfgs[b].speaker : 0))
            throw Error(19, "Failed to run model inference. Error: speaker id out of range (utterance " + std::to_string(b) + ")");
    IdBufs x;
    plan(C.dev_id, C.pin, [&](Arena& dev, Arena& pin) { x.carve(dev, pin, *this, tc_att); });
    d_cum = x.cum;
    Runner R(V, C, regions, x.spk.cond);

    begin_pass(C);
    // tables
    const int nxg = RX / GX;
    std::fill(x.ids_rows.h, x.ids_rows.h + RX, -1);
    std::fill(x.xend.h, x.xend.h + nxg, 0);
    std::fill(x.xseg_of_gran.h, x.xseg_of_gran.h + nxg, 0);
    for (size_t b = 0; b < B; b++) {
        const SegInfo& s = xsegs[b];
        for (int i = 0; i < s.len; i++) x.ids_rows.h[s.off + i] = (int)ids[offs[b] + i];
        const int g0 = s.off / GX, g1 = (b + 1 < B ? xsegs[b + 1].off : RX) / GX;
        for (int g = g0; g < g1; g++) { x.xend.h[g] = s.off + s.len; x.xseg_of_gran.h[g] = (int)b; }
        x.scales.h[b] = cfgs[b].noise_w; x.scales.h[B + b] = cfgs[b].length_scale; x.scales.h[2 * B + b] = cfgs[b].noise_scale;
    }
    std::copy(xsegs.begin(), xsegs.end(), x.xsegs.h);
    x.ids_rows.upload(st);
    x.xend.upload(st);
    x.xseg_of_gran.upload(st);
    x.xsegs.upload(st);
    x.scales.upload(st);
    if (x.xslot.d) {
        for (int g = 0; g < nxg; g++) x.xslot.h[g] = frames.slot_of[x.xseg_of_gran.h[g]];
        x.xslot.upload(st);
    }
    // per-id duration controls: each id's value on its X row, `none` on the gap rows
    auto per_id = [&](const auto& t, const auto& vals, auto none) {
        if (!t.d) return;
        std::fill(t.h, t.h + RX, none);
        for (size_t b = 0; b < B; b++) std::copy(vals.begin() + offs[b], vals.begin() + offs[b + 1], t.h + xsegs[b].off);
        t.upload(st);
    };
    per_id(x.dscale, dur_scale, 1.f);
    per_id(x.dframes, dur_frames, -1);
    if (x.seeds.d) {
        std::copy(seeds.begin(), seeds.end(), x.seeds.h);
        x.seeds.upload(st);
    }
    if (tc_att) {
        std::copy(tiles_o.begin(), tiles_o.end(), std::copy(tiles_s.begin(), tiles_s.end(), x.tiles.h));
        x.tiles.upload(st);
    }

    Level LX; LX.map = {x.xend.d, GX, 1, RX}; LX.valid_rows = (long long)ids.size(); LX.bias_slot = x.xslot.d;
    TfGemm gs{}, go{};
    bool tc_att_ok = tc_att;
    if (tc_att) {
        gs.a = x.qkv; gs.a_rows = RX; gs.a_cols = 3 * H; gs.lda = 3 * H;
        gs.b = x.qkv; gs.b_rows = RX; gs.b_cols = 3 * H; gs.ldb = 3 * H;
        gs.nth = att_nth_s; gs.y = x.att_s; gs.ldy = att_tp; gs.res = nullptr; gs.scale = 1.0f / sqrtf((float)(H / a.heads));
        gs.tiles = x.tiles.d; gs.ntiles = (int)tiles_s.size();
        go.a = x.att_s; go.a_rows = a.heads * RX; go.a_cols = att_tp; go.lda = att_tp;
        go.b = x.att_vt; go.b_rows = H; go.b_cols = RX; go.ldb = RX;
        go.nth = att_nth_o; go.y = x.att; go.ldy = H; go.res = x.att_orel; go.scale = 1.f;
        go.tiles = x.tiles.d + tiles_s.size(); go.ntiles = (int)tiles_o.size();
        tc_att_ok = gemm_tf_supported(gs) && gemm_tf_supported(go);
    }
    if (debug) {
        expose(*this, "x", x.xa, H, 0); expose(*this, "stats", x.stats, 2 * I, 0);
        expose(*this, "qkv0", x.qkv0, 3 * H, 0); expose(*this, "att0", x.att0, H, 0);
        if (tc_att_ok) {
            expose(*this, "p0", x.p0, att_tp, 0);      // head 0 probabilities
            expose(*this, "vt0", x.vt0, H, -1);        // stored as [H][RX]
        }
        expose(*this, "dp.g", x.g, H, 0); expose(*this, "logw", x.logw, 1, 0);
        for (size_t s = 0; s < x.dpf.size(); s++) {
            const std::string fs = "dp.f" + std::to_string(s) + ".";
            expose(*this, fs + "in", x.dpf[s][0], 2, 0); expose(*this, fs + "h", x.dpf[s][1], H, 0);
            expose(*this, fs + "h29", x.dpf[s][2], 32, 0); expose(*this, fs + "out", x.dpf[s][3], 2, 0);
        }
        expose(*this, "enc.emb", x.emb0, H, 0);
        for (int l = 0; l < a.layers; l++) {
            const std::string p = "enc." + std::to_string(l) + ".";
            const auto& c = x.encl[l];
            expose(*this, p + "qkv", c[IdBufs::ENC_QKV], 3 * H, 0);
            if (tc_att_ok) expose(*this, p + "vt", c[IdBufs::ENC_VT], H, -1);   // stored as [H][RX]
            expose(*this, p + "att", c[IdBufs::ENC_ATT], H, 0); expose(*this, p + "o", c[IdBufs::ENC_O], H, 0);
            expose(*this, p + "ln1", c[IdBufs::ENC_LN1], H, 0); expose(*this, p + "ffn1", c[IdBufs::ENC_FFN1], F, 0);
            expose(*this, p + "ffn2", c[IdBufs::ENC_FFN2], H, 0); expose(*this, p + "ln2", c[IdBufs::ENC_LN2], H, 0);
        }
    }
    if (x.epsw) {
        if (!eps_w.empty()) {
            std::vector<float> stage((size_t)RX * 2, 0.f);
            for (size_t b = 0; b < B; b++)
                if (!eps_w[b].empty()) memcpy(stage.data() + (size_t)xsegs[b].off * 2, eps_w[b].data(), eps_w[b].size() * 4);
            SB_CUDA(cudaMemcpyAsync(x.epsw, stage.data(), stage.size() * 4, cudaMemcpyHostToDevice, st));
            SB_CUDA(cudaStreamSynchronize(st));   // `stage` is pageable; injection is a test-only path
        } else if (x.seeds.d) {
            launch_randn_seeded(x.epsw, 2, 0, V.noise_seed, 2 * noise_call, x.seeds.d, x.xsegs.d, x.xseg_of_gran.d, LX.map,
                                st);
        } else {
            launch_randn(x.epsw, (long long)RX * 2, V.noise_seed, 2 * noise_call, st);
        }
        if (debug) expose(*this, "eps_w", x.epsw, 2, 0);
    }

    // ---------------- speaker conditioning (multi-speaker voices) ----------------
    x.spk.run(V, frames, st);

    // ---------------- text encoder ----------------
    // Every contraction here reaches the duration predictor, and ceil(duration) is a cliff: the dense layers and the two
    // attention contractions run on conv_tf.cu (wgmma, error-compensated tf32, chunk-flushed accumulation: fp32-class
    // accuracy, DESIGN.md section 4); backend 0 / 2 keep them on the fp32 CUDA-core kernels.
    R.begin("enc");
    launch_embed(x.ids_rows.d, V.emb, sqrtf((float)H), x.xa, RX, H, st);
    R.count(0, 4.0 * LX.valid_rows * H);
    // debug: every stage is copied right after its launch (xa and xb are overwritten in place)
    if (debug) d2d(x.emb0, x.xa, (size_t)RX * H, st);
    for (int l = 0; l < a.layers; l++) {
        const EncLayer& e = V.enc[l];
        float* const* cap = debug ? x.encl[l].data() : nullptr;
        {
            ConvCall o; o.y0 = x.qkv; o.ldy0 = 3 * H;
            if (tc_att_ok) { o.yt = x.att_vt; o.yt_col0 = 2 * H; o.ldyt = RX; }       // V leaves transposed: [H][RX]
            R.conv(e.qkv, x.xa, H, LX, o);
        }
        if (cap) {
            d2d(cap[IdBufs::ENC_QKV], x.qkv, (size_t)RX * 3 * H, st);
            if (tc_att_ok) d2d(cap[IdBufs::ENC_VT], x.att_vt, (size_t)H * RX, st);
        }
        if (tc_att_ok) {
            launch_gemm_tf(gs, st);
            launch_attn_softmax(x.att_s, att_tp, x.qkv, 3 * H, e.relk, e.relv, a.window, x.att_orel, H, H, a.heads, RX,
                                x.xsegs.d, x.xseg_of_gran.d, GX, max_tx, st);
            launch_gemm_tf(go, st);
            R.count(0, 0, 2);
        } else {
            launch_attention(x.qkv, 3 * H, e.relk, e.relv, a.window, x.att, H, H, a.heads, x.xsegs.d, (int)B, max_tx, st);
        }
        { double f = 0; for (auto& s : xsegs) f += 4.0 * (double)s.len * s.len * H; R.count(f, 16.0 * LX.valid_rows * H); }
        if (debug && l == 0) {      // first-layer attention operands / result (tests/test_gpu_parity.py)
            d2d(x.qkv0, x.qkv, (size_t)RX * 3 * H, st);
            d2d(x.att0, x.att, (size_t)RX * H, st);
            if (tc_att_ok) {
                d2d(x.p0, x.att_s, (size_t)RX * att_tp, st);
                // V went only to att_vt (the V columns of qkv0 are not written on this path)
                d2d(x.vt0, x.att_vt, (size_t)H * RX, st);
            }
        }
        if (cap) d2d(cap[IdBufs::ENC_ATT], x.att, (size_t)RX * H, st);
        { ConvCall o; o.y0 = x.xb; o.ldy0 = H; R.conv(e.o, x.att, H, LX, o); }
        if (cap) d2d(cap[IdBufs::ENC_O], x.xb, (size_t)RX * H, st);
        launch_ln(x.xa, x.xb, nullptr, e.g1, e.b1, x.xa, H, 0, LX.map, st);
        R.count(0, 12.0 * LX.valid_rows * H);
        if (cap) d2d(cap[IdBufs::ENC_LN1], x.xa, (size_t)RX * H, st);
        { ConvCall o; o.act = ACT_RELU; o.y0 = x.ffn; o.ldy0 = F; R.conv(e.ffn1, x.xa, H, LX, o); }
        if (cap) d2d(cap[IdBufs::ENC_FFN1], x.ffn, (size_t)RX * F, st);
        { ConvCall o; o.y0 = x.xb; o.ldy0 = H; R.conv(e.ffn2, x.ffn, F, LX, o); }
        if (cap) d2d(cap[IdBufs::ENC_FFN2], x.xb, (size_t)RX * H, st);
        launch_ln(x.xa, x.xb, nullptr, e.g2, e.b2, x.xa, H, 0, LX.map, st);
        R.count(0, 12.0 * LX.valid_rows * H);
        if (cap) d2d(cap[IdBufs::ENC_LN2], x.xa, (size_t)RX * H, st);
    }
    { ConvCall o; o.y0 = x.stats; o.ldy0 = 2 * I; R.conv(V.enc_proj, x.xa, H, LX, o); }
    R.end();

    // ---------------- stochastic duration predictor (reverse) ----------------
    R.begin("dp");
    { ConvCall o; o.y0 = x.d0; o.ldy0 = H; R.conv(V.dp_pre, x.xa, H, LX, o); }
    R.dds(V.dp_dds, x.d0, x.t1, x.t2, LX);
    { ConvCall o; o.y0 = x.g; o.ldy0 = H; R.conv(V.dp_proj, x.d0, H, LX, o); }
    launch_scale_copy2(x.epsw, x.scales.d, x.xseg_of_gran.d, x.zz, LX.map, st);
    // debug: zz, d0 and h29 are reused by every flow, so each flow's stages are captured as copies
    for (size_t s = 0; s < V.dp_flows.size(); s++) {
        const CFlowW& cf = V.dp_flows[s];
        if (debug) d2d(x.dpf[s][0], x.zz, (size_t)RX * 2, st);
        launch_flow_pre(x.zz, cf.ccol, cf.pre_w, cf.pre_b, x.g, x.d0, H, LX.map, st);
        R.count(2.0 * LX.valid_rows * H, 8.0 * LX.valid_rows * H);
        R.dds(cf.dds, x.d0, x.t1, x.t2, LX);
        if (debug) d2d(x.dpf[s][1], x.d0, (size_t)RX * H, st);
        { ConvCall o; o.y0 = x.h29; o.ldy0 = 32; R.conv(cf.proj, x.d0, H, LX, o); }
        if (debug) d2d(x.dpf[s][2], x.h29, (size_t)RX * 32, st);
        launch_spline(x.h29, 32, x.zz, cf.tcol, a.dp_bins, 1.0f / sqrtf((float)H), LX.map, st);
        R.count(0, 4.0 * LX.valid_rows * 34);
        if (debug) d2d(x.dpf[s][3], x.zz, (size_t)RX * 2, st);
    }
    launch_durations(x.zz, V.ea_m0, V.ea_logs0, x.scales.d + B, x.xsegs.d, (int)B, x.logw, x.cum, x.ylen.d, st,
                     x.dscale.d, x.dframes.d);
    R.end();

    // ---------------- host learns the frame counts (the graph's data-dependent shape) ----------------
    x.ylen.download(st);
    SB_CUDA(cudaStreamSynchronize(st));
    y_len.assign(x.ylen.h, x.ylen.h + B);
    long long tot_frames = 0;
    for (int y : y_len) tot_frames += y;
    if (tot_frames > (long long)(2.0e9 / 256 / 4)) throw Error(19, "Failed to run model inference. Error: predicted durations are unreasonably long");
    if (!eps_z.empty())
        for (size_t b = 0; b < B; b++)
            if (!eps_z[b].empty() && eps_z_frames[b] != (size_t)y_len[b])
                throw Error(19, "injected eps_z has " + std::to_string(eps_z_frames[b]) + " frames but the model produced " + std::to_string(y_len[b]));

    // ---------------- frame level (phase 2) workspace ----------------
    // The stream is idle here, so the pinned staging of the X tables can be reused for the Y tables.
    lay_out_frames(frames, y_len, a.hop(), xsegs);
    const ProsodyPlan pp = lay_out_prosody(*this, a.hop());
    const bool prosody = !pp.segs.empty();
    const ResamplePlan rp = lay_out_output(*this, a.hop(), pp);
    const bool resample = !rp.segs.empty();
    const LoudnessPlan lp = lay_out_loudness(*this);
    loud_ran.clear(); loud_lufs.clear(); loud_gain.clear(); pros_ran.clear();
    FrameBufs f;
    plan(C.dev_frame, C.pin, [&](Arena& dev, Arena& pin) { f.carve(dev, pin, *this, pp, rp, lp, d_out == nullptr); });
    d_osegs = resample ? f.rt.osegs.d : prosody ? f.pr.osegs.d : f.y.fsegs.d;
    if (debug) {
        expose(*this, "z_p", f.zp, I, 1); expose(*this, "z", f.s, I, 1);
        // flow.{f}: z after the coupling layer of the graph's flow.flows.{2f} (f = flow_n - 1 first).  The graph's Flip
        // layers are folded into the weights, so z keeps z_p's channel order throughout: after an odd number of
        // couplings the graph's z is this capture reversed along channels, after an even number it is the capture.
        for (size_t s = 0; s < f.flow.size(); s++) expose(*this, "flow." + std::to_string(a.flow_n - 1 - (int)s), f.flow[s], I, 1);
        if (!encode_only) f.dec.expose_to(*this);
    }
    Level LY = upload_frames(frames, f.y, st);
    if (prosody) f.pr.upload(pp, st);
    if (resample) f.rt.upload(rp, st);
    if (!lp.segs.empty()) {
        std::copy(lp.segs.begin(), lp.segs.end(), f.ld.segs.h);
        f.ld.segs.upload(st);
    }

    // ---------------- alignment expansion ----------------
    R.begin("align");
    const int RY = frames.RY;
    if (f.epsz) {
        if (!eps_z.empty()) {
            std::vector<float> stage((size_t)RY * I, 0.f);
            for (size_t b = 0; b < B; b++)
                if (!eps_z[b].empty()) memcpy(stage.data() + (size_t)frames.fsegs[b].off * I, eps_z[b].data(), eps_z[b].size() * 4);
            SB_CUDA(cudaMemcpyAsync(f.epsz, stage.data(), stage.size() * 4, cudaMemcpyHostToDevice, st));
            SB_CUDA(cudaStreamSynchronize(st));
        } else if (x.seeds.d) {
            launch_randn_seeded(f.epsz, I, 1, V.noise_seed, 2 * noise_call + 1, x.seeds.d, f.y.fsegs.d, f.y.ftile.d, LY.map,
                                st);
        } else {
            launch_randn(f.epsz, (long long)RY * I, V.noise_seed, 2 * noise_call + 1, st);
        }
        if (debug) expose(*this, "eps_z", f.epsz, I, 1);
    }
    launch_expand(x.stats, 2 * I, I, x.cum, f.epsz, x.scales.d + 2 * B, f.s, f.y.fsegs.d, f.y.ftile.d, LY.map, st);
    R.count(0, 4.0 * LY.valid_rows * 3 * I);
    R.end();
    if (debug) d2d(f.zp, f.s, (size_t)RY * I, st);

    // ---------------- residual-coupling flow (reverse) ----------------
    R.begin("flow");
    for (size_t step = 0; step < V.flows.size(); step++) {
        const CouplingW& cp = V.flows[step];
        { ConvCall o; o.y0 = f.h; o.ldy0 = H; R.conv(cp.pre, f.s + cp.cond_off, I, LY, o); }
        const int n = (int)cp.in.size();
        for (int l = 0; l < n; l++) {
            { ConvCall o; o.act = ACT_GATE; o.y0 = f.acts; o.ldy0 = H; R.conv(cp.in[l], f.h, H, LY, o); }
            ConvCall o;
            if (l < n - 1) { o.y0 = f.h; o.ldy0 = H; o.acc0 = 1; o.split = H; o.y1 = f.outb; o.ldy1 = H; o.acc1 = l > 0; }
            else { o.split = 0; o.y0 = f.outb; o.ldy0 = H; o.y1 = f.outb; o.ldy1 = H; o.acc1 = l > 0; }
            R.conv(cp.rs[l], f.acts, H, LY, o);
        }
        { ConvCall o; o.y0 = f.s + cp.tgt_off; o.ldy0 = I; o.acc0 = 1; o.scale = -1.f; R.conv(cp.post, f.outb, H, LY, o); }
        if (debug) d2d(f.flow[step], f.s, (size_t)RY * I, st);
    }
    R.end();

    // ---------------- HiFi-GAN ----------------
    if (encode_only) {
        z_dev = f.s;
        SB_CUDA(cudaEventRecord(C.ev_end, st));
        SB_CUDA(cudaStreamSynchronize(st));
        SB_CUDA(cudaGetLastError());
        SB_CUDA(cudaEventElapsedTime(&last_ms, C.ev_begin, C.ev_end));
        ran = true;
        return;
    }
    if (d_out) {
        if ((size_t)out_total > d_out_cap) throw Error(19, "caller-provided device output buffer is too small");
        d_wav = d_out;
    } else {
        d_wav = f.rs ? f.rs : f.pr.y ? f.pr.y : f.wav;
    }
    run_decoder(R, LY, f.y, f.dec, f.s, resample || prosody ? f.wav : d_wav);
    // the output stage: prosody on the decoder's waveform, the resample launch on what that left, loudness on the result
    const float* staged = f.wav; const FrameSeg* staged_segs = f.y.fsegs.d; int staged_hop = a.hop();
    if (prosody) {
        float* py = resample ? f.pr.y : d_wav;
        run_prosody(R, pp, f.pr, f.wav, py);
        staged = py; staged_segs = f.pr.osegs.d; staged_hop = 1;
    }
    if (resample) run_resample(R, rp, f.rt, staged, staged_segs, f.rt.posts.d, staged_hop, d_wav);
    if (!lp.segs.empty()) run_loudness(R, lp, f.ld, d_wav);
    SB_CUDA(cudaEventRecord(C.ev_end, st));
    SB_CUDA(cudaStreamSynchronize(st));
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaEventElapsedTime(&last_ms, C.ev_begin, C.ev_end));
    for (Region& r : regions) cudaEventElapsedTime(&r.ms, r.e0, r.e1);
    pros_ran = pp.shapes;
    if (!lp.segs.empty()) {
        loud_ran = loud_target;
        loud_lufs.assign(f.ld.lufs.h, f.ld.lufs.h + B);
        loud_gain.assign(f.ld.gain.h, f.ld.gain.h + B);
    }
    ran = true;
}

// ====================================================================== streaming halves
std::vector<Latent*> encode_latents(Voice* v, const long long* ids, const size_t* offs, size_t B, const SynthConfig* cfgs,
                                    const float* scale, const int* frames, const unsigned long long* seeds,
                                    const int* seeded) {
    std::unique_ptr<Job> j(create_job(v, ids, offs, B, nullptr, nullptr, nullptr, false));
    if (cfgs) set_job_configs(*j, cfgs);
    set_job_durations(*j, scale, frames);
    set_job_seeds(*j, seeds, seeded);
    j->encode_only = true;
    j->run(nullptr, 0);
    const size_t I = (size_t)v->a.inter;
    size_t total = 0;
    for (int f : j->y_len) total += (size_t)f;
    // one allocation for the whole pass: cudaMalloc synchronises the device, so B of them would stall other streams B times
    float* p = nullptr;
    SB_CUDA(cudaMalloc(&p, std::max<size_t>(total, 1) * I * 4));
    const int dev = v->device;
    std::shared_ptr<float> mem(p, [dev](float* q) { cudaSetDevice(dev); cudaFree(q); });
    std::vector<std::unique_ptr<Latent>> ls(B);
    size_t row = 0;
    for (size_t b = 0; b < B; b++) {
        Latent& L = *(ls[b] = std::unique_ptr<Latent>(new Latent()));
        L.v = v; L.mem = mem; L.z = p + row * I; L.frames = j->y_len[b];
        L.sid = j->cfgs[b].has_speaker ? j->cfgs[b].speaker : 0;
        SB_CUDA(cudaMemcpyAsync(L.z, j->z_dev + (size_t)j->frames.fsegs[b].off * I, (size_t)L.frames * I * 4,
                                cudaMemcpyDeviceToDevice, j->ctx->stream));
        row += (size_t)L.frames;
    }
    const int* cum = stage_cum(*j);
    SB_CUDA(cudaStreamSynchronize(j->ctx->stream));
    for (size_t b = 0; b < B; b++) {
        ls[b]->id_frames.resize(j->offs[b + 1] - j->offs[b]);
        cum_to_frames(*j, cum, b, ls[b]->id_frames.data());
    }
    std::vector<Latent*> out(B);
    for (size_t b = 0; b < B; b++) out[b] = ls[b].release();
    return out;
}

Latent* encode_latent(Voice* v, const long long* ids, size_t n) {
    const size_t offs[2] = {0, n};
    return encode_latents(v, ids, offs, 1, nullptr)[0];
}

// crossfade table of AudioSamples::crossfade (audio/ops/src/samples.rs:144-157) for a buffer of `len` samples
static void fill_fade(PcmPost& p, int fade, long long len) {
    const long long n = std::min<long long>(fade, len / 2);
    p.fade_n = (int)std::min<long long>(n, 48);
    const float att = (float)(p.fade_n - 1);
    for (int i = 0; i < p.fade_n; i++) p.tab[i] = sinf(((float)i / att) * 3.14159265358979f / 2.0f);
}

// The chunks are laid out as the segments of one frame level.  The pass runs the decoder, then its output stage: the
// prosody launches of the chunks with a pitch / tempo stream, which read the waveforms through the post-path, the
// resample launch, which reads their output or the waveforms through the post-path, and the i16 (or G.711) conversion,
// which applies the post-path itself when no resample launch ran.  The packed result comes back in one copy through the
// context's page-locked staging, and only then do the resamplers and prosody streams advance.
void decode_chunks(Voice* v, const ChunkPass& p, ChunkResult& out) {
    out.f32.clear(); out.i16.clear(); out.g711.clear(); out.ms = out.stretch_ms = out.pitch_ms = 0.f;
    const size_t n = p.chunks.size();
    if (n == 0) return;
    if (p.format < PCM_F32 || p.format > PCM_ALAW)
        throw Error(19, "format " + std::to_string(p.format) + " is not 0 (f32), 1 (i16), 2 (mu-law) or 3 (A-law)");
    const int hop = v->a.hop();
    FrameLayout l;
    std::vector<int> len(n);
    auto fail = [&p](size_t k, const std::string& what, const std::string& detail) {
        throw Error(19, p.single ? what : "chunk " + std::to_string(k) + ": " + what + detail);
    };
    for (size_t k = 0; k < n; k++) {
        const ChunkSpec& c = p.chunks[k];
        if (!c.z || c.z->v != v) fail(k, "the latent was not encoded by this voice", "");
        if (c.lo < 0 || c.lo >= c.hi || c.hi > c.z->frames)
            fail(k, "Invalid model audio output", " (frames [" + std::to_string(c.lo) + ", " + std::to_string(c.hi) +
                                                  ") of a latent of " + std::to_string(c.z->frames) + ")");
        if (c.trim_lo < 0 || c.trim_hi < 0 || c.trim_lo + c.trim_hi >= c.hi - c.lo)
            fail(k, "Invalid model audio output", " (trim)");
        // decoder.onnx takes the encoder's `g` (piper/src/lib.rs:706-735, 739-743)
        if (!assign_slot(l, *v, c.z->sid)) fail(k, "Failed to run model inference. Error: speaker id out of range", "");
        len[k] = (int)(c.hi - c.lo);
        if (const Resampler* r = c.rs) {
            if (r->v != v) fail(k, "the resampler was made for another voice", "");
            if (r->ended) fail(k, "the resampler's stream has already been flushed", "");
            for (size_t q = 0; q < k; q++)
                if (p.chunks[q].rs == r) fail(k, "the resampler of chunk " + std::to_string(q) + " appears twice in one call", "");
        }
        if (const ProsodyStream* w = c.ps) {
            if (!p.resample) fail(k, "a prosody stream needs a resampled chunk pass", "");
            if (w->v != v) fail(k, "the prosody stream was made for another voice", "");
            if (w->ended) fail(k, "the prosody stream has already been flushed", "");
            for (size_t q = 0; q < k; q++)
                if (p.chunks[q].ps == w)
                    fail(k, "the prosody stream of chunk " + std::to_string(q) + " appears twice in one call", "");
        }
        if ((c.rs || c.ps) && c.last != 0 && c.last != 1)
            fail(k, "last flag " + std::to_string(c.last) + " is neither 0 nor 1", "");
    }
    // samples of each chunk after its trims, what its prosody stream emits for them, and the resample launch
    std::vector<long long> n_in(n), n_res(n);     // n_res: what the resample launch takes (a warped chunk's output)
    std::vector<ProsodyStep> steps(n);
    std::vector<int> warped;
    ProsodyPlan pp;
    ResamplePlan rp;
    for (size_t k = 0; k < n; k++) {
        const ChunkSpec& c = p.chunks[k];
        n_in[k] = (c.hi - c.lo - c.trim_lo - c.trim_hi) * hop;
        n_res[k] = n_in[k];
        if (c.ps) {
            steps[k] = prosody_stream_step(*c.ps, n_in[k], c.last != 0);
            pp.add_stream(*c.ps, steps[k]);
            warped.push_back((int)k);
            n_res[k] = steps[k].j1 - steps[k].j0;
        }
        if (p.resample) rp.add(c.rs ? &c.rs->f : nullptr, n_res[k], c.rs, c.last != 0);
    }

    const auto release = [v](Context* c) { v->release(c); };
    const std::unique_ptr<Context, decltype(release)> ctx(v->acquire(), release);
    Context& C = *ctx;
    SB_CUDA(cudaSetDevice(v->device));
    lay_out_frames(l, len, hop, {});
    const size_t total = p.resample ? (size_t)rp.total : (size_t)l.total_samples;
    ChunkBufs b;
    plan(C.dev_frame, C.pin, [&](Arena& dev, Arena& pin) { b.carve(dev, pin, *v, l, p, rp, pp, total); });
    cudaStream_t st = C.stream;
    std::vector<Region> regions;
    Runner R(*v, C, regions, b.spk.cond);
    begin_pass(C);
    b.spk.run(*v, l, st);
    Level LY = upload_frames(l, b.y, st);
    for (size_t k = 0; k < n; k++) b.src.h[k] = GatherSeg{p.chunks[k].z->z, p.chunks[k].lo, l.fsegs[k].off, len[k]};
    b.src.upload(st);
    launch_gather_rows(b.src.d, b.y.ftile.d, GY, l.RY, v->a.inter, b.s, st);
    run_decoder(R, LY, b.y, b.dec, b.s, b.wav);
    // G.711 of resampled chunks: the gain scales the resampled samples just before the conversion, as a volume on the
    // delivered audio (resampling x * g is not bit for bit resampling x, then times g)
    const bool gain_after = p.resample && p.format >= PCM_MULAW;
    std::vector<float> out_gain;
    if (gain_after)
        for (const ChunkSpec& c : p.chunks) out_gain.push_back(c.gain);
    if (b.post.d) {
        for (size_t k = 0; k < n; k++) {
            PcmPost& q = b.post.h[k];
            q = PcmPost();
            q.gain = gain_after ? 1.f : p.chunks[k].gain;
            q.trim_lo = p.chunks[k].trim_lo * hop;
            q.trim_hi = p.chunks[k].trim_hi * hop;
            if (p.fade > 0) fill_fade(q, p.fade, n_in[k]);
        }
        b.post.upload(st);
    }
    // warped chunks: prosody on the post-path's samples, then the resample launch reads its output (n samples at
    // `off` as a segment of ceil(n / hop) frames less a trim, with no post-path of its own)
    const FrameSeg* rs_in = b.y.fsegs.d; const PcmPost* rs_post = b.post.d;
    if (!warped.empty()) {
        float* py = b.wav + l.total_samples;
        b.pr.upload(pp, st);
        for (size_t q = 0; q < warped.size(); q++)
            b.pr.carry.h[q] = prosody_carry(*p.chunks[warped[q]].ps, steps[warped[q]], warped[q]);
        b.pr.carry.upload(st);
        R.begin("stretch");
        launch_prosody_stream_stretch(pp, b.pr.segs.d, b.pr.carry.d, b.wav, b.y.fsegs.d, b.post.d, hop, b.pr.x, b.pr.s,
                                      b.pr.offsets, py, st);
        R.count(pp.stretch_flops, pp.stretch_bytes, 2 + (pp.smem_ints ? 1 : 0) + (pp.max_ola ? 1 : 0));
        R.end();
        if (pp.max_pitch) {
            R.begin("pitch");
            launch_prosody_pitch(b.pr.x, b.pr.s, b.pr.segs.d, (int)warped.size(), pp.max_pitch, py, st);
            R.count(pp.pitch_flops, pp.pitch_bytes);
            R.end();
        }
        std::copy(l.fsegs.begin(), l.fsegs.end(), b.rin.h);
        std::copy(b.post.h, b.post.h + n, b.rpost.h);
        for (size_t q = 0; q < warped.size(); q++) {
            const ProsodySeg& g = pp.segs[q];
            const long long m = g.j1 - g.j0, frames = (m + hop - 1) / hop;
            b.rin.h[warped[q]] = FrameSeg{0, (int)frames, 0, 0, l.total_samples + g.y_off};
            b.rpost.h[warped[q]] = PcmPost();
            b.rpost.h[warped[q]].trim_hi = frames * hop - m;
        }
        b.rin.upload(st);
        b.rpost.upload(st);
        rs_in = b.rin.d; rs_post = b.rpost.d;
    }
    if (p.resample) {
        b.rt.upload(rp, st, gain_after ? &out_gain : nullptr);
        run_resample(R, rp, b.rt, b.wav, rs_in, rs_post, hop, b.rs);
        if (b.pcm) launch_pcm(b.rs, b.rt.osegs.d, b.rt.posts.d, (int)n, 1, rp.max_out, b.max, p.format, b.pcm, st);
    } else if (b.pcm) {
        launch_pcm(b.wav, b.y.fsegs.d, b.post.d, (int)n, hop, (long long)*std::max_element(len.begin(), len.end()) * hop,
                   b.max, p.format, b.pcm, st);
    }
    SB_CUDA(cudaEventRecord(C.ev_end, st));
    const void* res = b.pcm ? (const void*)b.pcm : b.rs ? (const void*)b.rs : (const void*)b.wav;
    SB_CUDA(cudaMemcpyAsync(b.out_h, res, total * pcm_bytes(p.format), cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    SB_CUDA(cudaGetLastError());

    for (size_t k = 0; k < n; k++) {
        Resampler* r = p.chunks[k].rs;
        if (!r) continue;
        const ResampleSeg& s = rp.segs[k];
        r->consumed = s.c + n_res[k];
        r->emitted = s.j0 + s.n_out;
        r->cur ^= 1;
        r->h = s.h_out;
        r->ended = p.chunks[k].last != 0;
    }
    for (Region& g : regions) {
        if (g.name != "stretch" && g.name != "pitch") continue;
        cudaEventElapsedTime(&g.ms, g.e0, g.e1);
        (g.name == "stretch" ? out.stretch_ms : out.pitch_ms) = g.ms;
    }
    for (int k : warped) {
        ProsodyStream& w = *p.chunks[k].ps;
        prosody_stream_advance(w, steps[k], p.chunks[k].last != 0);
        w.last_ms[0] = out.stretch_ms; w.last_ms[1] = out.pitch_ms;
    }
    if (p.format == PCM_I16) out.i16.resize(n); else if (b.pcm) out.g711.resize(n); else out.f32.resize(n);
    for (size_t k = 0; k < n; k++) {
        const long long o = p.resample ? rp.segs[k].out_off : l.fsegs[k].out_off;
        const long long m = p.resample ? rp.segs[k].n_out : n_in[k];
        if (p.format == PCM_I16) {
            const int16_t* h = static_cast<const int16_t*>(b.out_h);
            out.i16[k].assign(h + o, h + o + m);
        } else if (b.pcm) {
            const uint8_t* h = static_cast<const uint8_t*>(b.out_h);
            out.g711[k].assign(h + o, h + o + m);
        } else {
            const float* h = static_cast<const float*>(b.out_h);
            out.f32[k].assign(h + o, h + o + m);
        }
    }
    cudaEventElapsedTime(&out.ms, C.ev_begin, C.ev_end);
}

namespace {
// The i16 conversion of a finished job in format `fmt` (PCM_I16 or a G.711 law), utterance b after gains[b], into
// stream-ordered scratch laid out like the job's waveforms.  The scratch goes back to the pool with the object, so
// device memory held after a run does not grow.
struct JobPcm {
    cudaStream_t st = nullptr;
    void* d_pcm = nullptr; unsigned* d_max = nullptr; PcmPost* d_post = nullptr;
    JobPcm(Job& j, int fmt, const float* gains) {
        if (!j.ran || j.encode_only) throw Error(19, "job has not produced audio");
        SB_CUDA(cudaSetDevice(j.v->device));
        st = j.ctx->stream;
        const int hop = j.out_hop;
        const size_t n = (size_t)j.out_total;
        long long mx = 0;
        for (size_t b = 0; b < j.B; b++) mx = std::max<long long>(mx, (long long)j.osegs[b].len * hop);
        SB_CUDA(cudaMallocAsync(&d_pcm, n * pcm_bytes(fmt) + 16, st));
        SB_CUDA(cudaMallocAsync(&d_max, sizeof(unsigned) * j.B, st));
        SB_CUDA(cudaMallocAsync(&d_post, sizeof(PcmPost) * j.B, st));
        std::vector<PcmPost> posts(j.B);
        for (size_t b = 0; b < j.B; b++) posts[b].gain = gains[b];
        // a loudness-normalised utterance keeps its level: fixed scale instead of its own peak
        for (size_t b = 0; b < j.loud_ran.size(); b++) posts[b].fixed_scale = std::isnan(j.loud_ran[b]) ? 0 : 1;
        // pageable source: the call returns once the entries are staged, so `posts` may go out of scope before the
        // copy runs
        SB_CUDA(cudaMemcpyAsync(d_post, posts.data(), sizeof(PcmPost) * j.B, cudaMemcpyHostToDevice, st));
        launch_pcm(j.d_wav, j.d_osegs, d_post, (int)j.B, hop, mx, d_max, fmt, d_pcm, st);
    }
    ~JobPcm() {
        cudaFreeAsync(d_pcm, st);
        cudaFreeAsync(d_max, st);
        cudaFreeAsync(d_post, st);
    }
};

void job_pcm_to_host(Job& j, int fmt, const float* gains, void* dst) {
    JobPcm pcm(j, fmt, gains);
    cudaError_t e = cudaMemcpyAsync(dst, pcm.d_pcm, (size_t)j.out_total * pcm_bytes(fmt), cudaMemcpyDeviceToHost, pcm.st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(pcm.st);
    if (e != cudaSuccess) throw Error(19, std::string("CUDA error: ") + cudaGetErrorString(e));
}

// gains[0 .. B), each finite, or 1 for every utterance when null.
std::vector<float> job_gains(const Job& j, const float* gains) {
    std::vector<float> g(j.B, 1.f);
    for (size_t b = 0; gains && b < j.B; b++) {
        if (!std::isfinite(gains[b]))
            throw Error(19, "utterance " + std::to_string(b) + ": gain " + std::to_string(gains[b]) + " is not finite");
        g[b] = gains[b];
    }
    return g;
}
}  // namespace

void job_i16_to_host(Job& j, float gain, int16_t* dst) {
    const std::vector<float> gains(j.B, gain);
    job_pcm_to_host(j, PCM_I16, gains.data(), dst);
}

int g711_format(long long law, const std::string& who) {
    if (law != G711_MULAW && law != G711_ALAW)
        throw Error(19, who + "G.711 law " + std::to_string(law) + " is neither 0 (mu-law) nor 1 (A-law)");
    return law == G711_MULAW ? PCM_MULAW : PCM_ALAW;
}

void job_g711_to_host(Job& j, int law, const float* gains, uint8_t* dst) {
    const int fmt = g711_format(law, "");
    const std::vector<float> g = job_gains(j, gains);
    job_pcm_to_host(j, fmt, g.data(), dst);
}

void job_flac_to_host(Job& j, const float* gains, uint8_t** outs, size_t* lens) {
    const std::vector<float> g = job_gains(j, gains);
    if (!j.ran || j.encode_only) throw Error(19, "job has not produced audio");
    for (size_t b = 0; b < j.B; b++)
        if (!flac_rate_supported(j.osr[b]))
            throw Error(19, "utterance " + std::to_string(b) + ": FLAC: sample rate " + std::to_string(j.osr[b]) +
                                " Hz is not one of the output rates");
    JobPcm pcm(j, PCM_I16, g.data());
    std::vector<FlacStream> streams(j.B);
    for (size_t b = 0; b < j.B; b++)
        streams[b] = FlacStream{j.osegs[b].out_off, (long long)j.osegs[b].len * j.out_hop, j.osr[b]};
    flac_encode(static_cast<const short*>(pcm.d_pcm), streams, pcm.st, outs, lens);
}

// Peak-normalised 16-bit PCM of every utterance of a finished job, through the context's page-locked staging buffer.
void job_pcm16(Job& j, float gain, std::vector<std::vector<int16_t>>& out) {
    Context& C = *j.ctx;
    SB_CUDA(cudaSetDevice(j.v->device));
    C.pin.reserve((size_t)j.out_total * 2);
    int16_t* h = C.pin.get<int16_t>((size_t)j.out_total);
    job_i16_to_host(j, gain, h);
    out.resize(j.B);
    for (size_t b = 0; b < j.B; b++)
        out[b].assign(h + j.osegs[b].out_off, h + j.osegs[b].out_off + (size_t)j.osegs[b].len * j.out_hop);
}

}  // namespace sb200
