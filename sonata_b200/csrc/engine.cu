// The batched phoneme-id -> waveform pass: packs B utterances into row segments, launches the
// kernel sequence of the Piper graph (SURVEY Appendix A; oracle/vits_oracle.py is the op-by-op
// restatement) and returns per-utterance waveforms.  Replaces VitsModel::infer_with_values +
// the `session.run` it wraps (piper/src/lib.rs:342-399); `speak_batch`'s sequential B=1 loop
// (:433-435) becomes ONE pass whose per-utterance results equal the B=1 results.
#include "engine.h"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <cstdlib>

namespace sb200 {

void throw_launch_error(const char* what) { throw Error(19, std::string("internal: ") + what); }

void check_launch(const char* what) {
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw Error(19, std::string("CUDA launch failed (") + what + "): " + cudaGetErrorString(e));
}


namespace {
constexpr int GX = 64;     // X-level granule (ids)
constexpr int HX = 16;     // min zero rows between X segments (DDSConv dilation 9 + margin)
constexpr int GY = 128;    // Y-level granule (frames)
constexpr int HY = 8;      // min zero frames between Y segments (>= decoder halo / 8)
inline int round_up(int x, int m) { return (x + m - 1) / m * m; }
}  // namespace

// ------------------------------------------------------------------ Context
void Context::ensure_dev(size_t bytes) {
    if (bytes <= dev.cap) return;
    if (dev.base) SB_CUDA(cudaFree(dev.base));
    dev.base = nullptr; dev.cap = 0;
    const size_t want = bytes + bytes / 8 + (64u << 20);
    void* p = nullptr;
    SB_CUDA(cudaMalloc(&p, want));
    dev.base = (char*)p; dev.cap = want;
}
void Context::ensure_pin(size_t bytes) {
    if (bytes <= pin_cap) return;
    if (pin) cudaFreeHost(pin);
    pin = nullptr; pin_cap = 0;
    void* p = nullptr;
    SB_CUDA(cudaMallocHost(&p, bytes * 2));
    pin = (char*)p; pin_cap = bytes * 2;
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
    if (dev.base) cudaFree(dev.base);
    if (pin) cudaFreeHost(pin);
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
    {
        std::shared_lock<std::shared_mutex> g(v->cfg_mu);   // read lock, like piper/src/lib.rs:343
        j->cfg = v->cfg;
    }
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
                        s.a_col0 = h * D; s.b_row0 = off + nt * ks; s.b_col0 = H + h * D; s.nkb = D / 32;
                        j->tiles_s.push_back(s);
                    }
                    // P.V: K runs over the utterance's keys in blocks of 32 (the softmax zero-fills up to the block end)
                    for (int c0 = 0; c0 < D; c0 += ko) {               // one tile per ko head-dim columns
                        TfTile o = t;
                        for (int m = 0; m < 2; m++) {
                            o.a_row0[m] = h * j->RX + off + (mp * 2 + m) * 128;
                            o.out_off[m] = (long long)(off + (mp * 2 + m) * 128) * H + (long long)h * D + c0;
                        }
                        o.a_col0 = 0; o.b_row0 = h * D + c0; o.b_col0 = off; o.nkb = (T + 31) / 32;
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

namespace {

struct Runner {
    Job& j; Voice& v; Context& c; const Arch& a; cudaStream_t st;
    Region* cur = nullptr;
    Runner(Job& job) : j(job), v(*job.v), c(*job.ctx), a(job.v->a), st(job.ctx->stream) {}

    void begin(const std::string& name) {
        j.regions.emplace_back();
        cur = &j.regions.back();
        cur->name = name;
        cur->e0 = c.next_event(); cur->e1 = c.next_event();
        cudaEventRecord(cur->e0, st);
    }
    void end() { cudaEventRecord(cur->e1, st); cur = nullptr; }
    void count(double flops, double bytes, int launches = 1) {
        if (cur) { cur->flops += flops; cur->bytes += bytes; cur->launches += launches; }
    }

    // generic conv launch
    struct Opt {
        float in_slope = 1.f; int act = ACT_NONE; float scale = 1.f;
        const float* res = nullptr; int ldres = 0;
        float* y0 = nullptr; int ldy0 = 0; int acc0 = 0; int split = -1;
        float* y1 = nullptr; int ldy1 = 0; int acc1 = 0;
        int orow_mul = 1, orow_add = 0;
        bool tc_ok = false;
        bool tf_ok = false;    // duration-critical layer: wgmma 3xTF32 with chunk-flushed accumulation (conv_tf.cu)
        float* yt = nullptr; int yt_col0 = 0, ldyt = 0;     // conv_tf only: column tiles >= yt_col0 stored transposed
    };
    // bias of a conv: the voice's, or this call's speaker-conditioned one (multi-speaker voices)
    const float* bias_of(const ConvW& w) const { return (j.d_cond && w.cond_off >= 0) ? j.d_cond + w.cond_off : w.bias; }
    void conv(const ConvW& w, const float* x, int ldx, const Level& lin, const Opt& o) {
        ConvArgs p{};
        p.x = x; p.ldx = ldx; p.rows_in = lin.map.rows; p.cin = w.cin; p.in_slope = o.in_slope;
        p.w = w.w; p.bias = bias_of(w); p.ldw = w.ldw; p.cout = w.cout; p.wtc = w.wtc; p.tc_nt = w.tc_nt; p.wtf = w.wtf;
        p.ntaps = w.ntaps; memcpy(p.tap_off, w.tap_off, sizeof(p.tap_off)); p.min_off = w.min_off; p.span = w.span;
        p.rows_q = lin.map.rows; p.orow_mul = o.orow_mul; p.orow_add = o.orow_add;
        p.map = lin.map;
        p.act = o.act; p.scale = o.scale; p.res = o.res; p.ldres = o.ldres;
        p.y0 = o.y0; p.ldy0 = o.ldy0; p.acc0 = o.acc0; p.split = o.split < 0 ? w.cout : o.split;
        p.y1 = o.y1; p.ldy1 = o.ldy1; p.acc1 = o.acc1;
        p.yt = o.yt; p.yt_col0 = o.yt_col0; p.ldyt = o.ldyt;

        // backend 1 (default): wgmma everywhere; 2: wgmma flow / decoder, fp32 CUDA cores for the text encoder and
        // the duration predictor (the round-1 configuration, kept for A/B runs); 0: fp32 CUDA cores everywhere
        // (each try_launch plans once and returns false without launching when the shape is not supported)
        if (v.backend == 1 && o.tf_ok && try_launch_conv_tf(p, st)) {}
        else if (o.yt) throw Error(19, "internal: a transposed conv output needs the conv_tf kernel");
        else if (v.backend >= 1 && o.tc_ok && try_launch_conv_tc(p, st)) {}
        else launch_conv_simt(p, st);
        const double vr = (double)lin.valid_rows;
        const int cout_w = (o.act == ACT_GATE) ? w.cout / 2 : w.cout;
        count(2.0 * vr * w.cin * w.cout * w.ntaps,
              4.0 * (vr * (w.cin + cout_w + ((o.res && o.res != x) ? w.cout : 0) + ((o.acc0 | o.acc1) ? w.cout : 0)) +
                     (double)w.ntaps * w.cin * w.cout));
    }

    void dds(const DDSW& d, float* x, float* t1, float* t2, const Level& L) {
        const int C = a.hidden;
        int dil = 1;
        for (int i = 0; i < 3; i++) {
            launch_dw_ln_gelu(x, d.wdw[i], d.bdw[i], a.dp_kernel, dil, d.g1[i], d.b1[i], t1, C, L.map, st);
            count(2.0 * L.valid_rows * C * a.dp_kernel, 8.0 * L.valid_rows * C);
            Opt o; o.y0 = t2; o.ldy0 = C; o.tf_ok = true;
            conv(d.c1x1[i], t1, C, L, o);
            launch_ln(t2, nullptr, x, d.g2[i], d.b2[i], x, C, 1, L.map, st);
            count(0, 12.0 * L.valid_rows * C);
            dil *= a.dp_kernel;
        }
    }
};

void h2d(void* dst, const void* src, size_t bytes, cudaStream_t st) {
    SB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st));
}

// decoder over an already-laid-out Y level: s [RY][inter] (gap rows zero) -> wav
void run_decoder(Runner& R, const Level& LY, const float* s, float* d_wav, const FrameSeg* d_fsegs,
                 const int* d_ftile, const int* d_yend) {
    Voice& v = R.v; const Arch& a = R.a; Job& j = R.j; Context& c = R.c;
    const int RY = LY.map.rows;
    R.begin("dec.pre");
    float* p0 = c.dev.get<float>((size_t)RY * a.up_init);
    { Runner::Opt o; o.y0 = p0; o.ldy0 = a.up_init; o.tc_ok = true; R.conv(v.conv_pre, s, a.inter, LY, o); }
    R.end();
    if (j.debug) { j.dbg["dec.pre"] = {p0, a.up_init}; j.dbg_level["dec.pre"] = 1; }

    // ping-pong stage buffers (debug: one set per stage so every stage can be fetched)
    size_t max_elems = 0;
    { int U = 1; for (auto& st : v.ups) { U *= st.u; max_elems = std::max(max_elems, (size_t)RY * U * st.cout); } }
    const int ntmp = (a.resblock == 2) ? 2 : 4;
    float* pool[6] = {nullptr};
    if (!j.debug) for (int i = 0; i < 2 + ntmp; i++) pool[i] = c.dev.get<float>(max_elems);

    const float* cur = p0; Level Lin = LY; int U = 1;
    for (size_t i = 0; i < v.ups.size(); i++) {
        const UpStageW& st = v.ups[i];
        const int Uo = U * st.u;
        Level Lo; Lo.map = {d_yend, GY * Uo, Uo, RY * Uo}; Lo.valid_rows = LY.valid_rows * Uo;
        const size_t elems = (size_t)RY * Uo * st.cout;
        float *up, *ys, *tmp[3];
        if (j.debug) {
            up = c.dev.get<float>(elems); ys = c.dev.get<float>(elems);
            for (int t = 0; t < 3; t++) tmp[t] = c.dev.get<float>(elems);
        } else {
            ys = pool[i & 1]; up = pool[2];
            tmp[0] = pool[3]; tmp[1] = ntmp > 2 ? pool[4] : nullptr; tmp[2] = ntmp > 2 ? pool[5] : nullptr;
        }
        R.begin("dec.up" + std::to_string(i));
        bool fused_done = false;
        if (v.backend >= 1 && st.fused.wtc) {
            // tensor-core path: all u phases in one launch (input read once, N = u*cout columns)
            ConvArgs pa{};
            pa.x = cur; pa.ldx = st.cin; pa.rows_in = Lin.map.rows; pa.cin = st.cin; pa.in_slope = 0.1f;
            pa.w = nullptr; pa.bias = st.fused.bias; pa.ldw = st.fused.ldw; pa.cout = st.fused.cout;
            pa.wtc = st.fused.wtc; pa.tc_nt = st.fused.tc_nt;
            pa.ntaps = st.fused.ntaps; memcpy(pa.tap_off, st.fused.tap_off, sizeof(pa.tap_off));
            pa.min_off = st.fused.min_off; pa.span = st.fused.span;
            pa.rows_q = Lin.map.rows; pa.orow_mul = st.u; pa.orow_add = 0; pa.phase_cols = st.cout;
            pa.map = Lin.map; pa.act = ACT_NONE; pa.scale = 1.f;
            pa.y0 = up; pa.ldy0 = st.cout; pa.split = st.fused.cout; pa.y1 = up; pa.ldy1 = st.cout;
            if (try_launch_conv_tc(pa, R.st)) {
                const double vr = (double)Lin.valid_rows;
                R.count(2.0 * vr * st.cin * st.cout * st.k, 4.0 * (vr * (st.cin + (double)st.u * st.cout) + (double)st.cin * st.cout * st.k));
                fused_done = true;
            }
        }
        for (int p = 0; p < st.u && !fused_done; p++) {
            Runner::Opt o; o.in_slope = 0.1f; o.y0 = up; o.ldy0 = st.cout; o.orow_mul = st.u; o.orow_add = p; o.tc_ok = true;
            R.conv(st.phase[p], cur, st.cin, Lin, o);
        }
        R.end();
        R.begin("dec.mrf" + std::to_string(i));
        const float third = 1.0f / (float)st.res.size();
        for (size_t jb = 0; jb < st.res.size(); jb++) {
            const ResBW& rb = st.res[jb];
            const float* xb = up;
            const size_t nd = rb.dils.size();
            for (size_t m = 0; m < nd; m++) {
                const bool last = (m + 1 == nd);
                const float* cin_ptr = xb;
                if (a.resblock != 2) {
                    Runner::Opt o1; o1.in_slope = 0.1f; o1.y0 = tmp[0]; o1.ldy0 = st.cout; o1.tc_ok = true;
                    R.conv(rb.c1[m], xb, st.cout, Lo, o1);
                    cin_ptr = tmp[0];
                }
                Runner::Opt o; o.in_slope = 0.1f; o.res = xb; o.ldres = st.cout; o.tc_ok = true;
                float* dst;
                if (last) { dst = ys; o.scale = third; o.acc0 = jb > 0 ? 1 : 0; }
                else dst = (a.resblock == 2) ? tmp[0] : tmp[1 + (m & 1)];
                o.y0 = dst; o.ldy0 = st.cout;
                R.conv(a.resblock == 2 ? rb.c1[m] : rb.c2[m], cin_ptr, st.cout, Lo, o);
                xb = dst;
            }
        }
        R.end();
        if (j.debug) {
            j.dbg["dec.up" + std::to_string(i)] = {up, st.cout}; j.dbg_level["dec.up" + std::to_string(i)] = Uo;
            j.dbg["dec.mrf" + std::to_string(i)] = {ys, st.cout}; j.dbg_level["dec.mrf" + std::to_string(i)] = Uo;
        }
        cur = ys; Lin = Lo; U = Uo;
    }
    R.begin("dec.post");
    launch_conv_post(cur, v.c_last, v.conv_post_w, d_wav, d_fsegs, d_ftile, U, Lin.map, R.st);
    R.count(2.0 * Lin.valid_rows * v.c_last * 7, 4.0 * Lin.valid_rows * (v.c_last + 1));
    R.end();
}

// Build the Y-level tables for given per-utterance frame counts; uploads them; returns the level.
Level build_y_layout(Job& j, Context& c, cudaStream_t st, const std::vector<int>& y_len, int hop) {
    const size_t B = y_len.size();
    j.fsegs.resize(B);
    int cur = 0; long long out = 0;
    for (size_t b = 0; b < B; b++) {
        FrameSeg& f = j.fsegs[b];
        f.off = cur; f.len = y_len[b];
        f.xoff = b < j.xsegs.size() ? j.xsegs[b].off : 0;
        f.xlen = b < j.xsegs.size() ? j.xsegs[b].len : 0;
        f.out_off = out;
        out += (long long)y_len[b] * hop;
        cur += round_up(y_len[b] + HY, GY);
    }
    j.RY = cur; j.total_samples = out;
    const int ntile = j.RY / GY;
    std::vector<int> yend(ntile, 0), ftile(ntile, 0);
    for (size_t b = 0; b < B; b++) {
        const int t0 = j.fsegs[b].off / GY;
        const int t1 = (b + 1 < B ? j.fsegs[b + 1].off : j.RY) / GY;
        for (int t = t0; t < t1; t++) { yend[t] = j.fsegs[b].off + j.fsegs[b].len; ftile[t] = (int)b; }
    }
    j.d_yend = c.dev.get<int>(ntile);
    j.d_ftile = c.dev.get<int>(ntile);
    j.d_fsegs = c.dev.get<FrameSeg>(B);
    const size_t need = 2 * ntile * sizeof(int) + B * sizeof(FrameSeg);
    // staging lives in the second half of the pinned buffer (the first half holds the X tables)
    char* pin = c.pin + c.pin_cap / 2;
    if (need > c.pin_cap / 2) throw Error(19, "internal: pinned staging too small");
    memcpy(pin, yend.data(), ntile * sizeof(int));
    memcpy(pin + ntile * sizeof(int), ftile.data(), ntile * sizeof(int));
    memcpy(pin + 2 * ntile * sizeof(int), j.fsegs.data(), B * sizeof(FrameSeg));
    h2d(j.d_yend, pin, ntile * sizeof(int), st);
    h2d(j.d_ftile, pin + ntile * sizeof(int), ntile * sizeof(int), st);
    h2d(j.d_fsegs, pin + 2 * ntile * sizeof(int), B * sizeof(FrameSeg), st);
    Level L; L.map = {j.d_yend, GY, 1, j.RY};
    L.valid_rows = 0; for (int y : y_len) L.valid_rows += y;
    return L;
}

size_t decoder_bytes(const Voice& v, int RY, bool debug) {
    const Arch& a = v.a;
    size_t tot = (size_t)RY * a.up_init * 4 + 4096;
    size_t max_elems = 0, sum = 0; int U = 1;
    for (auto& st : v.ups) { U *= st.u; const size_t e = (size_t)RY * U * st.cout; max_elems = std::max(max_elems, e); sum += e; }
    tot += debug ? sum * 5 * 4 : max_elems * 6 * 4;
    return tot + (1 << 20);
}

}  // namespace

void Job::run(float* d_out, size_t d_out_cap) {
    Voice& V = *v; Context& C = *ctx; const Arch& a = V.a;
    SB_CUDA(cudaSetDevice(V.device));
    cudaStream_t st = C.stream;
    const int H = a.hidden, I = a.inter, F = a.filter;
    regions.clear(); dbg.clear(); dbg_level.clear();
    C.events_used = 0;
    if (!C.ev_begin) { SB_CUDA(cudaEventCreate(&C.ev_begin)); SB_CUDA(cudaEventCreate(&C.ev_end)); }

    // ---------------- phase 1 workspace ----------------
    // tensor-core attention (two grouped GEMMs around a softmax): default backend, 96-wide heads, rows that fit the
    // softmax kernel's registers; otherwise the fp32 CUDA-core attention kernel
    const bool tc_att = V.backend == 1 && H / a.heads == 96 && max_tx <= 1280 && getenv("SB200_ATT_SIMT") == nullptr;
    // xa xb qkv(3H) att d0 t1 t2 g = 10 H; ffn; stats; h29 32; zz 2 + eps_w 2; logw 1; + attention scratch (scores for
    // every head, V^T, relative-value term)
    const size_t xfloats = (size_t)RX * (H * 10 + F + 2 * I + 32 + 2 + 2 + 1) +
                           (tc_att ? (size_t)a.heads * RX * att_tp + 2 * (size_t)RX * H : 0);
    const size_t tile_bytes = (tiles_s.size() + tiles_o.size()) * sizeof(TfTile);
    const size_t p1_bytes = xfloats * 4 + (size_t)RX * 20 + B * 64 + tile_bytes + (1 << 20) + (size_t)V.cond_rows * 4 + 1024 +
                            (debug ? (size_t)RX * (5 * H + att_tp) * 4 + 4096 +
                                     V.dp_flows.size() * ((size_t)RX * (H + 36) * 4 + 1024) : 0);
    // The arena must also hold phase 2; sizes are only known after the durations come back, so phase 1
    // runs in the front of the arena and phase 2 re-plans behind it (growing = realloc would lose phase-1
    // results, so grow conservatively up front from the mean-duration estimate, then verify).
    const double est_frames = 4.0 * (double)ids.size() + 256.0 * B;
    size_t est_p2 = decoder_bytes(V, (int)std::min<double>(est_frames, 2.0e9 / 256), debug) + (size_t)(est_frames * I * 4 * 6);
    C.ensure_dev(p1_bytes + est_p2);
    C.ensure_pin(std::max<size_t>((size_t)RX * 12 + B * 64 + tile_bytes + (1 << 16), 1 << 20));
    C.dev.used = 0; C.dev.dry = false;
    Runner R(*this);

    SB_CUDA(cudaEventRecord(C.ev_begin, st));
    // tables
    const int nxg = RX / GX;
    std::vector<int> xend(nxg, 0), xseg_of(nxg, 0);
    int* ids_rows_h = reinterpret_cast<int*>(C.pin);
    for (int r = 0; r < RX; r++) ids_rows_h[r] = -1;
    for (size_t b = 0; b < B; b++) {
        const SegInfo& s = xsegs[b];
        for (int i = 0; i < s.len; i++) ids_rows_h[s.off + i] = (int)ids[offs[b] + i];
        const int g0 = s.off / GX, g1 = (b + 1 < B ? xsegs[b + 1].off : RX) / GX;
        for (int g = g0; g < g1; g++) { xend[g] = s.off + s.len; xseg_of[g] = (int)b; }
    }
    int* xend_h = ids_rows_h + RX;
    memcpy(xend_h, xend.data(), nxg * sizeof(int));
    int* xseg_of_h = xend_h + nxg;
    memcpy(xseg_of_h, xseg_of.data(), nxg * sizeof(int));
    SegInfo* xsegs_h = reinterpret_cast<SegInfo*>(xseg_of_h + nxg);
    memcpy(xsegs_h, xsegs.data(), B * sizeof(SegInfo));
    // result slot of the frame counts, then (8-byte aligned) the attention tile tables
    const size_t ylen_off = ((size_t)RX * 4 + (size_t)nxg * 8 + B * sizeof(SegInfo) + 63) & ~(size_t)63;
    const size_t tiles_off = (ylen_off + B * sizeof(int) + 63) & ~(size_t)63;
    TfTile* tiles_h = reinterpret_cast<TfTile*>(C.pin + tiles_off);
    d_ids_rows = C.dev.get<int>(RX); d_xend = C.dev.get<int>(nxg); d_xseg_of_gran = C.dev.get<int>(nxg); d_xsegs = C.dev.get<SegInfo>(B);
    d_cum = C.dev.get<int>(RX); d_ylen = C.dev.get<int>(B);
    h2d(d_ids_rows, ids_rows_h, (size_t)RX * 4, st);
    h2d(d_xend, xend_h, (size_t)nxg * 4, st);
    h2d(d_xseg_of_gran, xseg_of_h, (size_t)nxg * 4, st);
    h2d(d_xsegs, xsegs_h, B * sizeof(SegInfo), st);
    d_tiles_s = d_tiles_o = nullptr;
    if (tc_att) {
        memcpy(tiles_h, tiles_s.data(), tiles_s.size() * sizeof(TfTile));
        memcpy(tiles_h + tiles_s.size(), tiles_o.data(), tiles_o.size() * sizeof(TfTile));
        d_tiles_s = C.dev.get<TfTile>(tiles_s.size() + tiles_o.size());
        d_tiles_o = d_tiles_s + tiles_s.size();
        h2d(d_tiles_s, tiles_h, tile_bytes, st);
    }

    Level LX; LX.map = {d_xend, GX, 1, RX}; LX.valid_rows = (long long)ids.size();
    float* xa = C.dev.get<float>((size_t)RX * H);
    float* xb = C.dev.get<float>((size_t)RX * H);
    float* qkv = C.dev.get<float>((size_t)RX * 3 * H);
    float* att = C.dev.get<float>((size_t)RX * H);
    float* ffn = C.dev.get<float>((size_t)RX * F);
    float* stats = C.dev.get<float>((size_t)RX * 2 * I);
    float* d0 = C.dev.get<float>((size_t)RX * H);
    float* t1 = C.dev.get<float>((size_t)RX * H);
    float* t2 = C.dev.get<float>((size_t)RX * H);
    float* g = C.dev.get<float>((size_t)RX * H);
    float* h29 = C.dev.get<float>((size_t)RX * 32);
    float* zz = C.dev.get<float>((size_t)RX * 2);
    float* logw = C.dev.get<float>((size_t)RX);
    float *att_s = nullptr, *att_vt = nullptr, *att_orel = nullptr;
    TfGemm gs{}, go{};
    bool tc_att_ok = tc_att;
    if (tc_att) {
        att_s = C.dev.get<float>((size_t)a.heads * RX * att_tp);
        att_vt = C.dev.get<float>((size_t)H * RX);
        att_orel = C.dev.get<float>((size_t)RX * H);
        gs.a = qkv; gs.a_rows = RX; gs.a_cols = 3 * H; gs.lda = 3 * H;
        gs.b = qkv; gs.b_rows = RX; gs.b_cols = 3 * H; gs.ldb = 3 * H;
        gs.nth = att_nth_s; gs.y = att_s; gs.ldy = att_tp; gs.res = nullptr; gs.scale = 1.0f / sqrtf((float)(H / a.heads));
        gs.tiles = d_tiles_s; gs.ntiles = (int)tiles_s.size();
        go.a = att_s; go.a_rows = a.heads * RX; go.a_cols = att_tp; go.lda = att_tp;
        go.b = att_vt; go.b_rows = H; go.b_cols = RX; go.ldb = RX;
        go.nth = att_nth_o; go.y = att; go.ldy = H; go.res = att_orel; go.scale = 1.f;
        go.tiles = d_tiles_o; go.ntiles = (int)tiles_o.size();
        tc_att_ok = gemm_tf_supported(gs) && gemm_tf_supported(go);
    }
    d_epsw = nullptr;
    if (cfg.noise_w != 0.f) {
        d_epsw = C.dev.get<float>((size_t)RX * 2);
        if (!eps_w.empty()) {
            std::vector<float> stage((size_t)RX * 2, 0.f);
            for (size_t b = 0; b < B; b++)
                if (!eps_w[b].empty()) memcpy(stage.data() + (size_t)xsegs[b].off * 2, eps_w[b].data(), eps_w[b].size() * 4);
            SB_CUDA(cudaMemcpyAsync(d_epsw, stage.data(), stage.size() * 4, cudaMemcpyHostToDevice, st));
            SB_CUDA(cudaStreamSynchronize(st));   // `stage` is pageable; injection is a test-only path
        } else {
            launch_randn(d_epsw, (long long)RX * 2, V.noise_seed, 2 * noise_call, st);
        }
    }

    // ---------------- speaker conditioning (multi-speaker voices) ----------------
    d_cond = nullptr;
    if (V.num_speakers > 1) {
        const long long sid = cfg.has_speaker ? cfg.speaker : 0;      // piper/src/lib.rs:353-358: speaker.unwrap_or(0)
        if (sid < 0 || sid >= V.emb_rows) throw Error(19, "Failed to run model inference. Error: speaker id out of range");
        d_cond = C.dev.get<float>((size_t)V.cond_rows);
        launch_cond_bias(V.cond_w, V.cond_base, V.emb_g + (size_t)sid * V.gin, V.cond_rows, V.gin, d_cond, st);
    }

    // ---------------- text encoder ----------------
    // Every contraction here reaches the duration predictor, and ceil(duration) is a cliff: the dense layers and the two
    // attention contractions run on conv_tf.cu (wgmma, error-compensated tf32, chunk-flushed accumulation: fp32-class
    // accuracy, DESIGN.md section 4); backend 0 / 2 keep them on the fp32 CUDA-core kernels.
    R.begin("enc");
    launch_embed(d_ids_rows, V.emb, sqrtf((float)H), xa, RX, H, st);
    R.count(0, 4.0 * LX.valid_rows * H);
    for (int l = 0; l < a.layers; l++) {
        const EncLayer& e = V.enc[l];
        {
            Runner::Opt o; o.y0 = qkv; o.ldy0 = 3 * H; o.tf_ok = true;
            if (tc_att_ok) { o.yt = att_vt; o.yt_col0 = 2 * H; o.ldyt = RX; }       // V leaves transposed: [H][RX]
            R.conv(e.qkv, xa, H, LX, o);
        }
        if (tc_att_ok) {
            launch_gemm_tf(gs, st);
            launch_attn_softmax(att_s, att_tp, qkv, 3 * H, e.relk, e.relv, a.window, att_orel, H, H, a.heads, RX, d_xsegs,
                                d_xseg_of_gran, GX, max_tx, st);
            launch_gemm_tf(go, st);
            R.count(0, 0, 2);
        } else {
            launch_attention(qkv, 3 * H, e.relk, e.relv, a.window, att, H, H, a.heads, d_xsegs, (int)B, max_tx, st);
        }
        { double f = 0; for (auto& s : xsegs) f += 4.0 * (double)s.len * s.len * H; R.count(f, 16.0 * LX.valid_rows * H); }
        if (debug && l == 0) {      // first-layer attention operands / result (tests/test_gpu_parity.py)
            float* qk = C.dev.get<float>((size_t)RX * 3 * H);
            float* at = C.dev.get<float>((size_t)RX * H);
            SB_CUDA(cudaMemcpyAsync(qk, qkv, (size_t)RX * 3 * H * 4, cudaMemcpyDeviceToDevice, st));
            SB_CUDA(cudaMemcpyAsync(at, att, (size_t)RX * H * 4, cudaMemcpyDeviceToDevice, st));
            dbg["qkv0"] = {qk, 3 * H}; dbg_level["qkv0"] = 0; dbg["att0"] = {at, H}; dbg_level["att0"] = 0;
            if (tc_att_ok) {
                float* sp = C.dev.get<float>((size_t)RX * att_tp);
                SB_CUDA(cudaMemcpyAsync(sp, att_s, (size_t)RX * att_tp * 4, cudaMemcpyDeviceToDevice, st));
                dbg["p0"] = {sp, att_tp}; dbg_level["p0"] = 0;     // head 0 probabilities
                // V went only to att_vt (the V columns of qkv0 are not written on this path): captured as [H][RX]
                float* vt = C.dev.get<float>((size_t)H * RX);
                SB_CUDA(cudaMemcpyAsync(vt, att_vt, (size_t)H * RX * 4, cudaMemcpyDeviceToDevice, st));
                dbg["vt0"] = {vt, H}; dbg_level["vt0"] = -1;
            }
        }
        { Runner::Opt o; o.y0 = xb; o.ldy0 = H; o.tf_ok = true; R.conv(e.o, att, H, LX, o); }
        launch_ln(xa, xb, nullptr, e.g1, e.b1, xa, H, 0, LX.map, st);
        R.count(0, 12.0 * LX.valid_rows * H);
        { Runner::Opt o; o.act = ACT_RELU; o.y0 = ffn; o.ldy0 = F; o.tf_ok = true; R.conv(e.ffn1, xa, H, LX, o); }
        { Runner::Opt o; o.y0 = xb; o.ldy0 = H; o.tf_ok = true; R.conv(e.ffn2, ffn, F, LX, o); }
        launch_ln(xa, xb, nullptr, e.g2, e.b2, xa, H, 0, LX.map, st);
        R.count(0, 12.0 * LX.valid_rows * H);
    }
    { Runner::Opt o; o.y0 = stats; o.ldy0 = 2 * I; o.tf_ok = true; R.conv(V.enc_proj, xa, H, LX, o); }
    R.end();
    if (debug) { dbg["x"] = {xa, H}; dbg_level["x"] = 0; dbg["stats"] = {stats, 2 * I}; dbg_level["stats"] = 0; }

    // ---------------- stochastic duration predictor (reverse) ----------------
    R.begin("dp");
    { Runner::Opt o; o.y0 = d0; o.ldy0 = H; o.tf_ok = true; R.conv(V.dp_pre, xa, H, LX, o); }
    R.dds(V.dp_dds, d0, t1, t2, LX);
    { Runner::Opt o; o.y0 = g; o.ldy0 = H; o.tf_ok = true; R.conv(V.dp_proj, d0, H, LX, o); }
    launch_scale_copy2(d_epsw, cfg.noise_w, zz, LX.map, st);
    if (debug) { dbg["dp.g"] = {g, H}; dbg_level["dp.g"] = 0; }
    // debug: each flow's input, DDSConv output, spline parameters and output (zz, d0 and h29 are reused: copies)
    auto capture = [&](const std::string& name, const float* src, int cols) {
        float* cp = C.dev.get<float>((size_t)RX * cols);
        SB_CUDA(cudaMemcpyAsync(cp, src, (size_t)RX * cols * 4, cudaMemcpyDeviceToDevice, st));
        dbg[name] = {cp, cols}; dbg_level[name] = 0;
    };
    for (size_t s = 0; s < V.dp_flows.size(); s++) {
        const CFlowW& cf = V.dp_flows[s];
        const std::string fs = "dp.f" + std::to_string(s) + ".";
        if (debug) capture(fs + "in", zz, 2);
        launch_flow_pre(zz, cf.ccol, cf.pre_w, cf.pre_b, g, d0, H, LX.map, st);
        R.count(2.0 * LX.valid_rows * H, 8.0 * LX.valid_rows * H);
        R.dds(cf.dds, d0, t1, t2, LX);
        if (debug) capture(fs + "h", d0, H);
        { Runner::Opt o; o.y0 = h29; o.ldy0 = 32; o.tf_ok = true; R.conv(cf.proj, d0, H, LX, o); }
        if (debug) capture(fs + "h29", h29, 32);
        launch_spline(h29, 32, zz, cf.tcol, a.dp_bins, 1.0f / sqrtf((float)H), LX.map, st);
        R.count(0, 4.0 * LX.valid_rows * 34);
        if (debug) capture(fs + "out", zz, 2);
    }
    launch_durations(zz, V.ea_m0, V.ea_logs0, cfg.length_scale, d_xsegs, (int)B, logw, d_cum, d_ylen, st);
    R.end();
    if (debug) { dbg["logw"] = {logw, 1}; dbg_level["logw"] = 0; }

    // ---------------- host learns the frame counts (the graph's data-dependent shape) ----------------
    int* ylen_h = reinterpret_cast<int*>(C.pin + ylen_off);
    SB_CUDA(cudaMemcpyAsync(ylen_h, d_ylen, B * sizeof(int), cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    y_len.assign(ylen_h, ylen_h + B);
    long long tot_frames = 0;
    for (int y : y_len) tot_frames += y;
    if (tot_frames > (long long)(2.0e9 / 256 / 4)) throw Error(19, "Failed to run model inference. Error: predicted durations are unreasonably long");
    if (!eps_z.empty())
        for (size_t b = 0; b < B; b++)
            if (!eps_z[b].empty() && eps_z_frames[b] != (size_t)y_len[b])
                throw Error(19, "injected eps_z has " + std::to_string(eps_z_frames[b]) + " frames but the model produced " + std::to_string(y_len[b]));

    // ---------------- phase 2 workspace (plan, then make sure it fits behind phase 1) ----------------
    {
        int cur = 0;
        for (int y : y_len) cur += round_up(y + HY, GY);
        const size_t need = C.dev.used + decoder_bytes(V, cur, debug) + (size_t)cur * (size_t)(5 * I + 3 * H) * 4 +
                            (size_t)tot_frames * a.hop() * 4 + (8 << 20);
        if (need > C.dev.cap) {
            // grow: allocate a bigger arena and carry the phase-1 results over
            Arena old = C.dev;
            C.dev.base = nullptr; C.dev.cap = 0;
            void* p = nullptr;
            SB_CUDA(cudaMalloc(&p, need + need / 8));
            C.dev.base = (char*)p; C.dev.cap = need + need / 8; C.dev.used = old.used;
            SB_CUDA(cudaMemcpyAsync(C.dev.base, old.base, old.used, cudaMemcpyDeviceToDevice, st));
            SB_CUDA(cudaStreamSynchronize(st));
            const ptrdiff_t delta = C.dev.base - old.base;
            auto mv = [&](auto*& ptr) { if (ptr) ptr = reinterpret_cast<std::remove_reference_t<decltype(ptr)>>(reinterpret_cast<char*>(ptr) + delta); };
            mv(d_ids_rows); mv(d_xend); mv(d_xsegs); mv(d_cum); mv(d_ylen); mv(d_epsw); mv(d_xseg_of_gran); mv(d_tiles_s); mv(d_tiles_o); mv(d_cond);
            mv(xa); mv(stats); mv(logw);
            for (auto& kv : dbg) kv.second.first = reinterpret_cast<float*>(reinterpret_cast<char*>(kv.second.first) + delta);
            SB_CUDA(cudaFree(old.base));
        }
    }
    Level LY = build_y_layout(*this, C, st, y_len, a.hop());

    // ---------------- alignment expansion ----------------
    R.begin("align");
    float* s = C.dev.get<float>((size_t)RY * I);
    d_epsz = nullptr;
    if (cfg.noise_scale != 0.f) {
        d_epsz = C.dev.get<float>((size_t)RY * I);
        if (!eps_z.empty()) {
            std::vector<float> stage((size_t)RY * I, 0.f);
            for (size_t b = 0; b < B; b++)
                if (!eps_z[b].empty()) memcpy(stage.data() + (size_t)fsegs[b].off * I, eps_z[b].data(), eps_z[b].size() * 4);
            SB_CUDA(cudaMemcpyAsync(d_epsz, stage.data(), stage.size() * 4, cudaMemcpyHostToDevice, st));
            SB_CUDA(cudaStreamSynchronize(st));
        } else {
            launch_randn(d_epsz, (long long)RY * I, V.noise_seed, 2 * noise_call + 1, st);
        }
    }
    launch_expand(stats, 2 * I, I, d_cum, d_epsz, cfg.noise_scale, s, d_fsegs, d_ftile, LY.map, st);
    R.count(0, 4.0 * LY.valid_rows * 3 * I);
    R.end();
    float* zp_dbg = nullptr;
    if (debug) {
        zp_dbg = C.dev.get<float>((size_t)RY * I);
        SB_CUDA(cudaMemcpyAsync(zp_dbg, s, (size_t)RY * I * 4, cudaMemcpyDeviceToDevice, st));
        dbg["z_p"] = {zp_dbg, I}; dbg_level["z_p"] = 1;
    }

    // ---------------- residual-coupling flow (reverse) ----------------
    R.begin("flow");
    float* h = C.dev.get<float>((size_t)RY * H);
    float* acts = C.dev.get<float>((size_t)RY * H);
    float* outb = C.dev.get<float>((size_t)RY * H);
    const int half = I / 2;
    for (const CouplingW& cp : V.flows) {
        { Runner::Opt o; o.y0 = h; o.ldy0 = H; o.tc_ok = true; R.conv(cp.pre, s + cp.cond_off, I, LY, o); }
        const int n = (int)cp.in.size();
        for (int l = 0; l < n; l++) {
            { Runner::Opt o; o.act = ACT_GATE; o.y0 = acts; o.ldy0 = H; o.tc_ok = true; R.conv(cp.in[l], h, H, LY, o); }
            Runner::Opt o; o.tc_ok = true;
            if (l < n - 1) { o.y0 = h; o.ldy0 = H; o.acc0 = 1; o.split = H; o.y1 = outb; o.ldy1 = H; o.acc1 = l > 0; }
            else { o.split = 0; o.y0 = outb; o.ldy0 = H; o.y1 = outb; o.ldy1 = H; o.acc1 = l > 0; }
            R.conv(cp.rs[l], acts, H, LY, o);
        }
        { Runner::Opt o; o.y0 = s + cp.tgt_off; o.ldy0 = I; o.acc0 = 1; o.scale = -1.f; o.tc_ok = true; R.conv(cp.post, outb, H, LY, o); }
    }
    (void)half;
    R.end();
    if (debug) { dbg["z"] = {s, I}; dbg_level["z"] = 1; }

    // ---------------- HiFi-GAN ----------------
    if (encode_only) {
        z_dev = s;
        SB_CUDA(cudaEventRecord(C.ev_end, st));
        SB_CUDA(cudaStreamSynchronize(st));
        SB_CUDA(cudaGetLastError());
        SB_CUDA(cudaEventElapsedTime(&last_ms, C.ev_begin, C.ev_end));
        ran = true;
        return;
    }
    if (d_out) {
        if ((size_t)total_samples > d_out_cap) throw Error(19, "caller-provided device output buffer is too small");
        d_wav = d_out; wav_external = true;
    } else {
        d_wav = C.dev.get<float>((size_t)total_samples + 4); wav_external = false;
    }
    run_decoder(R, LY, s, d_wav, d_fsegs, d_ftile, d_yend);
    SB_CUDA(cudaEventRecord(C.ev_end, st));
    SB_CUDA(cudaStreamSynchronize(st));
    SB_CUDA(cudaGetLastError());
    SB_CUDA(cudaEventElapsedTime(&last_ms, C.ev_begin, C.ev_end));
    for (Region& r : regions) cudaEventElapsedTime(&r.ms, r.e0, r.e1);
    ran = true;
}

// ====================================================================== streaming halves
Latent::~Latent() { if (z) { cudaSetDevice(v->device); cudaFree(z); } }

Latent* encode_latent(Voice* v, const long long* ids, size_t n) {
    const size_t offs[2] = {0, n};
    std::unique_ptr<Job> j(create_job(v, ids, offs, 1, nullptr, nullptr, nullptr, false));
    j->encode_only = true;
    j->run(nullptr, 0);
    std::unique_ptr<Latent> L(new Latent());
    L->v = v; L->frames = j->y_len[0];
    L->sid = j->cfg.has_speaker ? j->cfg.speaker : 0;
    const size_t bytes = (size_t)L->frames * v->a.inter * 4;
    SB_CUDA(cudaMalloc(&L->z, bytes));
    const float* src = j->z_dev + (size_t)j->fsegs[0].off * v->a.inter;
    SB_CUDA(cudaMemcpy(L->z, src, bytes, cudaMemcpyDeviceToDevice));
    return L.release();
}

namespace {
// decoder on z[lo:hi) with the result left on the device (job-owned arena): shared by the f32 and the PCM entry points
float* decode_chunk_device(Voice* v, const Latent* z, long long lo, long long hi, Job& j, size_t extra_bytes) {
    if (lo < 0 || hi > z->frames || lo >= hi) throw Error(19, "Invalid model audio output");
    const Arch& a = v->a;
    j.v = v; j.B = 1; j.ctx = v->acquire();
    Context& C = *j.ctx;
    SB_CUDA(cudaSetDevice(v->device));
    const int n = (int)(hi - lo);
    const int RY = round_up(n + HY, GY);
    C.ensure_dev(decoder_bytes(*v, RY, false) + (size_t)RY * a.inter * 4 + (size_t)n * a.hop() * 4 + extra_bytes + (size_t)v->cond_rows * 4 + (4 << 20));
    C.ensure_pin(std::max<size_t>(1 << 20, (size_t)n * a.hop() * 4 + 4096));
    C.dev.used = 0; C.events_used = 0;
    if (!C.ev_begin) { SB_CUDA(cudaEventCreate(&C.ev_begin)); SB_CUDA(cudaEventCreate(&C.ev_end)); }
    cudaStream_t st = C.stream;
    Runner R(j);
    SB_CUDA(cudaEventRecord(C.ev_begin, st));
    if (v->num_speakers > 1) {       // decoder.onnx takes the encoder's `g` (piper/src/lib.rs:706-735, 739-743)
        if (z->sid < 0 || z->sid >= v->emb_rows) throw Error(19, "Failed to run model inference. Error: speaker id out of range");
        j.d_cond = C.dev.get<float>((size_t)v->cond_rows);
        launch_cond_bias(v->cond_w, v->cond_base, v->emb_g + (size_t)z->sid * v->gin, v->cond_rows, v->gin, j.d_cond, st);
    }
    Level LY = build_y_layout(j, C, st, std::vector<int>{n}, a.hop());
    float* s = C.dev.get<float>((size_t)RY * a.inter);
    launch_fill_zero(s, (long long)RY * a.inter, st);
    SB_CUDA(cudaMemcpyAsync(s, z->z + (size_t)lo * a.inter, (size_t)n * a.inter * 4, cudaMemcpyDeviceToDevice, st));
    float* d_wav = C.dev.get<float>((size_t)j.total_samples + 4);
    run_decoder(R, LY, s, d_wav, j.d_fsegs, j.d_ftile, j.d_yend);
    SB_CUDA(cudaEventRecord(C.ev_end, st));
    return d_wav;
}
}  // namespace

void decode_latent_chunk(Voice* v, const Latent* z, long long lo, long long hi, std::vector<float>& out, float* ms) {
    Job j;
    float* d_wav = decode_chunk_device(v, z, lo, hi, j, 0);
    Context& C = *j.ctx;
    cudaStream_t st = C.stream;
    // through the context's page-locked staging buffer: a DMA copy instead of a pageable one
    const size_t bytes = (size_t)j.total_samples * 4;
    SB_CUDA(cudaMemcpyAsync(C.pin, d_wav, bytes, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    SB_CUDA(cudaGetLastError());
    out.resize((size_t)j.total_samples);
    memcpy(out.data(), C.pin, bytes);
    if (ms) cudaEventElapsedTime(ms, C.ev_begin, C.ev_end);
}

// crossfade table of AudioSamples::crossfade (audio/ops/src/samples.rs:144-157) for a buffer of `len` samples
static void fill_fade(PcmPost& p, int fade, long long len) {
    const long long n = std::min<long long>(fade, len / 2);
    p.fade_n = (int)std::min<long long>(n, 48);
    const float att = (float)(p.fade_n - 1);
    for (int i = 0; i < p.fade_n; i++) p.tab[i] = sinf(((float)i / att) * 3.14159265358979f / 2.0f);
}

void decode_latent_chunk_pcm(Voice* v, const Latent* z, long long lo, long long hi, long long trim_lo_frames,
                             long long trim_hi_frames, int fade, float gain, std::vector<int16_t>& out, float* ms) {
    Job j;
    const int hop = v->a.hop();
    const size_t total = (size_t)(hi - lo) * hop;
    float* d_wav = decode_chunk_device(v, z, lo, hi, j, total * 2 + 4096);
    Context& C = *j.ctx;
    cudaStream_t st = C.stream;
    PcmPost post;
    post.gain = gain; post.trim_lo = trim_lo_frames * hop; post.trim_hi = trim_hi_frames * hop;
    const long long m = (long long)total - post.trim_lo - post.trim_hi;
    if (m <= 0) throw Error(19, "Invalid model audio output");
    if (fade > 0) fill_fade(post, fade, m);
    short* d_i16 = C.dev.get<short>(total + 8);
    unsigned* d_max = C.dev.get<unsigned>(4);
    launch_i16(d_wav, j.d_fsegs, 1, hop, (long long)total, d_max, d_i16, post, st);
    SB_CUDA(cudaMemcpyAsync(C.pin, d_i16, (size_t)m * 2, cudaMemcpyDeviceToHost, st));
    SB_CUDA(cudaStreamSynchronize(st));
    SB_CUDA(cudaGetLastError());
    out.resize((size_t)m);
    memcpy(out.data(), C.pin, (size_t)m * 2);
    if (ms) cudaEventElapsedTime(ms, C.ev_begin, C.ev_end);
}

// Peak-normalised 16-bit PCM of every utterance of a finished job (to_i16_vec after the linear gain), converted on the
// device and copied through the context's page-locked staging buffer.
void job_pcm16(Job& j, float gain, std::vector<std::vector<int16_t>>& out) {
    if (!j.ran || j.encode_only) throw Error(19, "job has not produced audio");
    Voice& v = *j.v; Context& C = *j.ctx;
    SB_CUDA(cudaSetDevice(v.device));
    cudaStream_t st = C.stream;
    const int hop = v.a.hop();
    const size_t n = (size_t)j.total_samples;
    long long mx = 0;
    for (size_t b = 0; b < j.B; b++) mx = std::max<long long>(mx, (long long)j.y_len[b] * hop);
    short* d_i16 = nullptr; unsigned* d_max = nullptr;
    SB_CUDA(cudaMallocAsync(&d_i16, n * 2 + 16, st));
    SB_CUDA(cudaMallocAsync(&d_max, sizeof(unsigned) * j.B, st));
    PcmPost post; post.gain = gain;
    launch_i16(j.d_wav, j.d_fsegs, (int)j.B, hop, mx, d_max, d_i16, post, st);
    C.ensure_pin(n * 2 + 4096);                    // the tables staged there were consumed by the pass
    cudaError_t e = cudaMemcpyAsync(C.pin, d_i16, n * 2, cudaMemcpyDeviceToHost, st);
    cudaFreeAsync(d_i16, st);
    cudaFreeAsync(d_max, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) throw Error(19, std::string("CUDA error: ") + cudaGetErrorString(e));
    out.resize(j.B);
    const int16_t* h = reinterpret_cast<const int16_t*>(C.pin);
    for (size_t b = 0; b < j.B; b++)
        out[b].assign(h + j.fsegs[b].out_off, h + j.fsegs[b].out_off + (size_t)j.y_len[b] * hop);
}

}  // namespace sb200
