// Voice loading: Piper `*.onnx.json` config + `.svw` weight table -> device-resident, GEMM-ready
// weights.  Mirrors `sonata_piper::from_config_path` / `load_model_config` / `VitsModel::from_config`
// (piper/src/lib.rs:33-61, 88-110, 306-341); the weight re-layout below is what onnxruntime's
// session initialisation (pre-packing) does on the reference side.
#include "engine.h"
#include "json.hpp"
#include <algorithm>
#include <cstring>
#include <fstream>
#include <sstream>

namespace sb200 {

namespace {

std::string read_file(const std::string& p, bool& ok) {
    std::ifstream f(p, std::ios::binary);
    if (!f) { ok = false; return {}; }
    std::ostringstream ss;
    ss << f.rdbuf();
    ok = true;
    return ss.str();
}

using TensorMap = std::unordered_map<std::string, HostTensor>;

TensorMap parse_svw(const std::string& buf, const std::string& path) {
    TensorMap m;
    if (buf.size() < 12 || memcmp(buf.data(), "SVW1\0\0\0\0", 8) != 0)
        throw Error(17, "Faild to load model weights: `" + path + "` is not an SVW1 file");
    uint32_t count;
    memcpy(&count, buf.data() + 8, 4);
    size_t pos = 12;
    auto need = [&](size_t n) { if (pos + n > buf.size()) throw Error(17, "truncated weight file `" + path + "`"); };
    for (uint32_t t = 0; t < count; t++) {
        need(2);
        uint16_t nl; memcpy(&nl, buf.data() + pos, 2); pos += 2;
        need(nl);
        std::string name(buf.data() + pos, nl); pos += nl;
        need(2);
        uint8_t dt = (uint8_t)buf[pos], nd = (uint8_t)buf[pos + 1]; pos += 2;
        HostTensor ht;
        need(4 * (size_t)nd);
        for (int d = 0; d < nd; d++) { uint32_t v; memcpy(&v, buf.data() + pos, 4); pos += 4; ht.dims.push_back((int)v); }
        pos += (16 - pos % 16) % 16;
        const size_t n = ht.numel();
        need(4 * n);
        if (dt == 0) { ht.f.resize(n); memcpy(ht.f.data(), buf.data() + pos, 4 * n); }
        else { ht.is_int = true; ht.i.resize(n); memcpy(ht.i.data(), buf.data() + pos, 4 * n); }
        pos += 4 * n;
        m.emplace(std::move(name), std::move(ht));
    }
    return m;
}

const HostTensor& T(const TensorMap& m, const std::string& n) {
    auto it = m.find(n);
    if (it == m.end()) throw Error(17, "weight tensor `" + n + "` missing from voice file");
    return it->second;
}

struct Uploader {
    Voice* v;
    float* up(const std::vector<float>& h) {
        float* d = nullptr;
        SB_CUDA(cudaMalloc(&d, h.size() * sizeof(float) + 16));
        SB_CUDA(cudaMemcpy(d, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice));
        v->dev_allocs.push_back(d);
        return d;
    }
};

// Weight images of a conv, one per kernel that reads it: conv_simt.cu, conv_tf.cu, conv_tc.cu.
enum ConvImages { IMG_F32 = 1, IMG_TF32 = 2, IMG_BF16 = 4 };
// text encoder and duration predictor: conv_tf on backend 1, conv_simt on backends 0 and 2
constexpr int ENC_IMAGES = IMG_F32 | IMG_TF32;
// flow and decoder: conv_tc on backends 1 and 2, conv_simt on backend 0
constexpr int DEC_IMAGES = IMG_F32 | IMG_BF16;

// Uploads the bias bt [ldw] and the requested images of weights wt [ntaps][cin][ldw] of a laid-out conv.  A
// tensor-core image is built only for a shape its kernel takes.
void upload_conv(Uploader& U, ConvW& c, const std::vector<float>& wt, const std::vector<float>& bt, int images) {
    if (images & IMG_F32) c.w = U.up(wt);
    c.bias = U.up(bt);
    if (c.cin % 32 || c.cout % 32) return;
    if (images & IMG_TF32) {
        const size_t nf = conv_tf_weight_floats(c.cin, c.cout, c.ntaps);
        if (nf) {
            std::vector<float> img(nf);
            conv_tf_build_weights(wt.data(), c.ldw, c.cin, c.cout, c.ntaps, img.data());
            c.wtf = U.up(img);
        }
    }
    const int nt = tc_tile_for(c.cout);
    if (!(images & IMG_BF16) || !nt) return;
    std::vector<float> img(conv_tc_weight_floats(c.cin, c.cout, c.ntaps, nt));
    conv_tc_build_weights(wt.data(), c.ldw, c.cin, c.cout, c.ntaps, nt, img.data());
    c.wtc = U.up(img);
    c.tc_nt = nt;
}

// Conv1d weight [cout][cin][k] (+bias) -> ConvW with centred taps of dilation `dil` and the given images.
// `perm_out`: output column n takes source row perm_out[n]; `perm_in` likewise for inputs.
ConvW make_conv(Uploader& U, int images, const std::vector<const HostTensor*>& ws,
                const std::vector<const HostTensor*>& bs, int dil, const std::vector<int>* perm_out = nullptr,
                const std::vector<int>* perm_in = nullptr, int pad_cout_to = 0) {
    const int cin = ws[0]->dims[1], k = ws[0]->dims[2];
    int cout = 0;
    for (auto* w : ws) cout += w->dims[0];
    // stack the sources along cout
    std::vector<float> wcat((size_t)cout * cin * k), bcat(cout, 0.f);
    {
        size_t o = 0; int r = 0;
        for (size_t s = 0; s < ws.size(); s++) {
            memcpy(wcat.data() + o, ws[s]->f.data(), ws[s]->f.size() * sizeof(float));
            o += ws[s]->f.size();
            if (!bs.empty() && bs[s]) memcpy(bcat.data() + r, bs[s]->f.data(), bs[s]->f.size() * sizeof(float));
            r += ws[s]->dims[0];
        }
    }
    ConvW c = conv_layout(cin, pad_cout_to ? pad_cout_to : cout, centred_taps(k, dil));
    std::vector<float> wt((size_t)k * cin * c.ldw, 0.f), bt(c.ldw, 0.f);
    for (int n = 0; n < cout; n++) {
        const int sn = perm_out ? (*perm_out)[n] : n;
        bt[n] = bcat[sn];
        for (int ci = 0; ci < cin; ci++) {
            const int sc = perm_in ? (*perm_in)[ci] : ci;
            for (int t = 0; t < k; t++)
                wt[((size_t)t * cin + ci) * c.ldw + n] = wcat[((size_t)sn * cin + sc) * k + t];
        }
    }
    upload_conv(U, c, wt, bt, images);
    return c;
}

ConvW conv_named(Uploader& U, int images, const TensorMap& m, const std::string& name, int dil = 1,
                 bool has_bias = true, const std::vector<int>* perm_out = nullptr,
                 const std::vector<int>* perm_in = nullptr, int pad_cout_to = 0) {
    std::vector<const HostTensor*> bs;
    if (has_bias) bs.push_back(&T(m, name + ".bias")); else bs.push_back(nullptr);
    return make_conv(U, images, {&T(m, name + ".weight")}, bs, dil, perm_out, perm_in, pad_cout_to);
}

// DDSConv of the duration predictor
DDSW load_dds(Uploader& U, const TensorMap& m, const std::string& p, int C, int k) {
    DDSW d;
    for (int i = 0; i < 3; i++) {
        const HostTensor& w = T(m, p + "convs_sep." + std::to_string(i) + ".weight");   // [C][1][k]
        std::vector<float> wt((size_t)k * C);
        for (int c = 0; c < C; c++)
            for (int t = 0; t < k; t++) wt[(size_t)t * C + c] = w.f[(size_t)c * k + t];
        d.wdw[i] = U.up(wt);
        d.bdw[i] = U.up(T(m, p + "convs_sep." + std::to_string(i) + ".bias").f);
        d.c1x1[i] = conv_named(U, ENC_IMAGES, m, p + "convs_1x1." + std::to_string(i));
        d.g1[i] = U.up(T(m, p + "norms_1." + std::to_string(i) + ".gamma").f);
        d.b1[i] = U.up(T(m, p + "norms_1." + std::to_string(i) + ".beta").f);
        d.g2[i] = U.up(T(m, p + "norms_2." + std::to_string(i) + ".gamma").f);
        d.b2[i] = U.up(T(m, p + "norms_2." + std::to_string(i) + ".beta").f);
    }
    return d;
}

// `t` with axis `axis` widened to `width`: source index i lands at `off` + i (reversed: `off` + n-1-i), the rest is zero
HostTensor widen(const HostTensor& t, int width, int axis, int off, bool reversed) {
    HostTensor o;
    o.dims = t.dims;
    const int n = t.dims[axis];
    o.dims[axis] = width;
    size_t outer = 1, inner = 1;
    for (int d = 0; d < axis; d++) outer *= (size_t)t.dims[d];
    for (size_t d = axis + 1; d < t.dims.size(); d++) inner *= (size_t)t.dims[d];
    o.f.assign(outer * width * inner, 0.f);
    for (size_t a = 0; a < outer; a++)
        for (int i = 0; i < n; i++) {
            const int k = off + (reversed ? n - 1 - i : i);
            memcpy(o.f.data() + (a * width + k) * inner, t.f.data() + (a * n + i) * inner, inner * sizeof(float));
        }
    return o;
}

uint32_t first_code_point(const std::string& s) {
    if (s.empty()) return 0;
    const unsigned char c = (unsigned char)s[0];
    if (c < 0x80) return c;
    if ((c >> 5) == 6 && s.size() >= 2) return ((c & 0x1F) << 6) | (s[1] & 0x3F);
    if ((c >> 4) == 14 && s.size() >= 3) return ((c & 0x0F) << 12) | ((s[1] & 0x3F) << 6) | (s[2] & 0x3F);
    if ((c >> 3) == 30 && s.size() >= 4)
        return ((c & 0x07) << 18) | ((s[1] & 0x3F) << 12) | ((s[2] & 0x3F) << 6) | (s[3] & 0x3F);
    return c;
}

}  // namespace

std::vector<int> centred_taps(int k, int dil) {
    std::vector<int> offs(k);
    for (int t = 0; t < k; t++) offs[t] = (t - (k - 1) / 2) * dil;
    return offs;
}

ConvW conv_layout(int cin, int cout, const std::vector<int>& offs, bool pad_ldw) {
    if (offs.empty() || offs.size() > SB_MAX_TAPS) throw Error(17, "unsupported conv kernel size");
    ConvW c;
    c.cin = cin; c.cout = cout; c.ntaps = (int)offs.size();
    c.macs = c.ntaps * cin * cout;
    const int bn = pad_ldw ? conv_simt_bn_for(cout) : 1;
    c.ldw = (cout + bn - 1) / bn * bn;
    std::copy(offs.begin(), offs.end(), c.tap_off);
    c.min_off = *std::min_element(offs.begin(), offs.end());
    c.span = *std::max_element(offs.begin(), offs.end()) - c.min_off;
    return c;
}

int tc_tile_for(int cout) {
    if (cout <= 128) return cout;
    if (cout % 128 == 0) return 128;
    if (cout % 96 == 0) return 96;
    return 0;
}

// test hook: build a ConvW with every kernel's weight images from a raw [cout][cin][k] tensor (tools/conv_unit.py runs
// one conv on each backend)
ConvW debug_make_conv(Voice& v, const float* w, const float* bias, int cout, int cin, int k, int dil) {
    HostTensor hw, hb;
    hw.dims = {cout, cin, k}; hw.f.assign(w, w + (size_t)cout * cin * k);
    hb.dims = {cout}; hb.f.assign(cout, 0.f);
    if (bias) hb.f.assign(bias, bias + cout);
    Uploader U{&v};
    return make_conv(U, IMG_F32 | IMG_TF32 | IMG_BF16, {&hw}, {&hb}, dil);
}

// VitsModelCommons::phonemes_to_input_ids + get_meta_ids (piper/src/lib.rs:173-179, 232-250)
std::vector<long long> Voice::phonemes_to_ids(const char* utf8, std::vector<long long>* src_char) const {
    auto meta = [&](char ch) -> long long {
        auto it = phoneme_first_id.find((uint32_t)ch);
        if (it == phoneme_first_id.end())
            throw Error(19, std::string("phoneme_id_map has no entry for `") + ch + "`");
        return it->second;
    };
    const long long pad = meta('_'), bos = meta('^'), eos = meta('$');
    std::vector<long long> ids;
    ids.push_back(bos);
    if (src_char) src_char->assign(1, -1);
    const unsigned char* s = reinterpret_cast<const unsigned char*>(utf8);
    for (long long ch = 0; *s; ch++) {
        uint32_t cp; int n;
        if (*s < 0x80) { cp = *s; n = 1; }
        else if ((*s >> 5) == 6) { cp = *s & 0x1F; n = 2; }
        else if ((*s >> 4) == 14) { cp = *s & 0x0F; n = 3; }
        else if ((*s >> 3) == 30) { cp = *s & 0x07; n = 4; }
        else throw Error(20, "invalid UTF-8 sequence in phoneme string");
        for (int i = 1; i < n; i++) {
            if ((s[i] & 0xC0) != 0x80) throw Error(20, "invalid UTF-8 sequence in phoneme string");
            cp = (cp << 6) | (s[i] & 0x3F);
        }
        s += n;
        auto it = phoneme_first_id.find(cp);
        if (it != phoneme_first_id.end()) {   // unknown phonemes are dropped silently (:243)
            ids.push_back(it->second);
            ids.push_back(pad);
            if (src_char) { src_char->push_back(ch); src_char->push_back(ch); }
        }
    }
    ids.push_back(eos);
    if (src_char) src_char->push_back(-1);
    return ids;
}

Voice::~Voice() {
    if (device < 0) return;
    cudaSetDevice(device);
    for (Context* c : pool) delete c;
    for (void* p : dev_allocs) cudaFree(p);
}

Voice* load_voice(const std::string& config_path, int device) {
    bool ok;
    const std::string cfg_text = read_file(config_path, ok);
    if (!ok) throw Error(17, "Faild to load model config: `" + config_path + "`. Caused by: `cannot open file`");
    sbjson::ValuePtr root;
    try { root = sbjson::parse(cfg_text); }
    catch (const std::exception& e) {
        throw Error(17, "Faild to parse model config from file: `" + config_path + "`. Caused by: `" + e.what() + "`");
    }
    std::unique_ptr<Voice> v(new Voice());
    v->config_path = config_path;
    v->device = device;
    auto req = [&](const sbjson::Value* o, const char* k) -> const sbjson::Value* {
        const sbjson::Value* x = o ? o->get(k) : nullptr;
        if (!x) throw Error(17, "Faild to parse model config from file: `" + config_path + "`. Caused by: `missing field `" + k + "``");
        return x;
    };
    const sbjson::Value* r = root.get();
    if (auto* k = r->get("key")) if (k->kind == sbjson::Value::Str) v->key = k->str;
    const sbjson::Value* audio = req(r, "audio");
    v->sample_rate = (int)req(audio, "sample_rate")->num;
    if (auto* q = audio->get("quality")) if (q->kind == sbjson::Value::Str) v->quality = q->str;
    v->num_speakers = (int)req(r, "num_speakers")->num;
    if (auto* sm = req(r, "speaker_id_map")) for (auto& kv : sm->obj) v->speaker_id_map[kv.first] = (long long)kv.second->num;
    if (auto* s = r->get("streaming")) v->streaming = (s->kind == sbjson::Value::Bool && s->b);
    v->espeak_voice = req(req(r, "espeak"), "voice")->str;
    if (auto* l = r->get("language")) if (auto* c = l->get("code")) v->language_code = c->str;
    const sbjson::Value* inf = req(r, "inference");
    v->factory_cfg.noise_scale = (float)req(inf, "noise_scale")->num;
    v->factory_cfg.length_scale = (float)req(inf, "length_scale")->num;
    v->factory_cfg.noise_w = (float)req(inf, "noise_w")->num;
    v->factory_cfg.has_speaker = false;
    v->cfg = v->factory_cfg;                 // load_model_config: speaker: None (:54-59)
    v->num_symbols = (int)req(r, "num_symbols")->num;
    for (auto& kv : req(r, "phoneme_id_map")->obj) {
        if (kv.second->kind != sbjson::Value::Arr || kv.second->arr.empty()) continue;
        v->phoneme_first_id[first_code_point(kv.first)] = (long long)kv.second->arr[0]->num;
    }

    if (device == -1) return v.release();   // config-only handle (host logic, id mapping): no synthesis possible

    // weights: `<name>.onnx.json` -> `<name>.svw` (the reference opens `<name>.onnx`, :98-108)
    std::string stem = config_path;
    const std::string suf = ".json";
    if (stem.size() > suf.size() && stem.compare(stem.size() - suf.size(), suf.size(), suf) == 0)
        stem.resize(stem.size() - suf.size());
    else
        throw Error(19, "Invalid config filename format `" + config_path + "`");
    std::string wpath = stem;
    const std::string onnx = ".onnx";
    if (wpath.size() > onnx.size() && wpath.compare(wpath.size() - onnx.size(), onnx.size(), onnx) == 0)
        wpath.resize(wpath.size() - onnx.size());
    wpath += ".svw";
    const std::string wbuf = read_file(wpath, ok);
    if (!ok) throw Error(19, "Failed to initialize inference session: cannot open weight file `" + wpath + "`");
    TensorMap m = parse_svw(wbuf, wpath);

    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        throw Error(19, "Failed to initialize inference session: no CUDA device is visible (libsonata_b200 has no CPU path)");
    if (device < 0 || device >= ndev) throw Error(19, "Failed to initialize inference session: invalid CUDA device ordinal");
    SB_CUDA(cudaSetDevice(device));

    Arch& a = v->a;
    {
        const HostTensor& h = T(m, "hp.arch");
        if (!h.is_int || h.i.size() < 16) throw Error(17, "bad hp.arch tensor");
        const int* p = h.i.data();
        a.hidden = p[0]; a.inter = p[1]; a.filter = p[2]; a.heads = p[3]; a.layers = p[4]; a.kernel = p[5];
        a.window = p[6]; a.n_vocab = p[7]; a.resblock = p[8]; a.up_init = p[9]; a.flow_n = p[10];
        a.wn_layers = p[11]; a.flow_kernel = p[12]; a.dp_kernel = p[13]; a.dp_bins = p[14]; a.sample_rate = p[15];
        a.up_rates = T(m, "hp.up_rates").i;
        a.up_kernels = T(m, "hp.up_kernels").i;
        a.res_kernels = T(m, "hp.res_kernels").i;
        const HostTensor& rd = T(m, "hp.res_dils");
        for (int i = 0; i < rd.dims[0]; i++)
            a.res_dils.emplace_back(rd.i.begin() + (size_t)i * rd.dims[1], rd.i.begin() + (size_t)(i + 1) * rd.dims[1]);
    }
    const int H = a.hidden, I = a.inter;
    if (H % 32 || I % 32 || (I & 1) || a.filter % 32 || (a.flow_n & 1) || a.dp_bins != 10 || a.dp_kernel != 3 || a.hop() != 256)
        throw Error(17, "unsupported voice architecture (hidden " + std::to_string(H) + ", inter " + std::to_string(I) +
                        ", filter " + std::to_string(a.filter) + ", hop " + std::to_string(a.hop()) + ")");
    const int D = H / a.heads;
    if (D != 96 && D != 48) throw Error(17, "unsupported attention head size");
    if (H != 96 && H != 192 && H != 256) throw Error(17, "unsupported hidden width (LayerNorm kernels: 96 / 192 / 256)");

    Uploader U{v.get()};
    v->emb = U.up(T(m, "enc_p.emb.weight").f);
    for (int l = 0; l < a.layers; l++) {
        EncLayer e;
        const std::string p = "enc_p.encoder.attn_layers." + std::to_string(l) + ".";
        e.qkv = make_conv(U, ENC_IMAGES, {&T(m, p + "conv_q.weight"), &T(m, p + "conv_k.weight"), &T(m, p + "conv_v.weight")},
                          {&T(m, p + "conv_q.bias"), &T(m, p + "conv_k.bias"), &T(m, p + "conv_v.bias")}, 1);
        e.o = conv_named(U, ENC_IMAGES, m, p + "conv_o");
        e.relk = U.up(T(m, p + "emb_rel_k").f);
        e.relv = U.up(T(m, p + "emb_rel_v").f);
        const std::string n1 = "enc_p.encoder.norm_layers_1." + std::to_string(l);
        const std::string n2 = "enc_p.encoder.norm_layers_2." + std::to_string(l);
        e.g1 = U.up(T(m, n1 + ".gamma").f); e.b1 = U.up(T(m, n1 + ".beta").f);
        e.g2 = U.up(T(m, n2 + ".gamma").f); e.b2 = U.up(T(m, n2 + ".beta").f);
        const std::string f = "enc_p.encoder.ffn_layers." + std::to_string(l) + ".";
        e.ffn1 = conv_named(U, ENC_IMAGES, m, f + "conv_1");
        e.ffn2 = conv_named(U, ENC_IMAGES, m, f + "conv_2");
        v->enc.push_back(e);
    }
    v->enc_proj = conv_named(U, ENC_IMAGES, m, "enc_p.proj");

    v->dp_pre = conv_named(U, ENC_IMAGES, m, "dp.pre");
    v->dp_proj = conv_named(U, ENC_IMAGES, m, "dp.proj");
    v->dp_dds = load_dds(U, m, "dp.convs.", H, a.dp_kernel);
    {
        // reversed(flows)[:-2] + [EA]: Flip, CF4^-1, Flip, CF3^-1, Flip, CF2^-1, Flip, EA^-1.  The flips
        // only alternate which of the two channels conditions / is transformed (see DESIGN.md).
        const int order[3] = {7, 5, 3};
        for (int s = 0; s < 3; s++) {
            CFlowW cf;
            const std::string p = "dp.flows." + std::to_string(order[s]) + ".";
            cf.pre_w = U.up(T(m, p + "pre.weight").f);
            cf.pre_b = U.up(T(m, p + "pre.bias").f);
            cf.dds = load_dds(U, m, p + "convs.", H, a.dp_kernel);
            cf.proj = conv_named(U, ENC_IMAGES, m, p + "proj", 1, true, nullptr, nullptr, 32);
            cf.ccol = (s % 2 == 0) ? 1 : 0;
            cf.tcol = 1 - cf.ccol;
            v->dp_flows.push_back(cf);
        }
        v->ea_m0 = T(m, "dp.flows.0.m").f[0];
        v->ea_logs0 = T(m, "dp.flows.0.logs").f[0];
    }
    {
        const int half = I / 2;
        std::vector<int> rev(half);
        for (int i = 0; i < half; i++) rev[i] = half - 1 - i;
        std::vector<int> gate(2 * H);   // interleave (tanh_j, sigmoid_j)
        for (int j = 0; j < H; j++) { gate[2 * j] = j; gate[2 * j + 1] = H + j; }
        for (int step = 0; step < a.flow_n; step++) {
            const int f = a.flow_n - 1 - step;
            const bool reversed = (step % 2 == 0);   // an odd number of channel flips precede this layer
            const std::string p = "flow.flows." + std::to_string(2 * f) + ".";
            CouplingW c;
            c.cond_off = reversed ? half : 0;
            c.tgt_off = reversed ? 0 : half;
            if (half % 32 == 0) {
                c.pre = conv_named(U, DEC_IMAGES, m, p + "pre", 1, true, nullptr, reversed ? &rev : nullptr);
            } else {
                // A half that is not a whole number of 32-channel K-blocks (x_low: 48 of 96) keeps the tensor-core convs
                // by widening pre and post to all `inter` channels of z: pre reads the target half with zero weights,
                // post writes the conditioning half with zero weights and bias.  Exact zeros change no sum.
                const HostTensor w = widen(T(m, p + "pre.weight"), I, 1, c.cond_off, reversed);
                c.pre = make_conv(U, DEC_IMAGES, {&w}, {&T(m, p + "pre.bias")}, 1);
                c.cond_off = 0;
            }
            for (int l = 0; l < a.wn_layers; l++) {
                c.in.push_back(conv_named(U, DEC_IMAGES, m, p + "enc.in_layers." + std::to_string(l), 1, true, &gate));
                c.rs.push_back(conv_named(U, DEC_IMAGES, m, p + "enc.res_skip_layers." + std::to_string(l)));
            }
            if (half % 32 == 0) {
                c.post = conv_named(U, DEC_IMAGES, m, p + "post", 1, true, reversed ? &rev : nullptr);
            } else {
                const HostTensor w = widen(T(m, p + "post.weight"), I, 0, c.tgt_off, reversed);
                const HostTensor b = widen(T(m, p + "post.bias"), I, 0, c.tgt_off, reversed);
                c.post = make_conv(U, DEC_IMAGES, {&w}, {&b}, 1);
                c.tgt_off = 0;
            }
            v->flows.push_back(c);
        }
    }
    v->conv_pre = conv_named(U, DEC_IMAGES, m, "dec.conv_pre");
    {
        int C = a.up_init;
        const int nk = (int)a.res_kernels.size();
        for (size_t i = 0; i < a.up_rates.size(); i++) {
            UpStageW st;
            st.u = a.up_rates[i]; st.k = a.up_kernels[i]; st.cin = C; st.cout = C / 2;
            const HostTensor& w = T(m, "dec.ups." + std::to_string(i) + ".weight");   // [cin][cout][k]
            const HostTensor& b = T(m, "dec.ups." + std::to_string(i) + ".bias");
            // polyphase: output n = q*u + p reads input q + off through kernel index p + pad - off*u, for every off that
            // puts the index in [0, k)
            const int pad = (st.k - st.u) / 2;
            auto kidx = [&](int p, int off) { const int kk = p + pad - off * st.u; return kk >= 0 && kk < st.k ? kk : -1; };
            // phase p's weights, for the taps of c, into columns [col0, col0 + cout) of wt [ntaps][cin][ldw]
            auto put_phase = [&](const ConvW& c, int p, int col0, std::vector<float>& wt) {
                for (int t = 0; t < c.ntaps; t++) {
                    const int kk = kidx(p, c.tap_off[t]);
                    if (kk < 0) continue;
                    for (int ci = 0; ci < c.cin; ci++)
                        for (int n = 0; n < st.cout; n++)
                            wt[((size_t)t * c.cin + ci) * c.ldw + col0 + n] = w.f[((size_t)ci * st.cout + n) * st.k + kk];
                }
            };
            std::vector<int> all;    // union of the phases' taps
            for (int p = 0; p < st.u; p++) {
                std::vector<int> offs;      // descending: the order in which the fp32 kernel sums the taps
                for (int off = st.k; off >= -st.k; off--)
                    if (kidx(p, off) >= 0) offs.push_back(off);
                ConvW c = conv_layout(st.cin, st.cout, offs);
                std::vector<float> wt((size_t)c.ntaps * c.cin * c.ldw, 0.f), bt(c.ldw, 0.f);
                put_phase(c, p, 0, wt);
                std::copy(b.f.begin(), b.f.begin() + st.cout, bt.begin());
                upload_conv(U, c, wt, bt, IMG_F32);
                st.phase.push_back(c);
                for (int off : offs)
                    if (std::find(all.begin(), all.end(), off) == all.end()) all.push_back(off);
            }
            if (all.size() <= SB_MAX_TAPS && st.cout % 32 == 0) {
                // all phases as ONE conv (conv_tc): taps = union of the phase taps, column p*cout + co = phase p,
                // channel co.  Its zero taps are no work: macs counts the ConvTranspose's own.
                std::sort(all.begin(), all.end());
                ConvW f = conv_layout(st.cin, st.u * st.cout, all, false);
                f.macs = st.cin * st.cout * st.k;
                std::vector<float> wt((size_t)f.ntaps * f.cin * f.ldw, 0.f), bt(f.ldw, 0.f);
                for (int p = 0; p < st.u; p++) {
                    put_phase(f, p, p * st.cout, wt);
                    std::copy(b.f.begin(), b.f.begin() + st.cout, bt.begin() + p * st.cout);
                }
                upload_conv(U, f, wt, bt, IMG_BF16);
                st.fused = f;
            }
            C /= 2;
            for (int j = 0; j < nk; j++) {
                ResBW rb; rb.k = a.res_kernels[j]; rb.dils = a.res_dils[j];
                const std::string p = "dec.resblocks." + std::to_string(i * nk + j) + ".";
                for (size_t d = 0; d < rb.dils.size(); d++) {
                    if (a.resblock == 2) rb.c1.push_back(conv_named(U, DEC_IMAGES, m, p + "convs." + std::to_string(d), rb.dils[d]));
                    else {
                        rb.c1.push_back(conv_named(U, DEC_IMAGES, m, p + "convs1." + std::to_string(d), rb.dils[d]));
                        rb.c2.push_back(conv_named(U, DEC_IMAGES, m, p + "convs2." + std::to_string(d), 1));
                    }
                }
                st.res.push_back(rb);
            }
            v->ups.push_back(st);
        }
        v->c_last = C;
        const HostTensor& w = T(m, "dec.conv_post.weight");   // [1][C][7]
        std::vector<float> wt((size_t)7 * C);
        for (int c = 0; c < C; c++) for (int t = 0; t < 7; t++) wt[(size_t)t * C + c] = w.f[(size_t)c * 7 + t];
        v->conv_post_w = U.up(wt);
        if (C != 16 && C != 32 && C != 64) throw Error(17, "unsupported final decoder width");
    }
    if (v->num_speakers > 1) {
        // Multi-speaker voice: g = emb_g(sid) conditions the duration predictor (dp.cond), every coupling layer's WaveNet
        // (enc.cond_layer, 2H rows per layer) and the HiFi-GAN input (dec.cond) through 1x1 convs of a [gin, 1] vector,
        // i.e. g only adds a per-call vector to the BIAS of dp.pre, of every WaveNet in_layer and of conv_pre.  All those
        // rows are stacked into one [rows][gin] matrix (+ base bias = conv bias + cond bias); one small kernel per call
        // produces the effective biases (engine.cu).  Reference: `sid` input, piper/src/lib.rs:353-358.
        const HostTensor& eg = T(m, "emb_g.weight");
        if (eg.dims.size() != 2 || eg.dims[0] < v->num_speakers) throw Error(17, "emb_g.weight does not cover num_speakers");
        const int G = eg.dims[1];
        v->gin = G; v->emb_rows = eg.dims[0];
        v->emb_g = U.up(eg.f);
        std::vector<float> wc, base;
        auto add = [&](ConvW& c, const HostTensor& cw, const HostTensor& cb, int row0, const std::vector<int>* perm,
                       const std::vector<float>& conv_bias /* padded to ldw */) {
            if (cw.dims[1] != G) throw Error(17, "conditioning layer width does not match emb_g");
            c.cond_off = (int)base.size();
            for (int n = 0; n < c.ldw; n++) {
                const bool live = n < c.cout;
                const int src = live ? row0 + (perm ? (*perm)[n] : n) : 0;
                for (int k = 0; k < G; k++) wc.push_back(live ? cw.f[(size_t)src * G + k] : 0.f);
                base.push_back(live ? conv_bias[n] + cb.f[src] : 0.f);
            }
        };
        auto host_bias = [&](const ConvW& c) {
            std::vector<float> b(c.ldw);
            SB_CUDA(cudaMemcpy(b.data(), c.bias, (size_t)c.ldw * 4, cudaMemcpyDeviceToHost));
            return b;
        };
        add(v->dp_pre, T(m, "dp.cond.weight"), T(m, "dp.cond.bias"), 0, nullptr, host_bias(v->dp_pre));
        std::vector<int> gate(2 * H);
        for (int j = 0; j < H; j++) { gate[2 * j] = j; gate[2 * j + 1] = H + j; }
        for (int step = 0; step < a.flow_n; step++) {
            const int f = a.flow_n - 1 - step;
            const std::string p = "flow.flows." + std::to_string(2 * f) + ".enc.cond_layer.";
            for (int l = 0; l < a.wn_layers; l++)
                add(v->flows[step].in[l], T(m, p + "weight"), T(m, p + "bias"), 2 * H * l, &gate, host_bias(v->flows[step].in[l]));
        }
        add(v->conv_pre, T(m, "dec.cond.weight"), T(m, "dec.cond.bias"), 0, nullptr, host_bias(v->conv_pre));
        v->cond_rows = (int)base.size();
        v->cond_w = U.up(wc);
        v->cond_base = U.up(base);
    }
    SB_CUDA(cudaDeviceSynchronize());
    return v.release();
}

}  // namespace sb200
