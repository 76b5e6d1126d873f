// FLAC (RFC 9639) of 16-bit mono streams, encoded on the device: fixed blocks of 4096 samples, one CTA per frame.
//   flac_analyze_kernel  CONSTANT, the five FIXED predictors and LPC 1-8 with exact optimal Rice costs -> the choice
//                        and the frame's byte size;
//   flac_layout_kernel   the frames' byte offsets, and each stream's length and min / max frame size;
//   flac_pack_kernel     the frame's bits at its offset (per-sample bit offsets from a block scan), then CRC-8 and
//                        CRC-16.
// The host only lays out the frames, reads the size table back and prepends each stream's 42-byte STREAMINFO.
#include "engine.h"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace sb200 {

namespace {

constexpr int FB = 4096;               // block size of every frame but a stream's last
constexpr int FT = 256;                // threads per frame CTA
constexpr int SPT = FB / FT;           // consecutive samples per thread
constexpr int MAX_LPC = 8;
constexpr int KB = 31;                 // Rice parameters 0..30: a zigzag residual is < 2^31
constexpr int BUF_WORDS = 2064;        // a frame's bytes: at most VERBATIM's 8193 + 16 header + 2 CRC-16
constexpr int FLAC_LPC_PRECISION = 12;

struct FrameIn {
    long long x_off;                   // first sample in the input buffer
    int n;                             // block size
    int frame_no;                      // within its stream
    int rate_code, rate_hz;            // 4-bit sample-rate code; rate_hz is written for code 13
};
// What the analysis chose for a frame, and its size in bytes (header and both CRCs included).
struct Choice {
    int type;                          // 0 CONSTANT, 1 VERBATIM, 2 FIXED, 3 LPC
    int order, shift, porder;
    int coef[MAX_LPC];                 // the first multiplies x[n-1]
    int bytes;
};
struct StreamRange { int first, count; };

struct Smem {
    unsigned cnt[KB][512];             // per-bit counts of the zigzag residuals: partition p of order o at [2^o - 1 + p]
    unsigned long long tot[9];         // per partition order: sum over partitions of the minimal Rice cost
    int kmax[9];                       // per partition order: the largest optimal parameter
    unsigned char k[256];              // pack: the parameter of every partition of the chosen order
    unsigned buf[BUF_WORDS];           // pack: the frame's bytes, byte j at bits 8 (j & 3) of word j / 4
    double red[FT / 32][MAX_LPC + 1];  // autocorrelation partial sums per warp
    int lpc_ok[MAX_LPC + 1], lpc_shift[MAX_LPC + 1], lpc_q[MAX_LPC + 1][MAX_LPC];
    int scan[FT / 32];
    unsigned crc[FT / 32];
};

// The fixed predictors as coefficient lists (shift 0): x[n-1], 2x[n-1] - x[n-2], ...
__constant__ int c_fixed[5][4] = {{0, 0, 0, 0}, {1, 0, 0, 0}, {2, -1, 0, 0}, {3, -3, 1, 0}, {4, -6, 4, -1}};

// v's low len (<= 32) bits, most significant first, at bit pos of the frame buffer.
__device__ __forceinline__ void put_bits(unsigned* buf, int pos, unsigned v, int len) {
    while (len > 0) {
        const int byte = pos >> 3, room = 8 - (pos & 7), take = len < room ? len : room;
        const unsigned bits = (unsigned)((v >> (len - take)) & ((1u << take) - 1));
        atomicOr(&buf[byte >> 2], (bits << (room - take)) << ((byte & 3) * 8));
        pos += take; len -= take;
    }
}

// The frame header without its CRC-8, written from byte 0 of buf (null: only counted); returns its bytes.
__device__ __forceinline__ int frame_header(const FrameIn& f, unsigned* buf) {
    int b = 0;
    auto put = [&](unsigned v) { if (buf) put_bits(buf, 8 * b, v & 0xFF, 8); b++; };
    put(0xFF); put(0xF8);                                          // sync, blocking strategy 0 (fixed)
    const int bs_code = f.n == FB ? 12 : f.n <= 256 ? 6 : 7;
    put((unsigned)((bs_code << 4) | f.rate_code));
    put(0x08);                                                     // mono, 16 bits, reserved 0
    const unsigned v = (unsigned)f.frame_no;                      // UTF-8-style coded frame number
    if (v < 0x80) {
        put(v);
    } else {
        const int len = v < 0x800 ? 2 : v < 0x10000 ? 3 : v < 0x200000 ? 4 : v < 0x4000000 ? 5 : 6;
        put((0xFF00u >> len) | (v >> (6 * (len - 1))));
        for (int i = len - 2; i >= 0; i--) put(0x80 | ((v >> (6 * i)) & 0x3F));
    }
    if (bs_code == 6) put((unsigned)(f.n - 1));
    if (bs_code == 7) { put((unsigned)(f.n - 1) >> 8); put((unsigned)(f.n - 1)); }
    if (f.rate_code == 13) { put((unsigned)f.rate_hz >> 8); put((unsigned)f.rate_hz); }
    return b;
}

__device__ __forceinline__ uint8_t crc8(const uint8_t* p, int n) {       // polynomial 0x07, init 0
    unsigned c = 0;
    for (int i = 0; i < n; i++) {
        c ^= p[i];
        for (int j = 0; j < 8; j++) c = (c & 0x80) ? ((c << 1) ^ 0x07) & 0xFF : (c << 1) & 0xFF;
    }
    return (uint8_t)c;
}

// CRC-16 (polynomial 0x8005, init 0) arithmetic: a * b mod P over GF(2), and the CRC of a byte run from 0.
__device__ __forceinline__ unsigned crc16_mul(unsigned a, unsigned b) {
    unsigned r = 0;
    for (int i = 15; i >= 0; i--) {
        r = (r & 0x8000) ? ((r << 1) ^ 0x8005) & 0xFFFF : (r << 1) & 0xFFFF;
        if ((b >> i) & 1) r ^= a;
    }
    return r;
}
__device__ __forceinline__ unsigned crc16_run(const uint8_t* p, int lo, int hi) {
    unsigned c = 0;
    for (int i = lo; i < hi; i++) {
        c ^= (unsigned)p[i] << 8;
        for (int j = 0; j < 8; j++) c = (c & 0x8000) ? ((c << 1) ^ 0x8005) & 0xFFFF : (c << 1) & 0xFFFF;
    }
    return c;
}

// x[i0 - 8 .. i0 + SPT) of the frame into registers, 0 outside [0, n).
__device__ __forceinline__ void load_window(const short* __restrict__ x, int n, int i0, int (&w)[SPT + 8]) {
#pragma unroll
    for (int m = 0; m < SPT + 8; m++) {
        const int i = i0 - 8 + m;
        w[m] = (i >= 0 && i < n) ? (int)__ldg(x + i) : 0;
    }
}

// Zigzag residuals of the thread's samples for the predictor q (shift sh, `order` warm-up samples, which get 0).
__device__ __forceinline__ void residuals(const int (&w)[SPT + 8], const int (&q)[MAX_LPC], int sh, int order, int i0,
                                          int n, unsigned (&u)[SPT]) {
#pragma unroll
    for (int m = 0; m < SPT; m++) {
        int acc = 0;
#pragma unroll
        for (int j = 0; j < MAX_LPC; j++) acc += q[j] * w[8 + m - 1 - j];
        const int r = w[8 + m] - (acc >> sh);
        const int i = i0 + m;
        u[m] = (i < order || i >= n) ? 0u : (((unsigned)r << 1) ^ (unsigned)(r >> 31));
    }
}

// Per-bit counts of u over the partitions of order `leaf` (n divisible by 2^leaf), summed up the heap to order 0.
// Exact integer sums, so the result does not depend on the order the threads add in.
__device__ void rice_counts(Smem& S, const unsigned (&u)[SPT], int i0, int n, int leaf) {
    const int t = threadIdx.x, nl = 1 << leaf, L = n >> leaf, base = nl - 1;
    for (int e = t; e < KB * nl; e += FT) S.cnt[e / nl][base + e % nl] = 0;
    if (t < 9) { S.tot[t] = 0; S.kmax[t] = 0; }
    __syncthreads();
    if (i0 < n) {
        const int first = i0 / L;
        for (int b = 0; b < KB; b++) {
            int cur = first, bound = (first + 1) * L;
            unsigned acc = 0;
#pragma unroll
            for (int m = 0; m < SPT; m++) {
                const int i = i0 + m;
                if (i < n) {
                    if (i == bound) { atomicAdd(&S.cnt[b][base + cur], acc); acc = 0; cur++; bound += L; }
                    acc += (u[m] >> b) & 1u;
                }
            }
            atomicAdd(&S.cnt[b][base + cur], acc);
        }
    }
    __syncthreads();
    for (int o = leaf - 1; o >= 0; o--) {
        const int np = 1 << o;
        for (int e = t; e < KB * np; e += FT) {
            const int b = e / np, p = e % np;
            S.cnt[b][np - 1 + p] = S.cnt[b][2 * np - 1 + 2 * p] + S.cnt[b][2 * np - 1 + 2 * p + 1];
        }
        __syncthreads();
    }
}

// The optimal Rice parameter of every partition of every order 0..leaf (only order `only` when >= 0) that is valid for
// a predictor of `order`: S_k = sum(u >> k) from the counts, cost = S_k + samples * (k + 1), the smallest k on a tie.
// Adds into S.tot / S.kmax; with `only` it also stores the parameters in S.k.
__device__ void rice_eval(Smem& S, int n, int order, int leaf, int only) {
    for (int e = threadIdx.x; e < (2 << leaf) - 1; e += FT) {
        const int o = 31 - __clz(e + 1), p = e + 1 - (1 << o);
        if ((only >= 0 && o != only) || (n >> o) <= order) continue;
        const unsigned long long np = (unsigned long long)((n >> o) - (p == 0 ? order : 0));
        unsigned long long s = 0, best = ~0ull;
        int kb = 0;
        for (int b = KB - 1; b >= 0; b--) {
            s = 2 * s + S.cnt[b][e];
            const unsigned long long c = s + np * (unsigned long long)(b + 1);
            if (c <= best) { best = c; kb = b; }
        }
        atomicAdd(&S.tot[o], best);
        atomicMax(&S.kmax[o], kb);
        if (only >= 0) S.k[p] = (unsigned char)kb;
    }
    __syncthreads();
}

// The residual's bits for its best partition order (method, order, parameters and codes), smallest order on a tie.
__device__ __forceinline__ unsigned long long rice_best(const Smem& S, int n, int order, int leaf, int* porder) {
    unsigned long long best = ~0ull;
    for (int o = 0; o <= leaf; o++) {
        if ((n >> o) <= order) break;
        const unsigned long long bits = 6 + S.tot[o] + (unsigned long long)(1 << o) * (S.kmax[o] > 14 ? 5 : 4);
        if (bits < best) { best = bits; *porder = o; }
    }
    return best;
}

// Tukey(0.5) window of an n-sample frame at sample i (scipy.signal.windows.tukey(n, 0.5), symmetric).
__device__ __forceinline__ double tukey(int i, int n) {
    if (n <= 1) return 1.0;
    const int m = min(i, n - 1 - i);
    const double span = 0.5 * (double)(n - 1);
    if ((double)m >= 0.5 * span) return 1.0;
    return 0.5 * (1.0 + cos(3.14159265358979323846 * (-1.0 + 2.0 * (double)m / span)));
}

// Levinson-Durbin on R[0..8] and 12-bit quantisation with error feedback, one thread, all in double.  Order p is kept
// when the recursion reached it and some shift in 0..15 fits every coefficient in [-2048, 2047] (the largest such).
// (The loops over orders and coefficients unroll, so the arrays stay in registers.)
__device__ __forceinline__ void lpc_design(Smem& S, const double (&R)[MAX_LPC + 1]) {
#pragma unroll
    for (int p = 0; p <= MAX_LPC; p++) S.lpc_ok[p] = 0;
    double a[MAX_LPC + 1] = {0}, err = R[0];
    if (!(err > 0.0) || !isfinite(err)) return;
    const double qmax = (1 << (FLAC_LPC_PRECISION - 1)) - 1, qmin = -(1 << (FLAC_LPC_PRECISION - 1));
#pragma unroll
    for (int i = 1; i <= MAX_LPC; i++) {
        double acc = R[i];
#pragma unroll
        for (int j = 1; j < i; j++) acc -= a[j] * R[i - j];
        const double k = acc / err;
        double na[MAX_LPC + 1];
#pragma unroll
        for (int j = 1; j < i; j++) na[j] = a[j] - k * a[i - j];
#pragma unroll
        for (int j = 1; j < i; j++) a[j] = na[j];
        a[i] = k;
        err *= 1.0 - k * k;
        bool finite = isfinite(k);
#pragma unroll
        for (int j = 1; j <= i; j++) finite = finite && isfinite(a[j]);
        if (!finite) return;
        for (int s = 15; s >= 0; s--) {
            double e = 0.0;
            bool fits = true;
            int q[MAX_LPC];
#pragma unroll
            for (int j = 0; j < MAX_LPC; j++) {
                q[j] = 0;
                if (j < i && fits) {
                    const double v = a[j + 1] * (double)(1 << s) + e;
                    const double r = round(v);
                    fits = r >= qmin && r <= qmax;
                    q[j] = fits ? (int)r : 0;
                    e = v - r;
                }
            }
            if (fits) {
                S.lpc_ok[i] = 1; S.lpc_shift[i] = s;
#pragma unroll
                for (int j = 0; j < MAX_LPC; j++) S.lpc_q[i][j] = q[j];
                break;
            }
        }
        if (!(err > 0.0)) return;
    }
}

// The predictor of candidate c: 0..4 FIXED of that order, 5..12 LPC of order c - 4.  False when it does not apply.
__device__ __forceinline__ bool candidate(const Smem& S, int c, int n, int (&q)[MAX_LPC], int* sh, int* order) {
    *order = c < 5 ? c : c - 4;
    if (n <= *order || (c >= 5 && !S.lpc_ok[*order])) return false;
#pragma unroll
    for (int j = 0; j < MAX_LPC; j++) q[j] = c < 5 ? (j < 4 ? c_fixed[c][j] : 0) : S.lpc_q[*order][j];
    *sh = c < 5 ? 0 : S.lpc_shift[*order];
    return true;
}

__global__ void __launch_bounds__(FT) flac_analyze_kernel(const short* __restrict__ x, const FrameIn* __restrict__ frames,
                                                          Choice* __restrict__ out) {
    pdl_trigger(); pdl_wait();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Smem& S = *reinterpret_cast<Smem*>(smem_raw);
    const FrameIn f = frames[blockIdx.x];
    const short* xf = x + f.x_off;
    const int t = threadIdx.x, n = f.n, i0 = t * SPT, lane = t & 31, wid = t >> 5;
    const int leaf = min(8, __ffs(n) - 1);
    int w[SPT + 8];
    load_window(xf, n, i0, w);

    bool same = true;
    const int x0 = __ldg(xf);
#pragma unroll
    for (int m = 0; m < SPT; m++) same = same && (i0 + m >= n || w[8 + m] == x0);
    if (__syncthreads_and(same)) {
        if (t == 0) {
            Choice c{};
            c.type = 0;
            c.bytes = frame_header(f, nullptr) + 1 + 3 + 2;
            out[blockIdx.x] = c;
        }
        return;
    }

    // LPC design: autocorrelation of the windowed frame, lags 0..8, each thread over its own samples, then a fixed tree
    double R[MAX_LPC + 1];
    {
        double y[SPT + 8];
#pragma unroll
        for (int m = 0; m < SPT + 8; m++) {
            const int i = i0 - 8 + m;
            y[m] = (i >= 0 && i < n) ? (double)w[m] * tukey(i, n) : 0.0;
        }
#pragma unroll
        for (int l = 0; l <= MAX_LPC; l++) {
            double s = 0.0;
#pragma unroll
            for (int m = 8; m < SPT + 8; m++) s += y[m] * y[m - l];
            R[l] = s;
        }
    }
#pragma unroll
    for (int l = 0; l <= MAX_LPC; l++) {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) R[l] += __shfl_down_sync(0xffffffffu, R[l], d);
        if (lane == 0) S.red[wid][l] = R[l];
    }
    __syncthreads();
    if (t == 0) {
#pragma unroll
        for (int l = 0; l <= MAX_LPC; l++) {
            double s = 0.0;
            for (int v = 0; v < FT / 32; v++) s += S.red[v][l];
            R[l] = s;
        }
        lpc_design(S, R);
    }
    __syncthreads();

    // Candidates in tie order: FIXED 0..4, LPC 1..8; VERBATIM only when strictly smaller
    unsigned long long best = ~0ull;
    Choice bc{};
    for (int c = 0; c < 5 + MAX_LPC; c++) {
        int q[MAX_LPC], sh = 0, order = 0;
        if (!candidate(S, c, n, q, &sh, &order)) continue;       // uniform across the CTA
        unsigned u[SPT];
        residuals(w, q, sh, order, i0, n, u);
        rice_counts(S, u, i0, n, leaf);
        rice_eval(S, n, order, leaf, -1);
        if (t == 0) {
            int po = 0;
            const unsigned long long rb = rice_best(S, n, order, leaf, &po);
            const unsigned long long bits = 8 + 16ull * order + (c >= 5 ? 9 + 12ull * order : 0) + rb;
            if (bits < best) {
                best = bits;
                bc.type = c < 5 ? 2 : 3; bc.order = order; bc.shift = sh; bc.porder = po;
#pragma unroll
                for (int j = 0; j < MAX_LPC; j++) bc.coef[j] = q[j];
            }
        }
        __syncthreads();
    }
    if (t == 0) {
        const unsigned long long verbatim = 8 + 16ull * n;
        if (verbatim < best) { best = verbatim; bc = Choice{}; bc.type = 1; }
        bc.bytes = frame_header(f, nullptr) + 1 + (int)((best + 7) / 8) + 2;
        out[blockIdx.x] = bc;
    }
}

// Exclusive scan of the frames' sizes in stream order (each stream's frames are contiguous), then per stream: its
// first byte, its length and its smallest and largest frame.  One CTA; every sum is exact.
__global__ void __launch_bounds__(1024) flac_layout_kernel(const Choice* __restrict__ ch, int nframes,
                                                           const StreamRange* __restrict__ streams, int nstreams,
                                                           long long* __restrict__ off, long long* __restrict__ stats) {
    pdl_trigger(); pdl_wait();
    __shared__ long long warp_tot[32];
    __shared__ long long carry;
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    if (t == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < nframes; base += 1024) {
        const long long v = base + t < nframes ? ch[base + t].bytes : 0;
        long long s = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const long long o = __shfl_up_sync(0xffffffffu, s, d);
            if (lane >= d) s += o;
        }
        if (lane == 31) warp_tot[wid] = s;
        __syncthreads();
        long long before = carry;
        for (int v2 = 0; v2 < wid; v2++) before += warp_tot[v2];
        if (base + t < nframes) off[base + t] = before + s - v;
        __syncthreads();
        if (t == 1023) carry = before + s;
        __syncthreads();
    }
    for (int s = t; s < nstreams; s += 1024) {
        const StreamRange r = streams[s];
        long long* st = stats + 4 * (size_t)s;
        if (r.count == 0) { st[0] = st[1] = st[2] = st[3] = 0; continue; }
        long long lo = 1ll << 40, hi = 0;
        for (int k = 0; k < r.count; k++) {
            const long long b = ch[r.first + k].bytes;
            lo = b < lo ? b : lo; hi = b > hi ? b : hi;
        }
        const int last = r.first + r.count - 1;
        st[0] = off[r.first];
        st[1] = off[last] + ch[last].bytes - off[r.first];
        st[2] = lo; st[3] = hi;
    }
}

__global__ void __launch_bounds__(FT) flac_pack_kernel(const short* __restrict__ x, const FrameIn* __restrict__ frames,
                                                       const Choice* __restrict__ choices,
                                                       const long long* __restrict__ off, uint8_t* __restrict__ out) {
    pdl_trigger(); pdl_wait();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Smem& S = *reinterpret_cast<Smem*>(smem_raw);
    const FrameIn f = frames[blockIdx.x];
    const Choice c = choices[blockIdx.x];
    const short* xf = x + f.x_off;
    const int t = threadIdx.x, n = f.n, i0 = t * SPT, lane = t & 31, wid = t >> 5;
    const int F = c.bytes, words = (F + 3) / 4;
    for (int e = t; e < words; e += FT) S.buf[e] = 0;
    int w[SPT + 8];
    load_window(xf, n, i0, w);
    __syncthreads();

    const int H = frame_header(f, nullptr) + 1;
    int pos = 8 * H + 8;                                  // the subframe header is followed by ...
    if (c.type >= 2) pos += 16 * c.order + (c.type == 3 ? 9 + 12 * c.order : 0) + 6;   // ... the residual's codes
    int pbits = 4;
    if (c.type >= 2) {
        int q[MAX_LPC];
#pragma unroll
        for (int j = 0; j < MAX_LPC; j++) q[j] = c.coef[j];
        unsigned u[SPT];
        residuals(w, q, c.shift, c.order, i0, n, u);
        rice_counts(S, u, i0, n, c.porder);
        rice_eval(S, n, c.order, c.porder, c.porder);
        pbits = S.kmax[c.porder] > 14 ? 5 : 4;
        // bit lengths of the thread's codes (a partition's parameter before its first code), block exclusive scan
        const int L = n >> c.porder;
        int len[SPT], sum = 0;
#pragma unroll
        for (int m = 0; m < SPT; m++) {
            const int i = i0 + m;
            len[m] = 0;
            if (i >= c.order && i < n) {
                const int p = i / L, k = S.k[p];
                len[m] = (int)(u[m] >> k) + 1 + k + (i == (p == 0 ? c.order : p * L) ? pbits : 0);
            }
            sum += len[m];
        }
        int s = sum;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int o = __shfl_up_sync(0xffffffffu, s, d);
            if (lane >= d) s += o;
        }
        if (lane == 31) S.scan[wid] = s;
        __syncthreads();
        int at = pos + s - sum;
        for (int v = 0; v < wid; v++) at += S.scan[v];
#pragma unroll
        for (int m = 0; m < SPT; m++) {
            const int i = i0 + m;
            if (i < c.order || i >= n) continue;
            const int p = i / L, k = S.k[p];
            int b = at;
            if (i == (p == 0 ? c.order : p * L)) { put_bits(S.buf, b, (unsigned)k, pbits); b += pbits; }
            const int qz = (int)(u[m] >> k);
            put_bits(S.buf, b + qz, 1u, 1);
            if (k > 0) put_bits(S.buf, b + qz + 1, u[m] & ((1u << k) - 1), k);
            at += len[m];
        }
    } else if (c.type == 1) {
#pragma unroll
        for (int m = 0; m < SPT; m++)
            if (i0 + m < n) put_bits(S.buf, 8 * H + 8 + 16 * (i0 + m), (unsigned)(w[8 + m] & 0xFFFF), 16);
    }
    if (t == 0) {
        frame_header(f, S.buf);
        int b = 8 * H;
        const int type6 = c.type == 0 ? 0 : c.type == 1 ? 1 : c.type == 2 ? 8 | c.order : 32 | (c.order - 1);
        put_bits(S.buf, b, (unsigned)type6 << 1, 8); b += 8;
        if (c.type == 0) {
            put_bits(S.buf, b, (unsigned)(w[8] & 0xFFFF), 16);
        } else if (c.type >= 2) {
            for (int j = 0; j < c.order; j++, b += 16) put_bits(S.buf, b, (unsigned)(__ldg(xf + j) & 0xFFFF), 16);
            if (c.type == 3) {
                put_bits(S.buf, b, FLAC_LPC_PRECISION - 1, 4); b += 4;
                put_bits(S.buf, b, (unsigned)c.shift, 5); b += 5;
#pragma unroll
                for (int j = 0; j < MAX_LPC; j++)
                    if (j < c.order) put_bits(S.buf, b + 12 * j, (unsigned)c.coef[j] & 0xFFF, 12);
                b += 12 * c.order;
            }
            put_bits(S.buf, b, pbits == 5 ? 1u : 0u, 2); b += 2;
            put_bits(S.buf, b, (unsigned)c.porder, 4);
        }
    }
    __syncthreads();
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(S.buf);
    if (t == 0) put_bits(S.buf, 8 * (H - 1), crc8(bytes, H - 1), 8);
    __syncthreads();
    // CRC-16 of bytes [0, F - 2): each thread's run from 0, moved to its place by x^(8 * bytes after it), XOR-summed
    const int body = F - 2, per = (body + FT - 1) / FT;
    const int lo = min(body, t * per), hi = min(body, lo + per);
    unsigned crc = crc16_run(bytes, lo, hi);
    unsigned pw = 0x100;                                  // x^8 mod P
    for (int m = body - hi; m > 0; m >>= 1) {
        if (m & 1) crc = crc16_mul(crc, pw);
        pw = crc16_mul(pw, pw);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) crc ^= __shfl_xor_sync(0xffffffffu, crc, d);
    if (lane == 0) S.crc[wid] = crc;
    __syncthreads();
    if (t == 0) {
        unsigned all = 0;
        for (int v = 0; v < FT / 32; v++) all ^= S.crc[v];
        put_bits(S.buf, 8 * body, all, 16);
    }
    __syncthreads();
    uint8_t* dst = out + off[blockIdx.x];
    for (int e = t; e < F; e += FT) dst[e] = bytes[e];
}

// The frame header's 4-bit sample-rate code of an output rate (13: a 16-bit field in Hz follows), or -1.
int rate_code(long long rate) {
    switch (rate) {
        case 8000: return 4;
        case 11025: return 13;
        case 16000: return 5;
        case 22050: return 6;
        case 24000: return 7;
        case 32000: return 8;
        case 44100: return 9;
        case 48000: return 10;
        default: return -1;
    }
}

// `fLaC`, the STREAMINFO block header (last, type 0, 34 bytes) and STREAMINFO; the MD5 is left zero ("not computed").
void stream_info(uint8_t* h, long long rate, long long total, long long min_frame, long long max_frame) {
    memset(h, 0, FLAC_STREAMINFO_BYTES);
    memcpy(h, "fLaC", 4);
    h[4] = 0x80; h[5] = 0; h[6] = 0; h[7] = 34;
    uint8_t* s = h + 8;
    s[0] = FB >> 8; s[1] = FB & 0xFF; s[2] = FB >> 8; s[3] = FB & 0xFF;
    for (int i = 0; i < 3; i++) {
        s[4 + i] = (uint8_t)(min_frame >> (16 - 8 * i));
        s[7 + i] = (uint8_t)(max_frame >> (16 - 8 * i));
    }
    const unsigned long long v = ((unsigned long long)rate << 44) | (0ull << 41) | (15ull << 36) |
                                 ((unsigned long long)total & ((1ull << 36) - 1));
    for (int i = 0; i < 8; i++) s[10 + i] = (uint8_t)(v >> (56 - 8 * i));
}

size_t smem_bytes() { return (sizeof(Smem) + 15) & ~size_t(15); }

// Stream-ordered device scratch, returned to the pool when the encode ends, however it ends.
struct Scratch {
    cudaStream_t st;
    std::vector<void*> ptrs;
    void* get(size_t bytes) {
        void* p = nullptr;
        SB_CUDA(cudaMallocAsync(&p, bytes ? bytes : 16, st));
        ptrs.push_back(p);
        return p;
    }
    ~Scratch() { for (void* p : ptrs) cudaFreeAsync(p, st); }
};

}  // namespace

bool flac_rate_supported(long long rate) { return rate_code(rate) >= 0; }

void flac_encode(const short* d_x, const std::vector<FlacStream>& streams, cudaStream_t st, uint8_t** outs,
                 size_t* lens) {
    for (const FlacStream& s : streams)
        if (!flac_rate_supported(s.rate))
            throw Error(19, "FLAC: sample rate " + std::to_string(s.rate) + " Hz is not one of the output rates");
    const int S = (int)streams.size();
    std::vector<FrameIn> frames;
    std::vector<StreamRange> ranges(S);
    for (int s = 0; s < S; s++) {
        ranges[s].first = (int)frames.size();
        for (long long o = 0, k = 0; o < streams[s].n; o += FB, k++)
            frames.push_back(FrameIn{streams[s].off + o, (int)std::min<long long>(FB, streams[s].n - o), (int)k,
                                     rate_code(streams[s].rate), (int)streams[s].rate});
        ranges[s].count = (int)frames.size() - ranges[s].first;
    }
    const int F = (int)frames.size();
    std::vector<long long> stats(4 * (size_t)S, 0);
    Scratch sc{st, {}};
    uint8_t* d_out = nullptr;
    if (F > 0) {
        FrameIn* d_frames = static_cast<FrameIn*>(sc.get(sizeof(FrameIn) * F));
        Choice* d_ch = static_cast<Choice*>(sc.get(sizeof(Choice) * F));
        long long* d_off = static_cast<long long*>(sc.get(sizeof(long long) * F));
        StreamRange* d_rng = static_cast<StreamRange*>(sc.get(sizeof(StreamRange) * S));
        long long* d_stats = static_cast<long long*>(sc.get(sizeof(long long) * 4 * S));
        // pageable sources: each call returns once its bytes are staged
        SB_CUDA(cudaMemcpyAsync(d_frames, frames.data(), sizeof(FrameIn) * F, cudaMemcpyHostToDevice, st));
        SB_CUDA(cudaMemcpyAsync(d_rng, ranges.data(), sizeof(StreamRange) * S, cudaMemcpyHostToDevice, st));
        static PerDeviceOnce once;
        once.run([] {
            cudaFuncSetAttribute(flac_analyze_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes());
            cudaFuncSetAttribute(flac_pack_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes());
        });
        launch_pdl(flac_analyze_kernel, dim3(F), dim3(FT), smem_bytes(), st, d_x, d_frames, d_ch);
        launch_pdl(flac_layout_kernel, dim3(1), dim3(1024), 0, st, d_ch, F, d_rng, S, d_off, d_stats);
        g_launch_count += 2;
        SB_CUDA(cudaGetLastError());
        // the size table, then only the compressed bytes
        SB_CUDA(cudaMemcpyAsync(stats.data(), d_stats, sizeof(long long) * 4 * S, cudaMemcpyDeviceToHost, st));
        SB_CUDA(cudaStreamSynchronize(st));
        long long total = 0;
        for (int s = 0; s < S; s++) total += stats[4 * (size_t)s + 1];
        d_out = static_cast<uint8_t*>(sc.get((size_t)total));
        launch_pdl(flac_pack_kernel, dim3(F), dim3(FT), smem_bytes(), st, d_x, d_frames, d_ch, d_off, d_out);
        g_launch_count++;
        SB_CUDA(cudaGetLastError());
    }
    for (int s = 0; s < S; s++) { outs[s] = nullptr; lens[s] = 0; }
    try {
        for (int s = 0; s < S; s++) {
            const long long* q = &stats[4 * (size_t)s];
            const size_t len = FLAC_STREAMINFO_BYTES + (size_t)q[1];
            outs[s] = static_cast<uint8_t*>(malloc(len + 1));
            if (!outs[s]) throw Error(19, "FLAC: out of host memory");
            lens[s] = len;
            stream_info(outs[s], streams[s].rate, streams[s].n, q[2], q[3]);
            if (q[1] > 0)
                SB_CUDA(cudaMemcpyAsync(outs[s] + FLAC_STREAMINFO_BYTES, d_out + q[0], (size_t)q[1],
                                        cudaMemcpyDeviceToHost, st));
        }
        SB_CUDA(cudaStreamSynchronize(st));
    } catch (...) {
        for (int s = 0; s < S; s++) { free(outs[s]); outs[s] = nullptr; lens[s] = 0; }
        throw;
    }
}

}  // namespace sb200
