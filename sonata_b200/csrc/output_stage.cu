// The waveform output stage: what runs after the decoder, in this order: prosody (the stretch and the pitch stage), the
// formant stage, the volume stage, the break stage, resampling, the watermark, and loudness in place on what those
// leave.  Jobs, chunk passes and the
// test hooks plan, carve and launch it here only, so they run the same launches.
#include "engine.h"
#include <algorithm>
#include <cmath>

namespace sb200 {

void ResamplePlan::add(const ResampleFilter* f, long long n_in, const Resampler* r, bool last) {
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

void MeterPlan::add(int k, const LoudnessStream& s, long long samples, long long completes) {
    chunks.push_back(k); n.push_back(samples);
    win_off.push_back(win_total); step_off.push_back(steps_total); steps.push_back(completes);
    win_total += s.samples - s.steps * s.d.S + samples;
    steps_total += completes;
}

OutputPlan plan_job_output(Job& j, int hop, const std::vector<int>& cum, std::vector<long long>& bounds) {
    OutputPlan o;
    const size_t B = j.B;
    const std::vector<FrameSeg>& fs = j.frames.fsegs;
    const bool audio = !j.encode_only;
    // prosody: every utterance's decoder waveform, with its ratios or NaN, or with a contour planned from its ids' ends
    ProsodyPlan& pp = o.pp;
    bounds.clear();
    if (audio && j.contour.empty() && !j.pitch.empty()) {
        for (size_t b = 0; b < B; b++) {
            const long long n = (long long)fs[b].len * hop;
            pp.add(prosody_shape(j.v->sample_rate, n, j.pitch[b], j.tempo[b]), fs[b].out_off, n);
        }
    } else if (audio && !j.contour.empty()) {
        bounds.resize(j.ids.size());
        std::vector<long long> ends;
        std::vector<ContourPiece> pieces;
        for (size_t b = 0; b < B; b++) {
            const long long n = (long long)fs[b].len * hop;
            const size_t n_ids = j.offs[b + 1] - j.offs[b];
            ends.resize(n_ids);
            for (size_t i = 0; i < n_ids; i++) ends[i] = (long long)cum[j.xsegs[b].off + i] * hop;
            const float* r = j.contour.data() + j.offs[b];
            const bool has = std::any_of(r, r + n_ids, [](float v) { return !std::isnan(v) && v != 1.f; });
            const float pitch = j.pitch.empty() ? NAN : j.pitch[b], tempo = j.tempo.empty() ? NAN : j.tempo[b];
            const ProsodyShape sh = prosody_contour_plan(j.v->sample_rate, n, ends.data(), has ? r : nullptr, n_ids,
                                                         pitch, tempo, pieces, bounds.data() + j.offs[b]);
            pp.add(sh, fs[b].out_off, n, &pieces);
        }
    }
    // formants: each asking utterance's output of the pitch stage (or its decoder waveform), with its pitch ratio or
    // contour, in that stage's layout; the utterances that do not ask are copied into it
    if (audio && !j.formant.empty()) {
        FormantPlan& fp = o.fp;
        fp.total = pp.segs.empty() ? j.frames.total_samples : pp.y_total;
        for (size_t b = 0; b < B; b++) {
            long long in_off = fs[b].out_off, n = (long long)fs[b].len * hop;
            double ratio = 1.0;
            int c_off = 0, c_n = 0;
            if (!pp.segs.empty()) {
                const ProsodySeg& g = pp.segs[b];
                in_off = g.y_off; n = g.n2; ratio = g.p; c_off = g.c_off; c_n = g.c_n;
            }
            if (formant_asks(n, j.formant[b], ratio, pp.pieces.data() + c_off, c_n))
                fp.add(j.v->sample_rate, in_off, n, j.formant[b], ratio, c_off, c_n);
            else
                fp.copy(in_off, n);
        }
        if (fp.segs.empty()) fp = FormantPlan();
    }
    // each id's delivered end before any pause, which the volume and break stages share: the contour's bounds, or
    // those the utterance's ratios give
    if (audio && bounds.empty() && (!j.volume.empty() || !j.breaks.empty())) {
        bounds.resize(j.ids.size());
        std::vector<long long> ends;
        std::vector<ContourPiece> unused;
        for (size_t b = 0; b < B; b++) {
            const size_t n_ids = j.offs[b + 1] - j.offs[b];
            ends.resize(n_ids);
            for (size_t i = 0; i < n_ids; i++) ends[i] = (long long)cum[j.xsegs[b].off + i] * hop;
            prosody_contour_plan(j.v->sample_rate, (long long)fs[b].len * hop, ends.data(), nullptr, n_ids,
                                 j.pitch.empty() ? NAN : j.pitch[b], j.tempo.empty() ? NAN : j.tempo[b], unused,
                                 bounds.data() + j.offs[b]);
        }
    }
    // where each utterance is, and how long, after the stages before volume (the formant stage keeps their layout)
    const auto at = [&](size_t b) { return pp.segs.empty() ? fs[b].out_off : pp.segs[b].y_off; };
    const auto n2_of = [&](size_t b) { return pp.segs.empty() ? (long long)fs[b].len * hop : pp.segs[b].n2; };
    // volume: each asking utterance in place, its pieces over its ids' delivered ends
    if (audio && !j.volume.empty()) {
        for (size_t b = 0; b < B; b++) {
            const size_t n_ids = j.offs[b + 1] - j.offs[b];
            const float* lv = j.volume.data() + j.offs[b];
            if (!std::any_of(lv, lv + n_ids, [](float v) { return !std::isnan(v) && v != 0.f; })) continue;
            const std::vector<VolumePiece> pc = volume_pieces(bounds.data() + j.offs[b], lv, n_ids, n2_of(b));
            if (!pc.empty()) o.vp.add(at(b), n2_of(b), 0, volume_half(j.v->sample_rate), pc);
        }
    }
    // breaks: when any utterance asks, every utterance into the stage's own output, back to back (one that does not
    // ask is copied), and its ends moved past the pauses before them
    if (audio && !j.breaks.empty()) {
        std::vector<std::vector<BreakPiece>> bk(B);
        bool any = false;
        for (size_t b = 0; b < B; b++) {
            const size_t n_ids = j.offs[b + 1] - j.offs[b];
            bk[b] = break_plan(bounds.data() + j.offs[b], j.breaks.data() + j.offs[b], n_ids, n2_of(b),
                               j.v->sample_rate, "utterance " + std::to_string(b) + ": ");
            any |= !bk[b].empty();
        }
        if (any)
            for (size_t b = 0; b < B; b++) {
                const long long n2 = n2_of(b), d = bk[b].empty() ? 0 : bk[b].back().D;
                o.bp.add(at(b), n2, 0, 0, n2 + d, volume_half(j.v->sample_rate), bk[b]);
                for (size_t i = j.offs[b]; i < j.offs[b + 1]; i++) bounds[i] += break_shift(bk[b], bounds[i]);
            }
    }
    // what the job hands out: the frame layout itself, the prosody output (the formant stage keeps its layout), the
    // break output, or with output rates one resampled segment per utterance at its rate, back to back
    j.osr.assign(B, j.v->sample_rate);
    const BreakPlan& bp = o.bp;
    if (j.out_rates.empty() || !audio) {
        j.osegs = fs; j.out_hop = hop; j.out_total = j.frames.total_samples;
        if (!bp.segs.empty()) {
            for (size_t b = 0; b < B; b++) j.osegs[b] = FrameSeg{0, (int)bp.segs[b].n, 0, 0, bp.y_off[b]};
            j.out_hop = 1; j.out_total = bp.total;
        } else if (!pp.segs.empty()) {
            for (size_t b = 0; b < B; b++) j.osegs[b] = FrameSeg{0, (int)pp.segs[b].n2, 0, 0, pp.segs[b].y_off};
            j.out_hop = 1; j.out_total = pp.y_total;
        }
    } else {
        j.osegs.assign(B, FrameSeg{});
        for (size_t b = 0; b < B; b++) {
            const ResampleFilter* f = nullptr;
            if (j.out_rates[b]) {
                j.osr[b] = j.out_rates[b];
                f = &voice_resampler(*j.v, j.out_rates[b], "utterance " + std::to_string(b) + ": ");
            }
            o.rp.add(f, bp.segs.empty() ? n2_of(b) : bp.segs[b].n);
            j.osegs[b] = FrameSeg{0, (int)o.rp.segs[b].n_out, 0, 0, o.rp.segs[b].out_off};
        }
        j.out_hop = 1; j.out_total = o.rp.total;
    }
    // watermark: a marked voice's every utterance as the job hands it out, at its rate, into the stage's own output at
    // the same offsets
    if (audio && j.wm_on) {
        for (size_t b = 0; b < B; b++)
            o.wp.add(j.wm, j.osegs[b].out_off, (long long)j.osegs[b].len * j.out_hop, j.osr[b]);
        o.wp.total = j.out_total;
    }
    // loudness: every utterance as the job hands it out, at its rate, with its target or NaN
    if (audio && !j.loud_target.empty()) {
        LoudnessPlan& lp = o.lp;
        lp.segs.resize(B);
        for (size_t b = 0; b < B; b++) {
            LoudSeg& s = lp.segs[b];
            loudness_design(j.osr[b], s);
            s.off = j.osegs[b].out_off;
            s.n = (long long)j.osegs[b].len * j.out_hop;
            s.c0 = lp.chunks;
            s.target = j.loud_target[b];
            lp.chunks += (s.n + s.S - 1) / s.S;
        }
    }
    return o;
}

OutputPlan plan_chunk_output(const std::vector<ChunkSpec>& chunks, const std::vector<long long>& n_in, bool resample) {
    OutputPlan o;
    const size_t n = chunks.size();
    o.chunks = chunks;
    o.steps.resize(n); o.fsteps.resize(n); o.warp_of.assign(n, -1);
    o.n_res = n_in;
    for (size_t k = 0; k < n; k++) {
        const ChunkSpec& c = chunks[k];
        if (c.ps) {
            o.steps[k] = prosody_stream_step(*c.ps, n_in[k], c.last != 0);
            if (prosody_stream_warps(*c.ps)) {
                o.pp.add_stream(*c.ps, o.steps[k]);
                o.warp_of[k] = (int)o.warped.size();
                o.warped.push_back((int)k);
            }
            o.n_res[k] = o.steps[k].j1 - o.steps[k].j0;
            if (c.ps->fm) {
                o.fsteps[k] = formant_stream_step(*c.ps, o.steps[k].next.emitted, c.last != 0);
                o.fp.add_stream(*c.ps, o.fsteps[k]);
                o.formed.push_back((int)k);
                o.n_res[k] = o.fsteps[k].e1 - o.fsteps[k].e0;
            }
            if (!c.ps->vol.empty()) {
                // what the stages before it emit, at its delivered positions
                o.vp.add((long long)k, o.n_res[k], c.ps->fm ? o.fsteps[k].e0 : o.steps[k].j0, volume_half(c.ps->rate),
                         c.ps->vol, c.ps->vol_d);
                o.vp.y_off.push_back(o.vp.total);
                o.vp.total += o.n_res[k];
            }
            if (!c.ps->brk.empty()) {
                // the inputs [J0, J1) it receives, and every output up to O(J1) = J1 + the pauses at or before J1
                const ProsodyStream& w = *c.ps;
                const long long J1 = w.brk_in + o.n_res[k];
                if (J1 > w.brk_n2 || (c.last && J1 != w.brk_n2))
                    throw Error(19, "internal: a prosody stream with breaks would " + std::string(c.last ? "end" : "go on") +
                                        " after " + std::to_string(J1) + " inputs, not its " + std::to_string(w.brk_n2));
                const long long n_out = J1 + break_shift(w.brk, J1) - w.brk_out;
                o.bp.add((long long)k, o.n_res[k], w.brk_in, w.brk_out, n_out, volume_half(w.rate), w.brk, w.brk_d);
                o.n_res[k] = n_out;
            }
        }
        if (resample) o.rp.add(c.rs ? &c.rs->f : nullptr, o.n_res[k], c.rs, c.last != 0);
    }
    // watermark: when some chunk's stream marks, every chunk of the pass at its delivered rate, a marked one as its
    // stream emits it and the others copied, back to back
    if (resample && std::any_of(chunks.begin(), chunks.end(), [](const ChunkSpec& c) { return c.ws != nullptr; }))
        for (size_t k = 0; k < n; k++)
            o.wp.add_chunk(chunks[k].ws, o.rp.segs[k].out_off, o.rp.segs[k].n_out, chunks[k].last != 0);
    for (size_t k = 0; k < n; k++)
        if (const LoudnessStream* m = chunks[k].ls) {
            const long long d = !o.wp.segs.empty() ? o.wp.segs[k].n : resample ? o.rp.segs[k].n_out : o.n_res[k];
            o.mp.add((int)k, *m, d, loudness_stream_steps(*m, d, "chunk " + std::to_string(k) + ": "));
        }
    return o;
}

void OutputBufs::carve(Arena& dev, Arena& pin, const OutputPlan& p, long long in_total, float* d_out) {
    *this = OutputBufs();
    const ProsodyPlan& pp = p.pp;
    const FormantPlan& fp = p.fp;
    if (const size_t n = p.wp.segs.size()) {
        // the watermark is the last stage that writes: into d_out, and every stage before it into the pass's own
        wsegs.carve(dev, pin, n);
        if (p.streams()) { wosegs.carve(dev, pin, n); wposts.carve(dev, pin, n); }
        wy = d_out ? d_out : dev.get<float>((size_t)p.wp.total + 4);
        d_out = nullptr;
    }
    if (const size_t n = pp.segs.size()) {
        psegs.carve(dev, pin, n);
        if (!pp.pieces.empty()) pieces.carve(dev, pin, pp.pieces.size());     // a stream's table is its own
        if (pp.contour) apos = dev.get<long long>((size_t)pp.d_total);
        if (p.streams()) {
            pcarry.carve(dev, pin, n);
            px = dev.get<float>((size_t)pp.in_total + 4);
        } else {
            posegs.carve(dev, pin, n);
        }
        offsets = pp.d_total ? dev.get<int>((size_t)pp.d_total) : nullptr;
        ps = pp.s_total ? dev.get<float>((size_t)pp.s_total + 4) : nullptr;
    }
    if (const size_t n = fp.segs.size()) {
        fsegs.carve(dev, pin, n);
        if (p.streams()) {
            fcarry.carve(dev, pin, n);
            fwin = dev.get<float>((size_t)fp.in_total + 4);
        }
    }
    if (const size_t n = p.vp.segs.size()) {
        vsegs.carve(dev, pin, n);
        if (!p.vp.pieces.empty()) vpieces.carve(dev, pin, p.vp.pieces.size());
    }
    if (const size_t n = p.bp.segs.size()) {
        bsegs.carve(dev, pin, n);
        if (!p.bp.pieces.empty()) bpieces.carve(dev, pin, p.bp.pieces.size());
        if (!p.streams()) bosegs.carve(dev, pin, n);
    }
    if (p.streams() && (!pp.segs.empty() || !fp.segs.empty() || !p.vp.segs.empty() || !p.bp.segs.empty())) {
        rin.carve(dev, pin, p.chunks.size());
        rpost.carve(dev, pin, p.chunks.size());
    }
    if (const size_t n = p.rp.segs.size()) {
        rsegs.carve(dev, pin, n); rposts.carve(dev, pin, n); rosegs.carve(dev, pin, n);
    }
    if (const size_t n = p.lp.segs.size()) {
        lsegs.carve(dev, pin, n);
        lscratch = dev.get<double>((size_t)LD_SCRATCH * std::max<long long>(p.lp.chunks, 1));
        lufs.carve(dev, pin, n); gain.carve(dev, pin, n);
    }
    if (const size_t m = p.mp.chunks.size()) {
        const size_t steps = (size_t)std::max<long long>(p.mp.steps_total, 1);
        msegs.carve(dev, pin, m);
        mwin = dev.get<float>((size_t)p.mp.win_total + 4);
        me = dev.get<double>(8 * steps);
        mlufs.carve(dev, pin, steps); mgains.carve(dev, pin, steps); mclip.carve(dev, pin, m);
    }
    const bool staged = !pp.segs.empty() || !fp.segs.empty() || !p.bp.segs.empty() || !p.rp.segs.empty();
    in = staged || !d_out ? dev.get<float>((size_t)(in_total + pp.y_total + fp.total + p.vp.total + p.bp.total) + 4)
                          : d_out;
    py = in + in_total;
    fy = py + pp.y_total;
    vy = fy + fp.total;
    by = vy + p.vp.total;
    if (!p.rp.segs.empty()) ry = d_out ? d_out : dev.get<float>((size_t)p.rp.total + 4);
    else if (d_out && !p.bp.segs.empty()) by = d_out;
    else if (d_out && !fp.segs.empty()) fy = d_out;
    else if (d_out && !pp.segs.empty()) py = d_out;
}

void OutputBufs::upload(const OutputPlan& p, int hop, const FrameSeg* in_segs, const PcmPost* in_posts,
                        cudaStream_t st) {
    const ProsodyPlan& pp = p.pp;
    const FormantPlan& fp = p.fp;
    const size_t n = p.chunks.size();
    if (psegs.d) {
        std::copy(pp.segs.begin(), pp.segs.end(), psegs.h);
        psegs.upload(st);
        if (posegs.d) {
            for (size_t k = 0; k < pp.segs.size(); k++) posegs.h[k] = FrameSeg{0, (int)pp.segs[k].n2, 0, 0, pp.segs[k].y_off};
            posegs.upload(st);
        }
        if (pieces.d) {
            std::copy(pp.pieces.begin(), pp.pieces.end(), pieces.h);
            pieces.upload(st);
        }
        if (pcarry.d) {
            for (size_t q = 0; q < p.warped.size(); q++) {
                const int k = p.warped[q];
                pcarry.h[q] = prosody_carry(*p.chunks[k].ps, p.steps[k], k);
            }
            pcarry.upload(st);
        }
    }
    if (fsegs.d) {
        std::copy(fp.segs.begin(), fp.segs.end(), fsegs.h);
        fsegs.upload(st);
        if (fcarry.d) {
            for (size_t q = 0; q < p.formed.size(); q++) {
                const int k = p.formed[q], w = p.warp_of[k];
                fcarry.h[q] = formant_carry(*p.chunks[k].ps, p.fsteps[k], k, w < 0 ? nullptr : py + pp.segs[w].y_off);
            }
            fcarry.upload(st);
        }
    }
    // chunk passes: where each chunk's samples are after the stages, its input or its last stage's output
    std::vector<float*> at(n);
    for (size_t k = 0; k < n; k++) at[k] = in + in_segs[k].out_off;
    for (size_t q = 0; q < p.warped.size(); q++) at[p.warped[q]] = py + pp.segs[q].y_off;
    for (size_t q = 0; q < p.formed.size(); q++) at[p.formed[q]] = fy + fp.segs[q].y_off;
    // a job's utterances are in the last stage's output; a chunk is where the stages before it leave it (without one,
    // read through its post-path)
    float* base = !fp.segs.empty() ? fy : !pp.segs.empty() ? py : in;
    std::vector<char> staged(n, 0);
    for (int k : p.warped) staged[k] = 1;
    for (int k : p.formed) staged[k] = 1;
    if (vsegs.d) {
        // a job's utterances scaled in place; a chunk written to vy
        const VolumePlan& vp = p.vp;
        for (size_t q = 0; q < vp.segs.size(); q++) {
            VolumeSeg g = vp.segs[q];
            if (p.streams()) {
                const size_t k = (size_t)vp.at[q];
                g.chunk = (int)k;
                g.x = staged[k] ? at[k] : nullptr;
                g.y = at[k] = vy + vp.y_off[q];
                staged[k] = 1;
            } else {
                g.y = base + vp.at[q];
                g.x = g.y;
            }
            if (vp.p_off[q] >= 0) g.pc = vpieces.d + vp.p_off[q];
            vsegs.h[q] = g;
        }
        vsegs.upload(st);
        if (vpieces.d) {
            std::copy(vp.pieces.begin(), vp.pieces.end(), vpieces.h);
            vpieces.upload(st);
        }
    }
    if (bsegs.d) {
        // every segment written to by, longer by its pauses
        const BreakPlan& bp = p.bp;
        for (size_t q = 0; q < bp.segs.size(); q++) {
            BreakSeg g = bp.segs[q];
            g.y = by + bp.y_off[q];
            if (p.streams()) {
                const size_t k = (size_t)bp.at[q];
                g.chunk = (int)k;
                g.x = staged[k] ? at[k] : nullptr;
                at[k] = g.y;
            } else {
                g.x = base + bp.at[q];
                bosegs.h[q] = FrameSeg{0, (int)g.n, 0, 0, bp.y_off[q]};
            }
            if (bp.p_off[q] >= 0) g.bk = bpieces.d + bp.p_off[q];
            bsegs.h[q] = g;
        }
        bsegs.upload(st);
        if (bosegs.d) bosegs.upload(st);
        if (bpieces.d) {
            std::copy(bp.pieces.begin(), bp.pieces.end(), bpieces.h);
            bpieces.upload(st);
        }
    }
    if (rin.d) {
        // a chunk a stage ran on is read from that stage's output: its m samples as a segment of ceil(m / hop) frames
        // less a trim, with no post-path of its own
        for (size_t k = 0; k < n; k++) {
            rin.h[k] = in_segs[k];
            rpost.h[k] = in_posts ? in_posts[k] : PcmPost();
            if (!p.chunks[k].ps) continue;
            const long long m = p.n_res[k], frames = (m + hop - 1) / hop;
            rin.h[k] = FrameSeg{0, (int)frames, 0, 0, at[k] - in};
            rpost.h[k] = PcmPost();
            rpost.h[k].trim_hi = frames * hop - m;
        }
        rin.upload(st);
        rpost.upload(st);
    }
    if (rsegs.d) {
        // identity posts, for a launch whose input has no post-path or for the PCM conversion of its output
        for (size_t k = 0; k < p.rp.segs.size(); k++) {
            rsegs.h[k] = p.rp.segs[k];
            rposts.h[k] = PcmPost();
            if (!p.out_gain.empty()) rposts.h[k].gain = p.out_gain[k];
            if (!p.fixed_scale.empty()) rposts.h[k].fixed_scale = p.fixed_scale[k];
            rosegs.h[k] = FrameSeg{0, (int)p.rp.segs[k].n_out, 0, 0, p.rp.segs[k].out_off};
        }
        rsegs.upload(st); rposts.upload(st); rosegs.upload(st);
    }
    if (wsegs.d) {
        std::copy(p.wp.segs.begin(), p.wp.segs.end(), wsegs.h);
        for (size_t k = 0; wosegs.d && k < p.wp.segs.size(); k++) {
            // a stream's held samples and carried S, read from one set and written to the other
            if (const WatermarkStream* w = p.chunks[k].ws) {
                WatermarkSeg& g = wsegs.h[k];
                g.hold = w->hold[w->cur]; g.hold_out = w->hold[1 - w->cur];
                g.s_in = w->out > 0 ? w->s[w->cur] : nullptr; g.s_out = w->s[1 - w->cur];
            }
            wosegs.h[k] = FrameSeg{0, (int)p.wp.segs[k].n, 0, 0, p.wp.segs[k].y_off};
            wposts.h[k] = rposts.h[k];
        }
        wsegs.upload(st);
        if (wosegs.d) { wosegs.upload(st); wposts.upload(st); }
    }
    if (lsegs.d) {
        std::copy(p.lp.segs.begin(), p.lp.segs.end(), lsegs.h);
        lsegs.upload(st);
    }
    if (msegs.d) {
        // a metered chunk is what the resample launch delivers for it, or without one its samples after the stages
        const MeterPlan& mp = p.mp;
        for (size_t q = 0; q < mp.chunks.size(); q++) {
            const int k = mp.chunks[q];
            float* y = wy ? wy + p.wp.segs[k].y_off : ry ? ry + p.rp.segs[k].out_off : at[k];
            LoudStreamSeg g = loudness_stream_seg(*p.chunks[k].ls, y, mp.n[q], p.chunks[k].gain);
            g.win = mwin + mp.win_off[q]; g.e = me + 8 * mp.step_off[q];
            g.lufs = mlufs.d + mp.step_off[q]; g.gains = mgains.d + mp.step_off[q]; g.clipped = mclip.d + q;
            msegs.h[q] = g;
        }
        msegs.upload(st);
    }
}

Wave run_output_stage(Profile& prof, const OutputPlan& p, const OutputBufs& b, Wave in, cudaStream_t st) {
    const bool streams = p.streams();
    // a chunk pass's later stages read every chunk from one table: the stage outputs of its staged chunks, the input
    // of the others
    const Wave restaged{in.buf, b.rin.d, b.rpost.d, in.hop};
    Wave cur = in;
    const ProsodyPlan& pp = p.pp;
    if (const int n = (int)pp.segs.size()) {
        prof.begin("stretch");
        if (streams) {
            launch_prosody_stream_stretch(pp, b.psegs.d, b.pcarry.d, in.buf, in.segs, in.posts, in.hop, b.px, b.ps,
                                          b.offsets, b.py, st, b.apos);
            prof.count(pp.stretch_flops, pp.stretch_bytes, 2 + (pp.smem_ints ? 1 : 0) + (pp.max_ola ? 1 : 0));
        } else {
            // the offset chain and the overlap-add, which also copies the segments without a ratio
            if (pp.smem_ints)
                launch_prosody_offsets(in.buf, b.psegs.d, n, pp.smem_ints, b.offsets, st, b.pieces.d, b.apos);
            launch_prosody_ola(in.buf, b.psegs.d, n, pp.max_ola, b.offsets, b.ps, b.py, st, b.apos);
            prof.count(pp.stretch_flops, pp.stretch_bytes, pp.smem_ints ? 2 : 1);
        }
        prof.end();
        if (pp.max_pitch) {
            prof.begin("pitch");
            launch_prosody_pitch(streams ? b.px : in.buf, b.ps, b.psegs.d, n, pp.max_pitch, b.py, st, b.pieces.d);
            prof.count(pp.pitch_flops, pp.pitch_bytes);
            prof.end();
        }
        cur = streams ? restaged : Wave{b.py, b.posegs.d, nullptr, 1};
    }
    const FormantPlan& fp = p.fp;
    if (!fp.segs.empty()) {
        prof.begin("formant");
        if (streams) {
            launch_formant_stream(fp, b.fsegs.d, b.fcarry.d, in.buf, in.segs, in.posts, in.hop, b.fwin, b.fy, st);
            prof.count(fp.flops, fp.bytes, fp.max_runs ? 2 : 1);
        } else {
            for (const auto& c : fp.copies)
                SB_CUDA(cudaMemcpyAsync(b.fy + c.first, cur.buf + c.first, (size_t)c.second * 4, cudaMemcpyDeviceToDevice,
                                        st));
            launch_formant(cur.buf, b.fsegs.d, (int)fp.segs.size(), fp.max_runs, b.pieces.d, b.fy, st);
            prof.count(fp.flops, fp.bytes);
        }
        prof.end();
        cur = streams ? restaged : Wave{b.fy, cur.segs, cur.posts, cur.hop};
    }
    const VolumePlan& vp = p.vp;
    if (!vp.segs.empty()) {
        prof.begin("volume");
        launch_volume(b.vsegs.d, (int)vp.segs.size(), vp.max_n, in.buf, in.segs, in.posts, in.hop, st);
        prof.count(0, vp.bytes);
        prof.end();
        if (streams) cur = restaged;
    }
    const BreakPlan& bp = p.bp;
    if (!bp.segs.empty()) {
        prof.begin("break");
        launch_breaks(b.bsegs.d, (int)bp.segs.size(), bp.max_n, in.buf, in.segs, in.posts, in.hop, st);
        prof.count(0, bp.bytes);
        prof.end();
        cur = streams ? restaged : Wave{b.by, b.bosegs.d, nullptr, 1};
    }
    const ResamplePlan& rp = p.rp;
    if (!rp.segs.empty()) {
        prof.begin("resample");
        launch_resample(cur.buf, cur.segs, cur.posts ? cur.posts : b.rposts.d, cur.hop, b.rsegs.d, (int)rp.segs.size(),
                        rp.max_out, rp.smem, b.ry, st);
        prof.count(rp.flops, rp.bytes);
        prof.end();
        cur = Wave{b.ry, b.rosegs.d, b.rposts.d, 1};
    }
    const WatermarkPlan& wp = p.wp;
    if (!wp.segs.empty()) {
        // segments are read plainly: a job's waves carry no post-path, or the resampler's identity one, and a chunk
        // pass's resampled output keeps its post-path (the gain of G.711, the fixed scale) for the conversion
        prof.begin("watermark");
        launch_watermark(wp, b.wsegs.d, cur.buf, b.wy, st);
        prof.count(0, wp.bytes);
        prof.end();
        if (streams) cur = Wave{b.wy, b.wosegs.d, b.wposts.d, 1};
        else cur.buf = b.wy;
    }
    if (!p.lp.segs.empty()) {
        // the samples read and, where a target scales them, written
        double samples = 0, scaled = 0;
        for (const LoudSeg& s : p.lp.segs) {
            samples += (double)s.n;
            if (!std::isnan(s.target)) scaled += (double)s.n;
        }
        prof.begin("loudness");
        launch_loudness(cur.buf, b.lsegs.d, (int)p.lp.segs.size(), b.lscratch, b.lufs.d, b.gain.d, st);
        prof.count(2.0 * 22.0 * samples, 4.0 * (samples + scaled));
        prof.end();
        b.lufs.download(st);
        b.gain.download(st);
    }
    if (const size_t m = p.mp.chunks.size()) {
        double window = 0, samples = 0;
        for (size_t q = 0; q < m; q++) {
            window += (double)(b.msegs.h[q].p + b.msegs.h[q].n);
            samples += (double)b.msegs.h[q].n;
        }
        prof.begin("loudness");
        launch_loudness_stream(b.msegs.d, (int)m, st);
        // the window filtered twice; read, staged, read again and written
        prof.count(2.0 * 22.0 * window, 4.0 * (3.0 * window + samples));
        prof.end();
        b.mlufs.download(st); b.mgains.download(st); b.mclip.download(st);
    }
    return cur;
}

void advance_streams(const OutputPlan& p, const OutputBufs& b, const Profile& prof) {
    const float stretch_ms = prof.ms("stretch"), pitch_ms = prof.ms("pitch"), formant_ms = prof.ms("formant"),
                volume_ms = prof.ms("volume"), break_ms = prof.ms("break"), loudness_ms = prof.ms("loudness");
    for (size_t k = 0; k < p.chunks.size(); k++) {
        const ChunkSpec& c = p.chunks[k];
        if (Resampler* r = c.rs) {
            const ResampleSeg& s = p.rp.segs[k];
            r->consumed = s.c + p.n_res[k];
            r->emitted = s.j0 + s.n_out;
            r->cur ^= 1;
            r->h = s.h_out;
            r->ended = c.last != 0;
        }
        if (ProsodyStream* w = c.ps) {
            if (w->fm) formant_stream_advance(*w, p.fsteps[k]);
            if (!w->brk.empty()) {
                // the inputs it took (what the stages before it emitted), and the outputs emitted for them
                w->brk_in = w->fm ? p.fsteps[k].e1 : p.steps[k].j1;
                w->brk_out += p.n_res[k];
            }
            prosody_stream_advance(*w, p.steps[k], c.last != 0);
            const bool warps = prosody_stream_warps(*w);
            w->last_ms[0] = warps ? stretch_ms : 0.f; w->last_ms[1] = warps ? pitch_ms : 0.f;
            w->last_fm_ms = w->fm ? formant_ms : 0.f;
            w->last_vol_ms = w->vol.empty() ? 0.f : volume_ms;
            w->last_brk_ms = w->brk.empty() ? 0.f : break_ms;
        }
    }
    const float watermark_ms = prof.ms("watermark");
    for (size_t k = 0; k < p.chunks.size() && !p.wp.segs.empty(); k++)
        if (WatermarkStream* w = p.chunks[k].ws) {
            const WatermarkSeg& g = p.wp.segs[k];
            w->in += g.m;
            w->out += g.n;
            w->cur ^= 1;
            w->ended = p.chunks[k].last != 0;
            w->last_ms = watermark_ms;
        }
    const MeterPlan& mp = p.mp;
    for (size_t q = 0; q < mp.chunks.size(); q++) {
        LoudnessStream* m = p.chunks[mp.chunks[q]].ls;
        loudness_stream_advance(*m, mp.n[q], b.mlufs.h + mp.step_off[q], b.mgains.h + mp.step_off[q], b.mclip.h[q]);
        m->last_ms = loudness_ms;
    }
}

}  // namespace sb200
