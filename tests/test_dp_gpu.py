"""GPU (-m gpu): the stochastic duration predictor stage by stage against float64 (tests/dp_reference.py), each stage from
the kernel's own captured inputs so that errors do not compound, and the spline and duration kernels at their edges
through the sb200_debug_spline / sb200_debug_durations hooks.  Run with -s to print the per-stage error tables."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import sonata_b200
from oracle import vits_oracle as vo
from sonata_b200 import PiperSynthesisConfig, _native as N, voicegen, workload
from sonata_b200.job import SynthesisJob

pytestmark = pytest.mark.gpu
INT_MAX = 2 ** 31 - 1
# segments shorter than the DDSConv receptive field (+-13 rows), gaps next to dilation 9, the 256-thread scan block
DP_LENS = (1, 2, 9, 13, 255, 256, 257, 513)
# z_p = m + eps exp(logs) noise_scale: expf (2 ulp), two products and the add
Z_ULP = 6
VOICES = {"medium": ("medium", 1, None), "high": ("high", 1, None), "medium_spk4_sid3": ("medium", 4, 3)}


def _ids(n, utt):
    return workload.synthetic_ids(n // 2 + 1, utt=utt)[:n]


def _fp32_dds(W32, p, h, a, g=None):
    x = torch.from_numpy(np.ascontiguousarray(np.asarray(h, dtype=np.float32).T[None]))
    gg = None if g is None else torch.from_numpy(np.ascontiguousarray(np.asarray(g, dtype=np.float32).T[None]))
    return vo._dds(W32, p, x, a, g=gg)[0].T.numpy()


def _dp_job(voice, noise_w, ls, lens=DP_LENS, eps_seed=0, noise_scale=0.0, eps_z=None):
    quality, nspk, sid = VOICES[voice]
    cfg = voicegen.write_voice(voicegen.default_voice_dir(), quality, n_speakers=nspk)
    m = sonata_b200.from_config_path(cfg, device=0)
    m.set_fallback_synthesis_config(PiperSynthesisConfig(sid, noise_scale, ls, noise_w))
    ids = [_ids(n, 500 + i) for i, n in enumerate(lens)]
    rng = np.random.default_rng(eps_seed)
    eps = [rng.standard_normal((n, 2)).astype(np.float32) for n in lens]
    job = SynthesisJob(m, ids, eps if noise_w else None, eps_z, debug=True)
    job.run()
    names = ["x", "stats", "logw", "dp.g"] + [f"dp.f{s}.{k}" for s in range(3) for k in ("in", "h", "h29", "out")]
    out = []
    frames = job.lengths()[0]
    for b in range(len(ids)):
        d = {k: job.debug_fetch(k, b) for k in names}
        d["cum"], d["y_len"], d["z_p"] = job.durations(b), frames[b], job.debug_fetch("z_p", b)
        d["eps"] = eps[b]
        out.append(d)
    job.close()
    m.close()
    return out


def _check_durations(u, ls, report):
    """cum == int64 cumsum of ceil(exp(float64(logw)) * ls), ids within 1e-6 relative of an integer exempt (and
    reported); y_len = max(sum, 1)."""
    w = np.exp(u["logw"][:, 0].astype(np.float64)) * float(np.float32(ls))
    wc = np.ceil(w)
    near = np.abs(w - np.rint(w)) <= 1e-6 * np.maximum(w, 1.0)
    got = np.diff(np.concatenate([[0], u["cum"].astype(np.int64)]))
    assert np.all((got == wc) | near), (np.nonzero((got != wc) & ~near)[0], got[:8], wc[:8])
    assert np.all(np.abs(got - wc)[near] <= 1)
    assert u["y_len"] == max(int(got.sum()), 1)
    report["near_int"] = report.get("near_int", 0) + int(near.sum())


@pytest.mark.parametrize("voice", list(VOICES))
def test_duration_predictor_stages_against_fp64(voice):
    """Per utterance of one batch (lengths DP_LENS) and noise_w in {0, 0.8, 4} (4 puts spline inputs past +-5):
    * dp.g and every flow's DDSConv output h against float64 from the captured x / flow input, within
      DP_MULT x the fp32 oracle's error on the same inputs + DP_FLOOR;
    * h29 against the float64 proj of the captured h at the 3xTF32 conv tolerance;
    * the spline: its conditioning column passes through bit for bit, each flow's output is the next one's input bit
      for bit, and the transformed column is within dp_reference.spline_error_bound of the float64 inverse of the
      captured h29 and input, element by element;
    * logw against (z0 - m0) exp(-logs0) of the last flow's output within LOGW_ULP ulp;
    * cum / y_len exactly against the float64 durations of the kernel's logw, for length_scale 1, 0.45 and 1.7;
    * z_p (noise_scale 0) an exact row gather of stats by cum; with eps_z injected (noise_scale 0.667, noise_w 0.8),
      within Z_ULP ulp of m + eps exp(logs) noise_scale."""
    import dp_reference as dr
    from conv_unit import TF_TOL
    quality, nspk, sid = VOICES[voice]
    t = voicegen.make_tensors(quality, n_speakers=nspk)
    W32 = vo.to_torch(t)
    a = vo.arch_of(W32)
    H = a["hidden"]
    I = a["inter"]
    m0, logs0 = dr.ea_params(t)
    rows, fails, durs = [], [], []
    for noise_w in (0.0, 0.8, 4.0):
        utts = _dp_job(voice, noise_w, 1.0)
        for n, u in zip(DP_LENS, utts):
            row = {"noise_w": noise_w, "T": n}
            x = u["x"]
            ref = dr.dp_cond(t, x, sid)
            xt = torch.from_numpy(np.ascontiguousarray(x.T[None]))
            hp = vo._conv(W32, "dp.pre", xt)
            if sid is not None:
                hp = hp + vo._conv(W32, "dp.cond", vo.speaker_embedding(W32, sid))
            g32 = vo._conv(W32, "dp.proj", vo._dds(W32, "dp.convs.", hp, a))[0].T.numpy()
            e, e32 = float(np.abs(u["dp.g"] - ref).max()), float(np.abs(g32 - ref).max())
            row.update(g=e, g32=e32)
            if e > dr.DP_MULT * e32 + dr.DP_FLOOR:
                fails.append(("dp.g", row))
            z_in = u["dp.f0.in"]
            assert np.array_equal(z_in, u["eps"] * np.float32(noise_w)) if noise_w else not z_in.any()
            sp_err, sp_ratio, sp_in_tails = 0.0, 0.0, 0
            for s in range(3):
                f = f"dp.f{s}."
                zin, h, h29, zout = u[f + "in"], u[f + "h"], u[f + "h29"], u[f + "out"]
                if s:
                    assert np.array_equal(zin, u[f"dp.f{s - 1}.out"]), (s, n)
                cc, tc = dr.flow_cols(s)
                href = dr.flow_h(t, s, zin, u["dp.g"])
                p = f"dp.flows.{dr.FLOWS[s]}."
                zc = torch.from_numpy(np.ascontiguousarray(zin[:, cc])).view(1, 1, -1)
                h32 = _fp32_dds(W32, p + "convs.", vo._conv(W32, p + "pre", zc)[0].T.numpy(), a, u["dp.g"])
                e, e32 = float(np.abs(h - href).max()), float(np.abs(h32 - href).max())
                row[f"h{s}"], row[f"h{s}_32"] = e, e32
                if e > dr.DP_MULT * e32 + dr.DP_FLOOR:
                    fails.append((f + "h", row))
                pref = dr.flow_h29(t, s, h)
                e29 = float(np.abs(h29[:, :29] - pref).max())
                row[f"h29_{s}"] = e29
                assert e29 < TF_TOL * max(1.0, float(np.abs(pref).max())), (s, n, e29)
                assert np.array_equal(zout[:, cc], zin[:, cc]), (s, n)
                assert np.isfinite(zout[:, tc]).all(), (s, n, zout[:, tc])
                uw, uh, ud = dr.spline_logits(h29, H)
                yin = zin[:, tc]
                sref, sbound = dr.spline_error_bound(yin, uw, uh, ud)
                serr = np.abs(zout[:, tc] - sref)
                sp_err = max(sp_err, float(serr.max()))
                sp_ratio = max(sp_ratio, float((serr / sbound).max()))
                if not np.all(serr <= sbound):
                    fails.append((f + "out", n, noise_w, float((serr / sbound).max())))
                sp_in_tails += int((np.abs(yin) > dr.TAIL).sum())
                tails = np.abs(yin) > dr.TAIL
                assert np.array_equal(zout[tails, tc], zin[tails, tc]), (s, n)
            row.update(spline=sp_err, spline_of_bound=sp_ratio, tails=sp_in_tails)
            lw_ref = dr.ea_inverse(u["dp.f2.out"][:, 0], m0, logs0)
            e_lw = np.abs(u["logw"][:, 0] - lw_ref)
            row["logw_ulp"] = float((e_lw / (2.0 ** -24 * np.maximum(np.abs(lw_ref), 2.0 ** -126))).max())
            assert np.all(e_lw <= dr.LOGW_ULP * 2.0 ** -24 * np.abs(lw_ref) + 1e-30), (n, row)
            _check_durations(u, 1.0, row)
            # z_p with noise_scale 0: frame j takes the stats row of the first id with cum > j
            tok = np.searchsorted(u["cum"], np.arange(u["y_len"]), side="right")
            assert tok.max() < n or u["cum"][-1] == 0
            assert np.array_equal(u["z_p"], u["stats"][np.minimum(tok, n - 1), :I]), n
            rows.append(row)
        if noise_w == 0.8:
            rng = np.random.default_rng(11)
            ez = [rng.standard_normal((u["y_len"], I)).astype(np.float32) for u in utts]
            for n, u, e, un in zip(DP_LENS, utts, ez, _dp_job(voice, noise_w, 1.0, noise_scale=0.667, eps_z=ez)):
                assert np.array_equal(un["cum"], u["cum"]), n
                tok = np.minimum(np.searchsorted(u["cum"], np.arange(u["y_len"]), side="right"), n - 1)
                mu, lg = u["stats"][tok, :I].astype(np.float64), u["stats"][tok, I:].astype(np.float64)
                noise = e.astype(np.float64) * np.exp(lg) * float(np.float32(0.667))
                zerr = np.abs(un["z_p"] - (mu + noise))
                assert np.all(zerr <= Z_ULP * 2.0 ** -24 * (np.abs(mu) + np.abs(noise)) + 1e-30), (n, float(zerr.max()))
        for ls in (0.45, 1.7):
            near = 0
            for n, u in zip(DP_LENS, _dp_job(voice, noise_w, ls)):
                r = {}
                _check_durations(u, ls, r)
                near += r["near_int"]
            durs.append(f"noise_w={noise_w} length_scale={ls}: {near} ids within 1e-6 of an integer (exempt)")
    print(voice, "\n" + "\n".join(" ".join(f"{k}={v:.3g}" if isinstance(v, float) else f"{k}={v}" for k, v in r.items())
                                  for r in rows) + "\n" + "\n".join(durs))
    assert not fails, fails


def _spline(h29, z, tcol, valid):
    h = np.ascontiguousarray(h29, dtype=np.float32)
    zz = np.ascontiguousarray(z, dtype=np.float32).copy()
    err = N.sb200_error()
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    rc = N.lib().sb200_debug_spline(0, fp(h), h.shape[1], fp(zz), zz.shape[0], tcol, valid, C.byref(err))
    assert rc == 0, C.string_at(err.message).decode() if err.message else rc
    return zz


def test_spline_kernel_edges(lib_built):
    """spline_kernel through sb200_debug_spline on the edge parameter sets of dp_reference.edge_params (all-zero, sigma
    1 / 3 / 10, saturated bins, softplus's linear branch, the minimum derivative, a narrow tall bin next to it) and the
    inputs of dp_reference.edge_inputs.  Outside [-5, 5] and for NaN the output is the input bit for bit.  Inside it is
    finite and within dp_reference.spline_error_bound of the float64 inverse, element by element, and monotone along the
    sorted inputs up to that bound.  The other column is untouched and rows past valid_rows come out 0.  On the host, the
    kernel's arithmetic before the discriminant was clamped (spline_fp32) meets negative discriminants on these inputs,
    where it would return NaN as the fp32 graph does; the unclamped kernel was not run on the device."""
    import dp_reference as dr
    rng = np.random.default_rng(7)
    worst = {}
    for name, uw, uh, ud in dr.edge_params(rng):
        _, _, ch = dr.spline_fp32(np.zeros(1, np.float32), uw[None], uh[None], ud[None])
        y = dr.edge_inputs(ch[0])
        n = len(y)
        h29 = np.zeros((n + 5, 32), dtype=np.float32)
        h29[:, :10], h29[:, 10:20], h29[:, 20:29] = uw, uh, ud
        ins = (y >= -5) & (y <= 5)
        rep = lambda p: np.repeat(p[None], int(ins.sum()), 0)
        ref, bound = dr.spline_error_bound(y[ins], rep(uw), rep(uh), rep(ud))
        for tcol in (0, 1):
            z = np.empty((n + 5, 2), dtype=np.float32)
            z[:n, tcol] = y
            z[n:, tcol] = 1.0
            z[:, 1 - tcol] = rng.standard_normal(n + 5).astype(np.float32)
            out = _spline(h29, z, tcol, n)
            assert np.array_equal(out[:, 1 - tcol], z[:, 1 - tcol]), name
            assert not out[n:, tcol].any(), name
            got = out[:n, tcol]
            assert np.array_equal(got[~ins].view(np.uint32), y[~ins].view(np.uint32)), name
            gi = got[ins].astype(np.float64)
            assert np.isfinite(gi).all(), (name, y[ins][~np.isfinite(gi)])
            err = np.abs(gi - ref)
            ratio = err / bound
            assert np.all(err <= bound), (name, float(ratio.max()), y[ins][np.argmax(ratio)])
            order = np.argsort(y[ins], kind="stable")
            g, bo = gi[order], bound[order]
            drop = np.diff(g) < 0
            assert np.all(-np.diff(g)[drop] <= bo[:-1][drop] + bo[1:][drop]), name
            w = worst.setdefault(name, [0.0, 0.0])
            w[0], w[1] = max(w[0], float(err.max())), max(w[1], float(ratio.max()))
    print("spline per parameter set: max |got - fp64|, max fraction of the bound:",
          {k: f"{v[0]:.2e} {v[1]:.2f}" for k, v in worst.items()})


def _durations(z, segs, m0, logs0, ls, rows):
    zz = np.ascontiguousarray(z, dtype=np.float32)
    off = np.ascontiguousarray([s[0] for s in segs], dtype=np.int32)
    ln = np.ascontiguousarray([s[1] for s in segs], dtype=np.int32)
    logw = np.full(rows, -7.0, dtype=np.float32)
    cum = np.full(rows, -7, dtype=np.int32)
    y_len = np.zeros(len(segs), dtype=np.int32)
    err = N.sb200_error()
    rc = N.lib().sb200_debug_durations(0, zz.ctypes.data_as(C.POINTER(C.c_float)), rows,
                                       off.ctypes.data_as(C.POINTER(C.c_int32)), ln.ctypes.data_as(C.POINTER(C.c_int32)),
                                       len(segs), m0, logs0, ls, logw.ctypes.data_as(C.POINTER(C.c_float)),
                                       cum.ctypes.data_as(C.POINTER(C.c_int32)), y_len.ctypes.data_as(C.POINTER(C.c_int32)),
                                       C.byref(err))
    assert rc == 0, C.string_at(err.message).decode() if err.message else rc
    return logw, cum, y_len


def _layout(lens, gap=3):
    segs, cur = [], 0
    for n in lens:
        segs.append((cur, n))
        cur += n + gap
    return segs, cur


def test_duration_kernel_scan_and_saturation(lib_built):
    """durations_kernel through sb200_debug_durations: segment lengths around the warp (32) and block (256) sizes of the
    scan and past 4096 in one launch, cum / y_len exactly against an int64 host scan of the kernel's own w; rows
    between segments untouched; length_scale 0 gives w = 0 and y_len 1; a per-id w past 2^31 - 1, or a segment sum past
    it, saturates cum and y_len at INT32_MAX instead of wrapping."""
    lens = (1, 31, 32, 33, 255, 256, 257, 511, 512, 513, 4097)
    segs, rows = _layout(lens)
    rng = np.random.default_rng(3)
    z = rng.normal(0.5, 1.0, (rows, 2)).astype(np.float32)
    m0, logs0 = 0.1, -0.2
    for ls in (1.0, 0.45, 1.7, 0.0):
        logw, cum, y_len = _durations(z, segs, m0, logs0, ls, rows)
        inseg = np.zeros(rows, bool)
        for b, (o, n) in enumerate(segs):
            inseg[o:o + n] = True
            lw = logw[o:o + n]
            ref_lw = (z[o:o + n, 0].astype(np.float64) - np.float32(m0)) * math.exp(-np.float32(logs0))
            assert np.all(np.abs(lw - ref_lw) <= 6 * 2.0 ** -24 * np.abs(ref_lw) + 1e-30), b
            # the kernel's w: ceil of the fp32 product; within an ulp of the float64 one, so the scan is checked on the
            # ids away from an integer and the ids near one are bounded by one frame
            w64 = np.exp(lw.astype(np.float64)) * float(np.float32(ls))
            got = np.diff(np.concatenate([[0], cum[o:o + n].astype(np.int64)]))
            near = np.abs(w64 - np.rint(w64)) <= 1e-6 * np.maximum(w64, 1)
            assert np.all((got == np.ceil(w64)) | (near & (np.abs(got - np.ceil(w64)) <= 1))), (b, ls)
            assert y_len[b] == max(int(got.sum()), 1), (b, ls)
            if ls == 0.0:
                assert not got.any() and y_len[b] == 1
        assert np.all(cum[~inseg] == -7) and np.all(logw[~inseg] == -7.0)
    # overflow: per-id w ~ e^22 * 1e3 = 3.6e12 (past int32 on its own), and per-id w ~ 1.5 * 2^28 (the sum passes
    # 2^31 - 1 at the sixth id)
    big = np.full((rows, 2), 22.0, dtype=np.float32)
    logw, cum, y_len = _durations(big, segs, 0.0, 0.0, 1e3, rows)
    assert np.all(y_len == INT_MAX)
    for o, n in segs:
        assert np.all(cum[o:o + n] == INT_MAX)
    mid = np.full((rows, 2), np.float32(np.log(1.5 * 2.0 ** 28)), dtype=np.float32)
    logw, cum, y_len = _durations(mid, segs, 0.0, 0.0, 1.0, rows)
    for b, (o, n) in enumerate(segs):
        c = cum[o:o + n].astype(np.int64)
        ref = np.cumsum(np.exp(logw[o:o + n].astype(np.float64)))
        slack = 64.0 * np.arange(1, n + 1)              # the fp32 exp is within 2 ulp (32 each) of the float64 one
        assert np.all(np.diff(c) >= 0), b
        surely_below, surely_above = ref + slack < INT_MAX, ref - slack > INT_MAX
        assert np.all(np.abs(c - ref)[surely_below] <= slack[surely_below] + 1), b
        assert np.all(c[surely_above] == INT_MAX), b
        assert y_len[b] == (INT_MAX if n >= 6 else int(c[-1])), (b, y_len[b])


def test_overlong_durations_raise_and_zero_durations_give_one_frame(voice_paths, oracle_weights):
    """Through the public API: length_scale 1e9 on a 40-id utterance sums past 2^31 - 1 frames and must raise (the scan
    used to wrap into a small frame count); length_scale 0 gives every id 0 frames, y_len clamps to 1, and that frame is
    the oracle's expand of no token: 0 without noise."""
    m = sonata_b200.from_config_path(voice_paths["medium"], device=0)
    ids = workload.synthetic_ids(19, utt=12)
    assert len(ids) == 40
    m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.0, 1e9, 0.0))
    with pytest.raises(sonata_b200.OperationError):
        m.infer_with_values(ids)
    m.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.0, 0.0, 0.0))
    job = SynthesisJob(m, [ids], debug=True)
    job.run()
    assert job.lengths()[0] == [1]
    assert not job.durations(0).any()
    zp = job.debug_fetch("z_p", 0)
    st = {}
    vo.infer(oracle_weights("medium"), ids, [0, 0, 0], stages=st)
    assert st["y_len"] == 1
    assert zp.shape == (1, st["z_p"].shape[1]) and np.array_equal(zp[0], st["z_p"][0, :, 0].numpy())
    job.close()
    m.close()
