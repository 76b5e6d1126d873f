"""Host (no GPU): every case table of tests/waveform_edges.py reaches the edge it is named for, shown through the
library's device-free plan hooks (prosody and contour plans, the resampling filter and emit counts) and the float64
specifications; and those specifications are right at the short lengths, against direct restatements (an O(N^2) DFT
for the formant stage, the sum over the tap index for the resampler), so a failure of the GPU edge tests points at a
kernel rather than at numpy's edge handling."""
import math

import numpy as np
import pytest

import waveform_edges as we
from waveform_edges import fr, lr, pc, pr, rr


# ---------------------------------------------------------------- formant stage

def test_formant_lengths_reach_frame_hop_and_cta_edges(lib_built):
    L = we.FORMANT_LENGTHS
    hops = lambda n: -(-n // we.H)
    runs = lambda n: -(-hops(n) // we.FM_HOPS)
    assert {1, 2, 3} <= set(L)
    assert min(L) < we.H and any(n < fr.N for n in L)
    for edge in (we.H, 3 * we.H, fr.N):                              # a hop, 3 hops, a frame, and one sample either side
        assert {edge - 1, edge, edge + 1} <= set(L)
    assert [runs(n) for n in (we.FM_HOPS * we.H - 1, we.FM_HOPS * we.H, we.FM_HOPS * we.H + 1)] == [1, 1, 2]
    assert hops(we.FM_HOPS * we.H + 1) == we.FM_HOPS + 1                 # the second CTA holds one hop of one sample
    assert runs(2 * we.FM_HOPS * we.H + 1) == 3
    for rate in we.RATES:
        for n in L:
            for name, p, t, phi in we.FORMANT_RATIOS:
                Hs, N, D, n1, n2, F = we.prosody_plan(lib_built, rate, n, p, t)
                assert n2 == pr.plan(rate, n, p, t)["n2"], (rate, n, name)
                if t is None:           # the stage sees the table's length, rounded up to even n2 = 2 round(n / 2) at p = 0.5
                    assert n2 == (n + n % 2 if p == 0.5 else n), (rate, n, name, n2)
                else:
                    assert n2 == math.floor(n / t + 0.5), (rate, n, name)


def test_formant_ratio_corners():
    r = {name: (1.0 if p is None else p) / phi for name, p, t, phi in we.FORMANT_RATIOS}
    assert r["p2_phi0.5"] == 4.0                        # every k >= N / 8 reads the envelope past N / 2
    assert r["p0.5_phi2"] == 0.25
    assert r["p0.5_phi0.5"] == r["p2_phi2"] == 1.0      # skipped: the output is the input's bits
    assert not fr.asks(1000, 0.5, pitch=0.5) and not fr.asks(1000, 2.0, pitch=2.0)
    assert fr.asks(1000, 0.5, pitch=2.0) and fr.asks(1000, 2.0)
    assert {t for _, _, t, _ in we.FORMANT_RATIOS} == {None, 0.25, 4.0}


@pytest.mark.parametrize("rate", we.RATES)
def test_formant_contours_put_knots_on_frame_centres(lib_built, rate):
    seen = set()
    for n in we.FORMANT_LENGTHS:
        for name, ends, ratios, Q, m, d in we.formant_contours(n):
            shape, bounds = we.contour_plan(lib_built, rate, n, ends, ratios, None)
            pl = pc.plan(rate, n, ends, ratios, None)
            assert shape[4] == pl["n2"] == n, (n, name)
            np.testing.assert_array_equal(bounds, pl["bounds"])
            # the last piece starts at output Q exactly: the library's delivered end of the id before it, and the spec's
            assert bounds[-2] == Q and pl["Q"][-1] == Q, (n, name)
            centre = min(m * fr.H + fr.N // 2, n - 1)
            assert centre == Q - d, (n, name)
            fm, p = fr.frame_ratios(n, Q=pl["Q"], P=pl["p"])
            k = int(np.nonzero(fm == m)[0][0])
            assert p[k] == (pl["p"][-1] if d <= 0 else pl["p"][-2]), (n, name)
            if name == "last_clamped":
                assert m * fr.H + fr.N // 2 > n - 1                     # the centre is clamped
                assert np.count_nonzero(p == pl["p"][-1]) >= 1 and pl["B"][-1] - pl["B"][-2] == 1
            if name == "short_piece":
                assert pl["B"][2] - pl["B"][1] < fr.H
            seen.add(name)
    assert seen == {"last_clamped", "knot_at_m1", "knot_before_m1", "knot_after_m1", "knot_at_m32",
                    "knot_before_m32", "knot_after_m32", "short_piece"}


def test_formant_job_table(lib_built):
    totals, n2s = set(), set()
    for frames, p, t, contour, phi, n2 in we.FORMANT_JOB:
        n = 256 * sum(frames)
        totals.add(sum(frames))
        for rate in we.RATES:
            if contour is None:
                got = we.prosody_plan(lib_built, rate, n, p, t)[4]
            else:
                assert p is None
                got = we.contour_plan(lib_built, rate, n, we.job_ends(frames), contour, t)[0][4]
            assert got == n2, (frames, p, t, got)
        n2s.add(n2)
        assert fr.asks(n2, phi, pitch=p) or contour is not None
    assert {1, 2, 3, 4, 5, 33} <= totals
    assert {1023, 1024, 1025, 8191, 8192, 8193} <= n2s
    assert any(f[0] == 0 for f, *_ in we.FORMANT_JOB)           # an id with no frames


# ---------------------------------------------------------------- pitch / tempo

@pytest.mark.parametrize("rate", we.RATES)
def test_prosody_lengths_reach_hop_frame_and_run_edges(lib_built, rate):
    for cname, p, t in we.PROSODY_CORNERS:
        cases = dict(we.prosody_lengths(rate, p, t))
        Hs, N, D, *_ = we.prosody_plan(lib_built, rate, 1000, p, t)
        assert (cases["Hs-1"], cases["Hs"], cases["Hs+1"]) == (Hs - 1, Hs, Hs + 1)
        assert (cases["N-1"], cases["N"], cases["N+1"]) == (N - 1, N, N + 1) and N == 2 * Hs
        for name, n in cases.items():
            shape = we.prosody_plan(lib_built, rate, n, p, t)
            pl = pr.plan(rate, n, p, t)
            assert shape == (pl["Hs"], pl["N"], pl["D"], pl["n1"], pl["n2"], pl["F"]), (cname, name)
        runs = {}
        for target in we.PROSODY_N2:
            n = cases[f"n2>={target}"]
            n2 = we.prosody_plan(lib_built, rate, n, p, t)[4]
            assert n2 >= target and we.prosody_plan(lib_built, rate, n - 1, p, t)[4] < target, (cname, target)
            assert n2 - target < 4
            runs[target] = -(-n2 // we.PP_OUTS)
        assert runs == {255: 1, 256: 1, 257: 2, 513: 3}, (cname, runs)
        # the frame count changes across the table: one frame, and more than one
        Fs = {we.prosody_plan(lib_built, rate, n, p, t)[5] for n in cases.values()}
        if t is not None:
            assert 1 in Fs and max(Fs) >= 2, (cname, Fs)
    # where the ratios can reach them, the named n2 are reached exactly
    assert we.prosody_plan(lib_built, rate, dict(we.prosody_lengths(rate, None, 4.0))["n2>=255"], None, 4.0)[4] == 255
    assert we.prosody_plan(lib_built, rate, dict(we.prosody_lengths(rate, 2.0, None))["n2>=257"], 2.0, None)[4] == 257


@pytest.mark.parametrize("rate", we.RATES)
def test_prosody_contours_have_their_pieces(lib_built, rate):
    Hs = rate // 100
    for n in (Hs + 1, 2 * Hs + 1, 3 * Hs + 7):
        for name, ends, ratios in we.prosody_contours(n, rate):
            for tempo in (None, 0.25, 4.0):
                shape, bounds = we.contour_plan(lib_built, rate, n, ends, ratios, tempo)
                pl = pc.plan(rate, n, ends, ratios, tempo)
                assert shape == (pl["Hs"], pl["N"], pl["D"], pl["n1"], pl["n2"], pl["F"]), (n, name, tempo)
                np.testing.assert_array_equal(bounds, pl["bounds"])
                assert pl["one"] is None and pl["m"] >= 2
            B = pc.pieces(n, ends, ratios)[0]
            lens = np.diff(B)
            if name == "one_sample":
                assert 1 in lens
            elif name == "knot_1":
                assert B[1] == 1
            elif name == "knot_n-1":
                assert B[-2] == n - 1
            else:
                assert np.all(lens < Hs) and len(lens) >= 3


# ---------------------------------------------------------------- resampler

@pytest.mark.parametrize("in_rate,out_rate", we.RS_PAIRS)
def test_resample_lengths_reach_chain_and_run_edges(lib_built, in_rate, out_rate):
    up, down, taps = we.resample_filter(lib_built, in_rate, out_rate)
    assert (up, down) == rr.ratio(in_rate, out_rate)
    K = -(-len(taps) // up)
    assert len(taps) == 2 * 10 * max(up, down) + 1 and K == we.taps_per_phase(in_rate, out_rate)
    cases = dict(we.resample_lengths(in_rate, out_rate))
    assert (cases["1"], cases["2"], cases["K-1"], cases["K"], cases["K+1"]) == (1, 2, K - 1, K, K + 1)
    for name, n in cases.items():
        assert int(we.resample_emit(lib_built, in_rate, out_rate, [n])[0]) == rr.n_out(n, up, down), name
    runs = {}
    for target in we.RS_N_OUT:
        n = cases[f"n_out>={target}"]
        got = int(we.resample_emit(lib_built, in_rate, out_rate, [n])[0])
        assert got >= target and rr.n_out(n - 1, up, down) < target, target
        assert got - target < -(-up // down)
        if down >= up:
            assert got == target
        runs[target] = -(-got // we.RS_OUTS)
    assert runs[1025] == 2 and runs[2049] == 3
    # at n = K - 1, K and K + 1 the chains are clipped at both ends: some output has fewer terms than its phase's full
    # chain because input 0 is its first (kmax clips it), and some because input n - 1 is its last (kmin clips it)
    H = 10 * max(up, down)
    for n in (cases["K-1"], cases["K"], cases["K+1"]):
        head = tail = False
        for j in range(rr.n_out(n, up, down)):
            t = j * down + H
            full = [i for i in range(-2 * K, n + 2 * K) if 0 <= t - i * up <= 2 * H]
            got = [i for i in full if 0 <= i < n]
            head |= bool(got) and got[0] == 0 and full[0] < 0
            tail |= bool(got) and got[-1] == n - 1 and full[-1] > n - 1
        assert head and tail, n


# ---------------------------------------------------------------- loudness

@pytest.mark.parametrize("rate", lr.RATES)
def test_loudness_lengths_and_gates(rate):
    S = lr.step(rate)
    chunks = {name: -(-n // S) for name, n in we.loudness_lengths(rate)}
    blocks = {name: (n - 4 * S) // S + 1 for name, n in we.loudness_lengths(rate)}
    assert chunks["255S"] == 255 and chunks["256S"] == 256 and chunks["257S+1"] == 258
    assert chunks["70s"] > we.LD_THREADS and blocks["70s"] > we.LD_THREADS
    for name, n in we.loudness_lengths(rate):
        x = we.level_step(rate, n)
        assert len(x) == n
        g = we.relative_gate(x, rate)
        l = we.block_loudness(x, rate)
        hi, lo = we.steady_blocks(rate, n, "hi"), we.steady_blocks(rate, n, "lo")
        assert len(hi) > 50 and len(lo) > 50
        assert np.all(l[hi] > g) and np.all(l[hi] < g + 0.02), (name, float(np.min(l[hi] - g)))
        assert np.all(l[lo] < g) and np.all(l[lo] > g - 0.02), (name, float(np.max(l[lo] - g)))
        assert np.all(l > -70.0)
        a = we.at_absolute_gate(rate, n)
        la = we.block_loudness(a, rate)
        assert np.all(np.abs(la + 70.0) < 0.01), name
        assert np.any(la > -70.0) and np.any(la <= -70.0), name


# ---------------------------------------------------------------- the specifications at short lengths

def _formant_direct(y, rate, phi, pitch):
    """fr.apply restated with O(N^2) DFT matrices, full complex spectra, and np.interp for the envelope's reading."""
    N, Hh = fr.N, fr.H
    y = np.asarray(y, np.float64)
    n2 = len(y)
    p = 1.0 if pitch is None else float(np.float32(pitch))
    r = p / float(np.float32(phi))
    Qm = math.floor(rate // 250 / p + 0.5)
    k = np.arange(N)
    Fw = np.exp(-2j * np.pi * np.outer(k, k) / N)
    w = 0.5 - 0.5 * np.cos(2 * np.pi * k / N)
    qq = np.minimum(k, N - k)
    lift = np.array([1.0 if q == 0 else (0.5 * (1 + math.cos(math.pi * q / Qm)) if q < Qm else 0.0) for q in qq])
    out = np.zeros(n2)
    m = -3
    while m * Hh < n2:
        idx = m * Hh + k
        frame = np.array([y[i] if 0 <= i < n2 else 0.0 for i in idx]) * w
        X = Fw @ frame
        P = np.abs(X) ** 2
        eps = 1e-10 * np.mean(P[:N // 2 + 1]) + 1e-30
        c = (np.conj(Fw) @ (0.5 * np.log(P + eps))).real / N
        E = (Fw @ (c * lift)).real
        half = np.arange(N // 2 + 1)
        g = np.clip(np.interp(half * r, half, E[:N // 2 + 1]) - E[:N // 2 + 1], -fr.CLAMP, fr.CLAMP)
        Z = np.zeros(N, complex)
        Z[:N // 2 + 1] = X[:N // 2 + 1] * np.exp(g)
        Z[N // 2 + 1:] = np.conj(Z[1:N // 2][::-1])
        z = (np.conj(Fw) @ Z).real / N
        for i in range(N):
            if 0 <= idx[i] < n2:
                out[idx[i]] += w[i] * z[i] / 1.5
        m += 1
    return out


@pytest.mark.parametrize("n2", [1, 2, 3, 255, 257, 767, 1023, 1025])
def test_formant_spec_against_direct_dft(n2):
    rng = np.random.default_rng(n2)
    y = (0.4 * rng.standard_normal(n2)).astype(np.float32)
    y[n2 - 1] = 0.9
    for rate, phi, pitch in ((22050, 0.5, 2.0), (16000, 2.0, 0.5), (22050, 0.8, None), (16000, 1.0, 1.25)):
        ref = fr.apply(y, rate, phi, pitch)
        got = _formant_direct(y, rate, phi, pitch)
        assert ref.shape == (n2,)
        np.testing.assert_allclose(ref, got, rtol=0, atol=1e-12 * max(1.0, float(np.max(np.abs(got)))))


@pytest.mark.parametrize("in_rate,out_rate", [(22050, 48000), (22050, 8000), (16000, 11025), (16000, 48000),
                                              (22050, 44100), (16000, 8000)])
def test_resample_spec_against_direct_sum(in_rate, out_rate):
    up, down = rr.ratio(in_rate, out_rate)
    h = rr.taps64(up, down)
    H = (len(h) - 1) // 2
    K = we.taps_per_phase(in_rate, out_rate)
    rng = np.random.default_rng(up + down)
    for n in (1, 2, K - 1, K, K + 1):
        for x in (rng.standard_normal(n), np.eye(1, n, 0)[0], np.eye(1, n, n - 1)[0]):
            ref = rr.resample64(x, up, down)
            assert ref.shape == (rr.n_out(n, up, down),)
            direct = np.zeros(len(ref))
            for j in range(len(ref)):
                for i in range(n):
                    t = j * down + H - i * up
                    if 0 <= t <= 2 * H:
                        direct[j] += x[i] * h[t]
            np.testing.assert_allclose(ref, direct, rtol=0, atol=1e-12)
