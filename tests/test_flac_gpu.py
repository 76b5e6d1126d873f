"""GPU (-m gpu): FLAC streams encoded on the device.

flac_encode on crafted signals at every output rate and length class (bit-exact decode, every CRC, exact STREAMINFO,
the streamable subset), the exactness of every frame's choice against the host's Rice costs, jobs of every voice
quality at several rates with and without loudness targets and gains (against fetch_i16, fetch_g711 and flac_encode),
an utterance of a mixed C2-sized batch equal to itself alone, the frontends, and the launches."""
import io
import os
import sys
import wave

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import flac_reference as fr
import sonata_b200
from sonata_b200 import PiperSynthesisConfig, cli, voicegen, workload
from sonata_b200 import _native as N
from sonata_b200.core import AudioSamples, flac_encode, g711_encode
from sonata_b200.job import SynthesisJob
from sonata_b200.synth import AudioOutputConfig, SonataSpeechSynthesizer

pytestmark = pytest.mark.gpu

DEFAULT = PiperSynthesisConfig(None, 0.667, 1.0, 0.8)
RATES = (8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000)
LENGTHS = (0, 1, 15, 4095, 4096, 4097, 3 * 4096 + 17)


@pytest.fixture(scope="module")
def voices(lib_built):
    d = voicegen.default_voice_dir()
    paths = {q: voicegen.write_voice(d, q) for q in ("medium", "high", "low", "x_low")}
    paths["medium4"] = voicegen.write_voice(d, "medium", n_speakers=4)
    ms = {}

    def get(q):
        if q not in ms:
            ms[q] = sonata_b200.from_config_path(paths[q], device=0)
            ms[q].set_fallback_synthesis_config(DEFAULT)
        return ms[q]
    get.paths = paths
    yield get
    for m in ms.values():
        m.close()


def _signals(n):
    i = np.arange(n)
    rng = np.random.default_rng(n + 7)
    sig = {
        "zeros": np.zeros(n),
        "constant": np.full(n, -1234),
        "ramp": 2 * i - 12000,
        "alternating": np.where(i % 2 == 0, 32767, -32768),
        "noise": rng.integers(-32768, 32768, n),
        "sine": np.round(20000 * np.sin(2 * np.pi * 440.0 * i / 22050.0)),
        "sines": np.round(9000 * np.sin(0.013 * i) + 7000 * np.sin(0.31 * i + 1.0) + rng.normal(0, 30, n)),
        "impulse": np.where(i == n // 2, 30000, 0),
    }
    return {k: np.clip(v, -32768, 32767).astype(np.int16) for k, v in sig.items()}


def check_stream(data, x, rate):
    """Decodes `data` (every CRC checked by the decoder) and checks it against samples x at rate: the samples bit for
    bit, STREAMINFO exactly, and the streamable-subset constraints.  Returns the decoded stream."""
    s = fr.decode(data)
    np.testing.assert_array_equal(s.samples, np.asarray(x, np.int64))
    assert s.metadata == [(0, 34)]
    sizes = [f.size for f in s.frames]
    assert (s.min_block, s.max_block) == (4096, 4096)
    assert (s.min_frame, s.max_frame) == ((min(sizes), max(sizes)) if sizes else (0, 0))
    assert (s.sample_rate, s.channels, s.bits, s.total, s.md5) == (rate, 1, 16, len(x), bytes(16))
    assert len(data) == 42 + sum(sizes)
    nf = (len(x) + 4095) // 4096
    assert len(s.frames) == nf
    for k, f in enumerate(s.frames):
        last = k == nf - 1
        assert f.block_size == (len(x) - 4096 * k if last else 4096)
        assert f.bs_code == (12 if f.block_size == 4096 else 6 if f.block_size <= 256 else 7)
        assert f.rate_code == fr.RATE_CODES[rate] and f.sample_rate == rate
        assert f.wasted == 0 and f.escapes == 0
        assert f.porder <= 8
        if f.type == "LPC":
            assert 1 <= f.order <= 8 and f.precision == 12 and 0 <= f.shift <= 15
            assert all(-2048 <= q <= 2047 for q in f.coefs)
        if f.type == "FIXED":
            assert 0 <= f.order <= 4
    return s


def check_choices(s):
    """Every frame's choice is exact: its residual costs what rice_cost says, and it is no larger than VERBATIM and every
    FIXED order, with ties going FIXED (by order), then LPC, then VERBATIM."""
    pos = 0
    for f in s.frames:
        x = s.samples[pos:pos + f.block_size]
        pos += f.block_size
        n = len(x)
        if f.type == "CONSTANT":
            assert (x == x[0]).all()
            continue
        assert not (x == x[0]).all()
        verbatim = fr.subframe_cost(x, "VERBATIM")
        fixed = [fr.subframe_cost(x, "FIXED", o) if n > o else None for o in range(5)]
        if f.type in ("FIXED", "LPC"):
            res = fr.lpc_residual(x, f.coefs, f.shift)
            bits, po, ks = fr.rice_cost(res, f.order)
            assert (bits, po, ks) == (f.residual_bits, f.porder, f.params), (f.number, f.type, f.order)
        assert f.subframe_bits <= verbatim
        if f.type == "VERBATIM":
            assert f.subframe_bits == verbatim
            assert all(c is None or c > verbatim for c in fixed)
        elif f.type == "FIXED":
            assert f.subframe_bits == fixed[f.order]
            assert all(c is None or c > f.subframe_bits for c in fixed[:f.order])
            assert all(c is None or c >= f.subframe_bits for c in fixed[f.order:])
        else:
            assert all(c is None or c > f.subframe_bits for c in fixed)


@pytest.mark.parametrize("rate", RATES)
def test_crafted_signals(lib_built, rate):
    for n in LENGTHS:
        for name, x in _signals(n).items():
            data = flac_encode(x, rate)
            s = check_stream(data, x, rate)
            check_choices(s)
            if n and name in ("zeros", "constant"):
                assert all(f.type == "CONSTANT" for f in s.frames)
            if n > 4 and name == "ramp":
                assert s.frames[0].type == "FIXED" and s.frames[0].order == 2 and s.frames[0].params == [0] * len(s.frames[0].params)
            if name in ("alternating", "noise") and n:
                assert len(data) <= 42 + sum(f.size for f in s.frames)
                assert all(f.subframe_bits <= 8 + 16 * f.block_size for f in s.frames)
            assert flac_encode(x, rate) == data, (rate, n, name)         # deterministic
    assert len(flac_encode(np.zeros(0, np.int16), rate)) == 42


def test_frames_depend_only_on_their_samples(lib_built):
    """A frame's bytes are the same whatever precedes it in its stream, apart from its header's frame number."""
    x = _signals(4 * 4096)["sines"]
    a = fr.decode(flac_encode(x, 22050))
    b_data = flac_encode(x[4096:], 22050)
    b = fr.decode(b_data)
    da = flac_encode(x, 22050)
    for fa, fb in zip(a.frames[1:], b.frames):
        body_a = da[fa.offset + len(fa.header) + 1:fa.offset + fa.size - 2]
        body_b = b_data[fb.offset + len(fb.header) + 1:fb.offset + fb.size - 2]
        assert body_a == body_b


def _ids(n, utt):
    return list(workload.synthetic_ids(n, utt=utt))


def _launches(fn):
    n0 = N.lib().sb200_launch_count()
    r = fn()
    return r, N.lib().sb200_launch_count() - n0


@pytest.mark.parametrize("quality", ["medium", "high", "low", "x_low"])
def test_jobs(voices, quality):
    m = voices(quality)
    voice_rate = m.audio_output_info().sample_rate
    rates = [None, 8000, 48000, None, 8000, 48000]
    targets = [None, None, None, -16.0, -16.0, -16.0]
    batches = [_ids(14 + 6 * b, 60 + b) for b in range(len(rates))]
    job = SynthesisJob(m, batches, seeds=[700 + b for b in range(len(rates))], output_rates=rates, loudness=targets)
    job.run()
    i16 = job.fetch_i16()
    got = job.fetch_flac()
    for b in range(len(rates)):
        rate = rates[b] or voice_rate
        s = check_stream(got[b], i16[b], rate)
        check_choices(s)
        assert got[b] == flac_encode(i16[b], rate), (quality, b)
    assert job.fetch_flac() == got                                      # two fetches, the same bytes
    gains = [0.5 + 0.1 * b for b in range(len(rates))]
    with_gain = job.fetch_flac(gains)
    for law in ("mulaw", "alaw"):
        g711 = job.fetch_g711(law, gains)
        for b in range(len(rates)):
            dec = fr.decode(with_gain[b]).samples.astype(np.int16)
            assert g711_encode(dec, law).tobytes() == g711[b], (quality, law, b)
    with pytest.raises(sonata_b200.OperationError, match="utterance 2: gain"):
        job.fetch_flac([1, 1, float("inf"), 1, 1, 1])
    job.close()


def test_job_without_audio(voices):
    m = voices("medium")
    job = SynthesisJob(m, [_ids(10, 1)])
    with pytest.raises(sonata_b200.OperationError, match="has not produced audio"):
        job.fetch_flac()
    job.close()


def test_launches(voices):
    m = voices("medium")
    batches = [_ids(30, 3), _ids(9, 4), _ids(14, 5)]

    def make():
        return SynthesisJob(m, batches, seeds=[1, 2, 3], output_rates=[0, 48000, 8000], loudness=[None, -16.0, None])
    job = make()
    _, n_run = _launches(job.run)
    regions = [r["name"] for r in job.profile()]
    wav = [a.samples.as_slice().copy() for a in job.fetch()]
    i16, n_i16 = _launches(job.fetch_i16)
    assert n_i16 == 2
    streams, n_flac = _launches(job.fetch_flac)
    assert n_flac == 2 + 3                      # the i16 conversion, then analysis, layout and pack
    assert [r["name"] for r in job.profile()] == regions
    other = make()
    _, n_run2 = _launches(other.run)            # a job that fetches no FLAC launches what it launched before
    assert n_run2 == n_run
    other.close()
    for a, w in zip(job.fetch(), wav):
        np.testing.assert_array_equal(a.samples.as_slice(), w)
    assert job.fetch_i16()[0].tolist() == i16[0].tolist()
    job.close()


@pytest.mark.parametrize("size", ["small", "c2"])
def test_mixed_batch_equals_alone(voices, size):
    m = voices("medium4")
    B, n = (6, 24) if size == "small" else (32, 256)
    batches = [_ids(n - 3 * (b % 5), 300 + b) for b in range(B)]
    rates = [(0, 8000, 48000, 22050, 11025, 16000)[b % 6] for b in range(B)]
    targets = [(None, -23.0, -16.0, None, -30.0)[b % 5] for b in range(B)]
    configs = [PiperSynthesisConfig(b % 4, 0.667, 1.0, 0.8) for b in range(B)]
    seeds = [4000 + b for b in range(B)]
    gains = [1.0 - 0.02 * b for b in range(B)]
    mixed = m.infer_batch_flac(batches, configs, seeds, rates, targets, gains)
    for b in range(B):
        alone = m.infer_batch_flac([batches[b]], [configs[b]], [seeds[b]], [rates[b]], [targets[b]], [gains[b]])
        assert mixed[b] == alone[0], b
    for b in (0, B - 1):
        job = SynthesisJob(m, [batches[b]], seeds=[seeds[b]], output_rates=[rates[b]], loudness=[targets[b]],
                           configs=[configs[b]])
        job.run()
        x = job.fetch()[0].samples.as_slice() * np.float32(gains[b])
        a = AudioSamples(x)
        want = a.to_i16_fixed() if targets[b] is not None else a.to_i16_vec()
        np.testing.assert_array_equal(fr.decode(mixed[b]).samples, want)
        job.close()


def test_speak_batch_flac(voices):
    m = voices("medium")
    phs = ["hɛloʊ wɜːld", "ə sɛkənd wʌn"]
    got = m.speak_batch_flac(phs, seeds=[3, 4], output_rates=[None, 16000])
    job = SynthesisJob(m, [m.phonemes_to_input_ids(p) for p in phs], seeds=[3, 4], output_rates=[None, 16000])
    job.run()
    assert got == job.fetch_flac()
    job.close()
    with pytest.raises(sonata_b200.OperationError):
        m.infer_batch_flac([[1, 2]], output_rates=[12345])
    assert m.infer_batch_flac([]) == []


LONG = "hɛloʊ wɜːld ðɪs ɪz ə lɔŋɡɚ sɛntəns ðæt ɪz spoʊkən ɪn tʃʌŋks ænd ðɛn sʌm moʊr wɜːdz"


def _wav_samples(path):
    with wave.open(str(path), "rb") as w:
        return w.getframerate(), np.frombuffer(w.readframes(w.getnframes()), "<i2")


def test_frontends(voices, tmp_path):
    m = voices("medium")
    synth = SonataSpeechSynthesizer(m)
    text = LONG + "\n" + "ænd ə sɛkənd wʌn"
    oc = AudioOutputConfig(10, 60, 50, 20)
    for extra in ({}, {"output_rate": 8000}, {"loudness": -16.0}):
        synth.synthesize_to_file(tmp_path / "o.wav", text, oc, seed=5, **extra)
        synth.synthesize_to_file(tmp_path / "o.flac", text, oc, seed=5, encoding="flac", **extra)
        rate, want = _wav_samples(tmp_path / "o.wav")
        s = fr.decode((tmp_path / "o.flac").read_bytes())
        assert s.sample_rate == rate == extra.get("output_rate", 22050)
        np.testing.assert_array_equal(s.samples, want)
    (tmp_path / "in.txt").write_text(text + "\n", encoding="utf-8")
    for mode in ("lazy", "parallel"):
        buf = io.BytesIO()
        req = {"text": text, "mode": mode, "seed": 5, "volume": 60, "encoding": "flac", "output_rate": 8000}
        cli.process_request(synth, DEFAULT, req, None, buf)
        cli.process_request(synth, DEFAULT, req, str(tmp_path / f"{mode}.flac"))
        assert buf.getvalue() == (tmp_path / f"{mode}.flac").read_bytes()
        assert buf.getvalue() == synth.synthesize_flac(text, AudioOutputConfig(None, 60), seed=5, output_rate=8000)
        m.set_fallback_synthesis_config(DEFAULT)
    out = tmp_path / "c.flac"
    assert cli.main([voices.paths["medium"], "-f", str(tmp_path / "in.txt"), "-o", str(out), "--encoding", "flac",
                     "--seed", "5", "--loudness", "-16"]) == 0
    synth.synthesize_to_file(tmp_path / "c.wav", text + "\n", seed=5, loudness=-16.0)
    np.testing.assert_array_equal(fr.decode(out.read_bytes()).samples, _wav_samples(tmp_path / "c.wav")[1])
    m.set_fallback_synthesis_config(DEFAULT)
