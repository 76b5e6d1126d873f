"""GPU (-m gpu): G.711 mu-law / A-law results encoded on the device.

The device encoders over every 16-bit value, jobs of every voice quality at several output rates and loudness targets
(fetch_g711 and copy_out against the encoding of fetch_i16), an utterance of a mixed C2-sized batch equal to itself
alone, the launches and profile regions of the encoded routes, realtime streams (plain, one-shot, resampled and a
StreamBatch of mixed streams), and the synthesizer's and CLI's modes."""
import ctypes as C
import io
import os
import struct
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import g711_reference as gr
import sonata_b200
from sonata_b200 import PiperSynthesisConfig, cli, voicegen, workload
from sonata_b200 import _native as N
from sonata_b200.core import AudioSamples
from sonata_b200.job import SynthesisJob
from sonata_b200.piper import StreamBatch, VitsStreamingModel
from sonata_b200.synth import AudioOutputConfig, RealtimeBatch, SonataSpeechSynthesizer

pytestmark = pytest.mark.gpu

DEFAULT = PiperSynthesisConfig(None, 0.667, 1.0, 0.8)
LAWS = ("mulaw", "alaw")
CS, PAD = 20, 3


@pytest.fixture(scope="module")
def voices(lib_built):
    d = voicegen.default_voice_dir()
    paths = {q: voicegen.write_voice(d, q) for q in ("medium", "high", "low", "x_low")}
    paths["medium4"] = voicegen.write_voice(d, "medium", n_speakers=4)
    ms = {}

    def get(q):
        if q not in ms:
            ms[q] = (VitsStreamingModel(paths["medium"], device=0) if q == "stream"
                     else sonata_b200.from_config_path(paths[q], device=0))
            ms[q].set_fallback_synthesis_config(DEFAULT)
        return ms[q]
    get.paths = paths
    yield get
    for m in ms.values():
        m.close()


def _ids(n, utt):
    return list(workload.synthetic_ids(n, utt=utt))


def _launches(fn):
    n0 = N.lib().sb200_launch_count()
    r = fn()
    return r, N.lib().sb200_launch_count() - n0


@pytest.mark.parametrize("law", [0, 1])
def test_device_hook_every_value(lib_built, law):
    x = gr.VALUES.astype(np.int16)
    out = np.zeros(x.size, np.uint8)
    err = N.sb200_error()
    assert N.lib().sb200_debug_g711(0, law, x.ctypes.data_as(C.POINTER(C.c_int16)), x.size,
                                    out.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(err)) == 0
    np.testing.assert_array_equal(out, gr.TABLES[LAWS[law]])


@pytest.mark.parametrize("quality", ["medium", "high", "low", "x_low"])
def test_jobs(voices, quality):
    m = voices(quality)
    rates = [None, 8000, 48000, None, 8000, 48000]
    targets = [None, None, None, -16.0, -16.0, -16.0]
    batches = [_ids(14 + 6 * b, 60 + b) for b in range(len(rates))]
    job = SynthesisJob(m, batches, seeds=[700 + b for b in range(len(rates))], output_rates=rates, loudness=targets)
    job.run()
    i16 = job.fetch_i16()
    samples = job.lengths()[1]
    gains = [0.5 + 0.1 * b for b in range(len(rates))]
    i16_g = [AudioSamples(a.samples.as_slice() * np.float32(g)) for a, g in zip(job.fetch(), gains)]
    for fmt, law in ((2, "mulaw"), (3, "alaw")):
        got = job.fetch_g711(law)
        for b in range(len(rates)):
            assert len(got[b]) == samples[b] == len(i16[b])
            assert got[b] == gr.encode_bytes(i16[b], law), (quality, law, b)
        # per-utterance gains: the i16 samples of the scaled signal
        with_gain = job.fetch_g711(law, gains)
        for b in range(len(rates)):
            ref = i16_g[b].to_i16_fixed() if targets[b] is not None else i16_g[b].to_i16_vec()
            assert with_gain[b] == gr.encode_bytes(ref, law), (quality, law, b)
        buf = np.zeros(sum(samples), np.uint8)
        assert job.copy_out(buf.ctypes.data, buf.nbytes, fmt) == buf.nbytes == sum(samples)
        assert buf.tobytes() == b"".join(got)
        with pytest.raises(sonata_b200.OperationError, match="too small"):
            job.copy_out(buf.ctypes.data, buf.nbytes - 1, fmt)
    for bad in (4, -1):
        with pytest.raises(sonata_b200.OperationError, match=f"format {bad}"):
            job.copy_out(buf.ctypes.data, buf.nbytes * 4, bad)
    err = N.sb200_error()
    outs = (C.POINTER(C.c_uint8) * len(rates))()
    lens = (C.c_size_t * len(rates))()
    assert m._lib.sb200_job_fetch_g711(job._h, 5, None, outs, lens, C.byref(err)) == 19
    assert b"law 5" in C.string_at(err.message)
    N.lib().sb200_string_free(err.message)
    bad = np.array([1, 1, float("inf"), 1, 1, 1], np.float32)
    assert m._lib.sb200_job_fetch_g711(job._h, 0, bad.ctypes.data_as(C.POINTER(C.c_float)), outs, lens,
                                       C.byref(err)) == 19
    assert b"utterance 2" in C.string_at(err.message)
    N.lib().sb200_string_free(err.message)
    job.close()


def test_launches_and_regions(voices):
    m = voices("medium")
    batches = [_ids(30, 3), _ids(9, 4), _ids(14, 5)]
    job = SynthesisJob(m, batches, seeds=[1, 2, 3], output_rates=[0, 48000, 8000], loudness=[None, -16.0, None])
    job.run()
    regions = [r["name"] for r in job.profile()]
    wav = [a.samples.as_slice().copy() for a in job.fetch()]
    _, n_i16 = _launches(job.fetch_i16)
    for law in LAWS:
        _, n = _launches(lambda: job.fetch_g711(law))
        assert n == n_i16 == 2
    buf = np.zeros(sum(len(w) for w in wav) * 2, np.uint8)
    for fmt in (1, 2, 3):
        _, n = _launches(lambda: job.copy_out(buf.ctypes.data, buf.nbytes, fmt))
        assert n == 2
    assert [r["name"] for r in job.profile()] == regions
    for a, w in zip(job.fetch(), wav):
        np.testing.assert_array_equal(a.samples.as_slice(), w)
    job.close()


@pytest.mark.parametrize("size", ["small", "c2"])
def test_mixed_batch_equals_alone(voices, size):
    m = voices("medium4")
    B, n = (6, 24) if size == "small" else (32, 256)
    batches = [_ids(n - 3 * (b % 5), 300 + b) for b in range(B)]
    rates = [(0, 8000, 48000, 22050, 11025, 16000)[b % 6] for b in range(B)]
    targets = [(None, -23.0, -16.0, None, -30.0)[b % 5] for b in range(B)]
    laws = [LAWS[(b // 2) % 2] for b in range(B)]
    configs = [PiperSynthesisConfig(b % 4, 0.667, 1.0, 0.8) for b in range(B)]
    seeds = [4000 + b for b in range(B)]
    mixed = m.infer_batch_g711(batches, laws, configs, seeds, rates, targets)
    for b in range(B):
        alone = m.infer_batch_g711([batches[b]], laws[b], [configs[b]], [seeds[b]], [rates[b]], [targets[b]])
        assert mixed[b] == alone[0], b
    # and each is the encoding of what the i16 route gives
    job = SynthesisJob(m, batches, seeds=seeds, output_rates=rates, loudness=targets, configs=configs)
    job.run()
    for b, x in enumerate(job.fetch_i16()):
        assert mixed[b] == gr.encode_bytes(x, laws[b])
    job.close()


def _f32_chunks(m, ph, seed, rate=None):
    return [c.as_slice().copy() for c in m.stream_synthesis(ph, CS, PAD, seed=seed, output_rate=rate)]


LONG = "hɛloʊ wɜːld ðɪs ɪz ə lɔŋɡɚ sɛntəns ðæt ɪz spoʊkən ɪn tʃʌŋks ænd ðɛn sʌm moʊr wɜːdz"
SHORT = "hɪ"


@pytest.mark.parametrize("law", LAWS)
@pytest.mark.parametrize("rate", [None, 8000])
@pytest.mark.parametrize("ph", [LONG, SHORT], ids=["chunked", "one_shot"])
def test_stream_chunks(voices, law, rate, ph):
    m = voices("stream")
    ref = _f32_chunks(m, ph, 11, rate)
    got = list(m.stream_synthesis(ph, CS, PAD, seed=11, output_rate=rate, encoding=law))
    assert len(got) == len(ref)
    for g, r in zip(got, ref):
        assert isinstance(g, bytes)
        assert g == gr.encode_bytes(AudioSamples(r).to_i16_vec(), law)
    scaled = list(m.stream_synthesis(ph, CS, PAD, seed=11, output_rate=rate, encoding=law, gain=0.3))
    for g, r in zip(scaled, ref):
        assert g == gr.encode_bytes(AudioSamples(r * np.float32(0.3)).to_i16_vec(), law)


def test_decoder_pass_launches(voices):
    m = voices("stream")
    enc = m.infer_encoder_batch([_ids(40, 9), _ids(50, 10)], seeds=[9, 10])
    chunks = [(enc[0], 0, 30, 0, 3), (enc[1], 10, 45, 3, 0)]
    i16, n_i16 = _launches(lambda: m.infer_decoder_batch(chunks, pcm16=True, fade=42, gains=[1.0, 0.5]))
    for law in LAWS:
        got, n = _launches(lambda: m.infer_decoder_batch(chunks, fade=42, gains=[1.0, 0.5], encoding=law))
        assert n == n_i16
        for g, x in zip(got, i16):
            assert g == gr.encode_bytes(x, law)
    with pytest.raises(sonata_b200.OperationError, match="two output formats"):
        m.infer_decoder_batch(chunks, pcm16=True, encoding="alaw")


def test_stream_batch_equals_alone(voices):
    m = voices("stream")
    K = 32
    words = LONG.split()
    phs = [" ".join(words[:2 + (k * 5) % (len(words) - 1)]) for k in range(K)]
    encs = [(None, "mulaw", "alaw")[k % 3] for k in range(K)]
    rates = [(None, None, 8000, 48000)[k % 4] for k in range(K)]
    sb = StreamBatch(m, CS, PAD)
    keys = [sb.add(phs[k], seed=900 + k, output_rate=rates[k], encoding=encs[k]) for k in range(K)]
    got = {k: [] for k in keys}
    while len(sb):
        for key, item in sb.step():
            assert not isinstance(item, Exception), item
            got[key].append(item)
    for k in range(K):
        alone = list(m.stream_synthesis(phs[k], CS, PAD, seed=900 + k, output_rate=rates[k], encoding=encs[k]))
        if encs[k] is None:
            assert len(alone) == len(got[keys[k]])
            for a, b in zip(alone, got[keys[k]]):
                np.testing.assert_array_equal(a.as_slice(), b.as_slice())
        else:
            assert got[keys[k]] == alone, k


def _wav_data(path):
    b = open(path, "rb").read()
    assert b[:4] == b"RIFF" and b[8:12] == b"WAVE"
    pos, chunks = 12, {}
    while pos < len(b):
        cid, size = b[pos:pos + 4], struct.unpack("<I", b[pos + 4:pos + 8])[0]
        chunks[cid] = b[pos + 8:pos + 8 + size]
        pos += 8 + size + (size & 1)
    return chunks


@pytest.mark.parametrize("law", LAWS)
def test_frontends(voices, law, tmp_path):
    m = voices("stream")
    synth = SonataSpeechSynthesizer(m)
    text = LONG + "\n" + "ænd ə sɛkənd wʌn"
    oc = AudioOutputConfig(10, 60, 50, 20)
    for extra in ({}, {"output_rate": 8000}, {"loudness": -16.0}):
        fixed = "loudness" in extra
        lazy = list(synth.synthesize_lazy(text, oc, seed=5, encoding=law, **extra))
        assert lazy == [a.samples.as_g711_bytes(law, fixed) for a in synth.synthesize_lazy(text, oc, seed=5, **extra)]
        par = list(synth.synthesize_parallel(text, oc, seed=5, encoding=law, **extra))
        assert par == [a.samples.as_g711_bytes(law, fixed)
                       for a in synth.synthesize_parallel(text, oc, seed=5, **extra)]
        f = tmp_path / "o.wav"
        synth.synthesize_to_file(f, text, oc, seed=5, encoding=law, **extra)
        c = _wav_data(f)
        assert c[b"data"] == b"".join(par)
        assert struct.unpack("<HHI", c[b"fmt "][:8]) == ({"mulaw": 7, "alaw": 6}[law], 1,
                                                          extra.get("output_rate", 22050))
    for extra in ({}, {"output_rate": 8000}):
        st = list(synth.synthesize_streamed(text, oc, CS, PAD, seed=5, encoding=law, **extra))
        assert st == [c.as_g711_bytes(law) for c in synth.synthesize_streamed(text, oc, CS, PAD, seed=5, **extra)]
        rb = RealtimeBatch(m, CS, PAD)
        k_enc = rb.add(text, oc, seed=5, encoding=law, **extra)
        k_pcm = rb.add(text, oc, seed=5, **extra)
        items = {k_enc: [], k_pcm: []}
        while len(rb):
            for key, item in rb.step():
                items[key].append(item)
        assert items[k_enc] == st
        assert [c.as_g711_bytes(law) for c in items[k_pcm]] == st
    (tmp_path / "in.txt").write_text(text + "\n", encoding="utf-8")
    for mode in ("lazy", "parallel", "realtime"):
        buf = io.BytesIO()
        req = {"text": text, "mode": mode, "seed": 5, "volume": 60, "encoding": law, "output_rate": 8000,
               "chunk_size": CS, "chunk_padding": PAD}
        cli.process_request(synth, DEFAULT, req, None, buf)
        if mode == "realtime":
            want = [c.as_g711_bytes(law) for c in synth.synthesize_streamed(
                text, AudioOutputConfig(None, 60), CS, PAD, seed=5, output_rate=8000)]
        else:
            want = [a.samples.as_g711_bytes(law) for a in synth.synthesize_parallel(
                text, AudioOutputConfig(None, 60), seed=5, output_rate=8000)]
        assert buf.getvalue() == b"".join(want), mode
        m.set_fallback_synthesis_config(DEFAULT)
    out = tmp_path / "c.wav"
    assert cli.main([voices.paths["medium"], "-f", str(tmp_path / "in.txt"), "-o", str(out), "--encoding", law,
                     "--seed", "5", "--loudness", "-16"]) == 0
    want = b"".join(a.samples.as_g711_bytes(law, True) for a in synth.synthesize_parallel(text + "\n", seed=5,
                                                                                            loudness=-16.0))
    assert _wav_data(out)[b"data"] == want
    m.set_fallback_synthesis_config(DEFAULT)
