"""CPU: G.711 mu-law / A-law encoding.

The library's host encoder (sb200_debug_g711 on device -1) and AudioSamples.as_g711_bytes against a table restatement
of both laws over every 16-bit value (and against audioop where it can still be imported), the known answers, refusals
of bad laws and formats, the G.711 WAV writer field by field, and the synthesizer's modes on a fake model."""
import ctypes as C
import io
import os
import struct
import sys
import warnings

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import g711_reference as gr
from sonata_b200 import Audio, AudioInfo, AudioSamples, OperationError, PhonemizationError
from sonata_b200 import _native as N
from sonata_b200 import cli
from sonata_b200.core import g711_encode, g711_wave_bytes
from sonata_b200.piper import _encoding_list
from sonata_b200.synth import AudioOutputConfig, SonataSpeechSynthesizer

LAWS = {"mulaw": 0, "alaw": 1}


def _hook(law, x, device=-1):
    x = np.ascontiguousarray(x, np.int16)
    out = np.zeros(x.size, np.uint8)
    err = N.sb200_error()
    rc = N.lib().sb200_debug_g711(device, law, x.ctypes.data_as(C.POINTER(C.c_int16)), x.size,
                                  out.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(err))
    msg = ""
    if err.message:
        msg = C.string_at(err.message).decode()
        N.lib().sb200_string_free(err.message)
    return rc, out, msg


@pytest.mark.parametrize("law", ["mulaw", "alaw"])
def test_every_value(lib_built, law):
    x = gr.VALUES.astype(np.int16)
    rc, out, _ = _hook(LAWS[law], x)
    assert rc == 0
    np.testing.assert_array_equal(out, gr.TABLES[law])
    np.testing.assert_array_equal(g711_encode(x, law), gr.TABLES[law])
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", DeprecationWarning)
            import audioop
    except ImportError:
        return
    fn = audioop.lin2ulaw if law == "mulaw" else audioop.lin2alaw
    np.testing.assert_array_equal(np.frombuffer(fn(x.astype("<i2").tobytes(), 2), np.uint8), gr.TABLES[law])


def test_known_answers(lib_built):
    x = np.array([0, 32767, -32768], np.int16)
    assert _hook(0, x)[1].tolist() == [0xFF, 0x80, 0x00]
    assert _hook(1, x)[1].tolist() == [0xD5, 0xAA, 0x2A]
    assert gr.encode(x, "mulaw").tolist() == [0xFF, 0x80, 0x00]
    assert gr.encode(x, "alaw").tolist() == [0xD5, 0xAA, 0x2A]


@pytest.mark.parametrize("fixed", [False, True])
def test_as_g711_bytes_is_the_encoding_of_the_i16_samples(fixed):
    rng = np.random.default_rng(7)
    s = AudioSamples((rng.standard_normal(5000) * 0.3).astype(np.float32))
    for law in ("mulaw", "alaw"):
        i16 = s.to_i16_fixed() if fixed else s.to_i16_vec()
        assert s.as_g711_bytes(law, fixed_scale=fixed) == gr.encode_bytes(i16, law)
    assert AudioSamples([]).as_g711_bytes("alaw") == b""
    assert AudioSamples(np.zeros(3, np.float32)).as_g711_bytes("mulaw") == b"\xff\xff\xff"


def test_bad_laws_are_refused(lib_built):
    for law in (-1, 2, 7):
        rc, _, msg = _hook(law, np.zeros(4, np.int16))
        assert rc == 19 and f"law {law}" in msg
    with pytest.raises(OperationError, match="neither 'mulaw' nor 'alaw'"):
        AudioSamples([0.1]).as_g711_bytes("ulaw")
    with pytest.raises(OperationError, match="utterance 2: encoding 'pcmu'"):
        _encoding_list(["mulaw", "alaw", "pcmu"], 3)
    with pytest.raises(OperationError, match="utterance 0: encoding None"):
        _encoding_list(None, 2)
    with pytest.raises(OperationError, match="3 entries for 2 utterances"):
        _encoding_list(["mulaw"] * 3, 2)
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args(["v.json", "--encoding", "ulaw"])
    synth = SonataSpeechSynthesizer(FakeModel())
    with pytest.raises(OperationError, match="request: encoding 'ulaw'"):
        cli.process_request(synth, None, {"text": "ab", "encoding": "ulaw"}, None, io.BytesIO())
    with pytest.raises(OperationError, match="encoding 'x'"):
        list(synth.synthesize_lazy("ab", encoding="x"))


def _parse_wav(b):
    assert b[:4] == b"RIFF" and b[8:12] == b"WAVE"
    assert struct.unpack("<I", b[4:8])[0] == len(b) - 8
    chunks, pos = {}, 12
    while pos < len(b):
        cid, size = b[pos:pos + 4], struct.unpack("<I", b[pos + 4:pos + 8])[0]
        chunks[cid] = b[pos + 8:pos + 8 + size]
        pos += 8 + size + (size & 1)
    return chunks


@pytest.mark.parametrize("law,tag", [("mulaw", 7), ("alaw", 6)])
@pytest.mark.parametrize("n", [0, 7, 8])
def test_wave_writer(law, tag, n):
    data = bytes(range(n))
    c = _parse_wav(g711_wave_bytes(data, law, 8000))
    assert list(c) == [b"fmt ", b"fact", b"data"]
    assert len(c[b"fmt "]) == 18
    fmt_tag, ch, rate, byte_rate, align, bits, cb = struct.unpack("<HHIIHHH", c[b"fmt "])
    assert (fmt_tag, ch, rate, byte_rate, align, bits, cb) == (tag, 1, 8000, 8000, 1, 8, 0)
    assert struct.unpack("<I", c[b"fact"])[0] == n
    assert c[b"data"] == data


class FakeModel:
    """Sentences of 4 samples per character, a ramp scaled by the sentence's length; streams in two chunks."""

    def audio_output_info(self):
        return AudioInfo(22050, 1, 2)

    def phonemize_text(self, text):
        raise PhonemizationError("no espeak here")

    def _wave(self, ph):
        return (np.linspace(-0.5, 0.8, 4 * len(ph)) * len(ph) / 8).astype(np.float32)

    def speak_one_sentence(self, ph):
        return Audio(self._wave(ph), 22050, 1.0)

    def speak_batch(self, phs, **kw):
        return [Audio(self._wave(p), 22050, 1.0) for p in phs]

    def stream_synthesis(self, ph, chunk_size, chunk_padding, **kw):
        w = self._wave(ph)
        return iter([AudioSamples(w[:len(w) // 2]), AudioSamples(w[len(w) // 2:])])


@pytest.mark.parametrize("law", ["mulaw", "alaw"])
def test_fake_model_modes_are_the_host_encoding(law, tmp_path):
    s = SonataSpeechSynthesizer(FakeModel())
    text = "abc\nde\nfghij"
    cfg = AudioOutputConfig(rate=10, volume=70, pitch=50, appended_silence_ms=10)
    for oc in (None, cfg):
        lazy = list(s.synthesize_lazy(text, oc, encoding=law))
        assert lazy == [a.samples.as_g711_bytes(law) for a in s.synthesize_lazy(text, oc)]
        par = list(s.synthesize_parallel(text, oc, encoding=law))
        assert par == [a.samples.as_g711_bytes(law) for a in s.synthesize_parallel(text, oc)]
        st = list(s.synthesize_streamed(text, oc, 72, 3, encoding=law))
        assert st == [c.as_g711_bytes(law) for c in s.synthesize_streamed(text, oc, 72, 3)]
    assert lazy[0].endswith(bytes([gr.SILENCE[law]]) * 220)
    f = tmp_path / "o.wav"
    s.synthesize_to_file(f, text, cfg, encoding=law)
    c = _parse_wav(f.read_bytes())
    assert c[b"data"] == b"".join(par) and struct.unpack("<I", c[b"fact"])[0] == len(b"".join(par))
    with pytest.raises(OperationError, match="No speech data"):
        s.synthesize_to_file(f, "\n\n", encoding=law)


@pytest.mark.parametrize("mode", ["lazy", "parallel", "realtime"])
def test_cli_writes_the_host_encoding(mode, tmp_path):
    s = SonataSpeechSynthesizer(FakeModel())
    out = io.BytesIO()
    req = {"text": "abc\nde", "mode": mode, "encoding": "alaw", "volume": 40}
    s.model.set_fallback_synthesis_config = lambda c: None
    cli.process_request(s, _Cfg(), req, None, out)
    oc = AudioOutputConfig(None, 40, None, None)
    if mode == "realtime":
        want = b"".join(c.as_g711_bytes("alaw") for c in s.synthesize_streamed("abc\nde", oc, 100, 3))
    else:
        want = b"".join(a.samples.as_g711_bytes("alaw") for a in s.synthesize_lazy("abc\nde", oc))
    assert out.getvalue() == want
    pcm = io.BytesIO()
    cli.process_request(s, _Cfg(), dict(req, encoding="pcm16"), None, pcm)
    assert len(pcm.getvalue()) == 2 * len(want)


class _Cfg:
    noise_scale, length_scale, noise_w = 0.667, 1.0, 0.8
