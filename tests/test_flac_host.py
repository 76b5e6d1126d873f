"""Host (no GPU): the FLAC test decoder against the CRCs' check values and small streams assembled field by field here
(every subframe type, a short last frame with a 16-bit block-size field, 11.025 kHz, an escape partition, wasted bits),
its Rice-cost rule, the Python validation and refusals of FLAC output, and the new C prototypes."""
import io
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import flac_reference as fr
from sonata_b200 import AudioInfo, OperationError, PhonemizationError
from sonata_b200 import _native as N
from sonata_b200 import cli
from sonata_b200.core import flac_encode
from sonata_b200.synth import SonataSpeechSynthesizer


class BitWriter:
    def __init__(self):
        self.bits = []

    def put(self, v, n):
        for i in range(n - 1, -1, -1):
            self.bits.append((v >> i) & 1)

    def signed(self, v, n):
        self.put(v & ((1 << n) - 1), n)

    def rice(self, r, k):
        u = 2 * r if r >= 0 else -2 * r - 1
        self.put(0, 0)
        self.bits.extend([0] * (u >> k) + [1])
        self.put(u & ((1 << k) - 1), k)

    def pad(self):
        while len(self.bits) % 8:
            self.bits.append(0)

    def bytes(self):
        assert len(self.bits) % 8 == 0
        return bytes(np.packbits(np.array(self.bits, np.uint8)))


def streaminfo(rate, total, min_frame=0, max_frame=0, block=4096):
    w = BitWriter()
    w.put(block, 16); w.put(block, 16); w.put(min_frame, 24); w.put(max_frame, 24)
    w.put(rate, 20); w.put(0, 3); w.put(15, 5); w.put(total, 36); w.put(0, 128)
    return b"fLaC" + bytes([0x80, 0, 0, 34]) + w.bytes()


def frame(number, n, rate_code, body, rate_hz=None, bs_code=None):
    """One frame: the header with its CRC-8, the subframe written by body(w), padding and CRC-16."""
    w = BitWriter()
    w.put(0xFFF8, 16)
    if bs_code is None:
        bs_code = 12 if n == 4096 else 6 if n <= 256 else 7
    w.put(bs_code, 4); w.put(rate_code, 4); w.put(0, 4); w.put(4, 3); w.put(0, 1)
    assert number < 0x80
    w.put(number, 8)
    if bs_code == 6:
        w.put(n - 1, 8)
    if bs_code == 7:
        w.put(n - 1, 16)
    if rate_code == 13:
        w.put(rate_hz, 16)
    head = w.bytes()
    w.put(fr.crc8(head), 8)
    body(w)
    w.pad()
    b = w.bytes()
    return b + fr.crc16(b).to_bytes(2, "big")


def test_crc_check_values():
    assert fr.crc8(b"123456789") == 0xF4
    assert fr.crc16(b"123456789") == 0xFEE8


def _residual_part(w, res, order, porder, ks, method=0, escape_bits=None):
    w.put(method, 2); w.put(porder, 4)
    n = len(res) + order
    i = 0
    for p, k in enumerate(ks):
        m = (n >> porder) - (order if p == 0 else 0)
        if escape_bits is not None and p == 0:
            w.put(15 if method == 0 else 31, 4 + method); w.put(escape_bits, 5)
            for r in res[i:i + m]:
                w.signed(int(r), escape_bits)
        else:
            w.put(k, 4 + method)
            for r in res[i:i + m]:
                w.rice(int(r), k)
        i += m


def test_decoder_on_assembled_streams():
    rng = np.random.default_rng(5)
    x_const = np.full(4096, -77)
    x_verb = rng.integers(-32768, 32768, 300)          # a short last frame: 16-bit size field
    x_fixed = (np.arange(4096) * 3 - 5000)
    x_lpc = (1000 * np.sin(np.arange(4096) * 0.05)).astype(np.int64)
    coefs, shift = [1500, -750], 10
    frames = [frame(0, 4096, 13, lambda w: (w.put(0, 8), w.signed(-77, 16)), rate_hz=11025)]

    def fixed_body(w):
        w.put(0x08 | 2, 7); w.put(0, 1)
        for v in x_fixed[:2]:
            w.signed(int(v), 16)
        res = fr.fixed_residual(x_fixed, 2)
        _residual_part(w, res, 2, 3, [1] * 8)
    frames.append(frame(1, 4096, 13, fixed_body, rate_hz=11025))

    def lpc_body(w):
        w.put(0x20 | 1, 7); w.put(0, 1)
        for v in x_lpc[:2]:
            w.signed(int(v), 16)
        w.put(11, 4); w.put(shift, 5)
        for q in coefs:
            w.signed(q, 12)
        res = fr.lpc_residual(x_lpc, coefs, shift)
        _residual_part(w, res, 2, 1, [20, 9], method=1, escape_bits=16)
    frames.append(frame(2, 4096, 13, lpc_body, rate_hz=11025))

    def verb_body(w):
        w.put(1, 7); w.put(0, 1)
        for v in x_verb:
            w.signed(int(v), 16)
    frames.append(frame(3, 300, 13, verb_body, rate_hz=11025))
    data = streaminfo(11025, 3 * 4096 + 300, min(map(len, frames)), max(map(len, frames))) + b"".join(frames)
    s = fr.decode(data)
    want = np.concatenate([x_const, x_fixed, x_lpc, x_verb])
    np.testing.assert_array_equal(s.samples, want)
    assert (s.sample_rate, s.channels, s.bits, s.total, s.md5) == (11025, 1, 16, 3 * 4096 + 300, bytes(16))
    assert [f.type for f in s.frames] == ["CONSTANT", "FIXED", "LPC", "VERBATIM"]
    assert [f.bs_code for f in s.frames] == [12, 12, 12, 7]
    assert all(f.sample_rate == 11025 for f in s.frames)
    lp = s.frames[2]
    assert (lp.order, lp.precision, lp.shift, lp.coefs, lp.method, lp.porder, lp.escapes) == (2, 12, 10, coefs, 1, 1, 1)
    assert s.frames[1].residual_bits == 6 + 8 * 4 + sum(int(u >> 1) + 2 for u in fr.zigzag(fr.fixed_residual(x_fixed, 2)))
    # one flipped bit breaks a CRC
    bad = bytearray(data)
    bad[len(data) - 10] ^= 0x10
    with pytest.raises(fr.FlacError, match="CRC-16"):
        fr.decode(bytes(bad))
    bad = bytearray(data)
    bad[42 + 4] ^= 0x01                                       # the frame number
    with pytest.raises(fr.FlacError, match="CRC-8"):
        fr.decode(bytes(bad))


def test_decoder_short_frames_and_wasted_bits():
    x = np.array([4, 8, -12, 16, 20, 24, 28], np.int64)      # wasted bits: 2

    def body(w):
        w.put(1, 7); w.put(1, 1); w.put(1, 2)                  # VERBATIM, wasted-bits flag, unary 1 -> 2 bits
        for v in x >> 2:
            w.signed(int(v), 14)
    data = streaminfo(8000, 7) + frame(0, 7, 4, body)
    s = fr.decode(data)
    np.testing.assert_array_equal(s.samples, x)
    assert s.frames[0].wasted == 2 and s.frames[0].bs_code == 6
    assert fr.decode(streaminfo(48000, 0)).samples.size == 0


def test_rice_cost_rule():
    r = np.array([0, -1, 1, 5, -7, 2, 0, 0, 3, -2, 40, -50], np.int64)
    bits, o, ks = fr.rice_cost(r, 0)
    u = fr.zigzag(r)
    brute = []
    for po in range(0, 3):
        size = len(r) >> po
        parts = [min(range(31), key=lambda k: (sum(int(v) >> k for v in u[p * size:(p + 1) * size]) + size * (k + 1), k))
                 for p in range(1 << po)]
        tot = sum(sum(int(v) >> k for v in u[p * size:(p + 1) * size]) + size * (k + 1) for p, k in enumerate(parts))
        brute.append((6 + tot + (1 << po) * 4, po, parts))
    assert (bits, o, ks) == min(brute, key=lambda t: (t[0], t[1]))
    # a partition whose optimal parameter exceeds 14 costs 5 bits per parameter
    big = np.full(16, 1 << 20, np.int64)
    assert fr.rice_cost(big, 0)[0] == 6 + 5 + 16 * ((2 << 20 >> 20) + 21)
    # the warm-up samples are not coded: partition 0 holds (n >> o) - order residuals
    res = fr.fixed_residual(np.arange(32) * 7, 2)
    assert res.tolist() == [0] * 30
    assert fr.rice_cost(res, 2) == (6 + 4 + 30, 0, [0])


def test_flac_encode_validation():
    x = np.zeros(10, np.int16)
    for rate in (0, 12000, 96000, 22050.0, True, "8000"):
        with pytest.raises(OperationError, match="sample rate"):
            flac_encode(x, rate)
    for bad in (np.zeros(10, np.int32), np.zeros(10, np.float32), [0, 1, 2], np.zeros((2, 5), np.int16)):
        with pytest.raises(OperationError, match="int16"):
            flac_encode(bad, 8000)
    with pytest.raises(OperationError, match="device"):
        flac_encode(x, 8000, device=-1)


class FakeModel:
    def audio_output_info(self):
        return AudioInfo(22050, 1, 2)

    def phonemize_text(self, text):
        raise PhonemizationError("no espeak here")


def test_modes_refuse_flac():
    s = SonataSpeechSynthesizer(FakeModel())
    for call, where in ((lambda: list(s.synthesize_lazy("ab", encoding="flac")), "synthesize_lazy"),
                        (lambda: list(s.synthesize_parallel("ab", encoding="flac")), "synthesize_parallel"),
                        (lambda: list(s.synthesize_streamed("ab", encoding="flac")), "synthesize_streamed")):
        with pytest.raises(OperationError, match=re.escape(where) + " cannot deliver 'flac': a FLAC stream is one whole"):
            call()
    # the encodings refused before keep their messages
    for bad in ("ulaw", "pcmu", "x"):
        with pytest.raises(OperationError, match=f"encoding '{bad}' is neither 'mulaw' nor 'alaw'"):
            list(s.synthesize_lazy("ab", encoding=bad))


def test_stream_modes_refuse_flac():
    from sonata_b200.piper import StreamBatch, VitsStreamingModel
    from sonata_b200.synth import RealtimeBatch

    class M(FakeModel):
        pass
    sb = StreamBatch.__new__(StreamBatch)
    sb.model, sb.chunk_size, sb.chunk_padding, sb._pending, sb._active, sb._next_key = M(), 20, 3, [], [], 0
    with pytest.raises(OperationError, match="StreamBatch cannot deliver 'flac'"):
        sb.add("ab", encoding="flac")
    rb = RealtimeBatch.__new__(RealtimeBatch)
    rb.model = M()
    with pytest.raises(OperationError, match="RealtimeBatch cannot deliver 'flac'"):
        rb.add("ab", encoding="flac")
    vm = VitsStreamingModel.__new__(VitsStreamingModel)
    with pytest.raises(OperationError, match="stream_synthesis cannot deliver 'flac'"):
        vm.stream_synthesis("ab", 20, 3, encoding="flac")
    with pytest.raises(OperationError, match="decoder chunk pass cannot deliver 'flac'"):
        vm.infer_decoder_batch([], encoding="flac")


def test_cli_choices():
    assert cli.build_parser().parse_args(["v.json", "--encoding", "flac"]).encoding == "flac"
    with pytest.raises(SystemExit):
        cli.build_parser().parse_args(["v.json", "--encoding", "FLAC"])
    s = SonataSpeechSynthesizer(FakeModel())
    with pytest.raises(OperationError, match="FLAC output is not available in realtime mode"):
        cli.process_request(s, None, {"text": "ab", "mode": "realtime", "encoding": "flac"}, None, io.BytesIO())
    with pytest.raises(OperationError, match="request: encoding 'ulaw'"):
        cli.process_request(s, None, {"text": "ab", "encoding": "ulaw"}, None, io.BytesIO())


def test_prototypes_and_header():
    sig = N.SIGNATURES
    assert "sb200_job_fetch_flac" in sig and "sb200_flac_encode" in sig
    assert len(sig["sb200_job_fetch_flac"][1]) == 5 and len(sig["sb200_flac_encode"][1]) == 7
    h = open(os.path.join(ROOT, "include", "sonata_b200.h"), encoding="utf-8").read()
    assert re.search(r"int32_t sb200_job_fetch_flac\(sb200_job\* job, const float\* gains, uint8_t\*\* outs, "
                     r"size_t\* lens, sb200_error\* err\);", h)
    assert re.search(r"int32_t sb200_flac_encode\(int32_t device, const int16_t\* x, size_t n, uint32_t sample_rate, "
                     r"uint8_t\*\* out, size_t\* len,\s+sb200_error\* err\);", h)


def test_library_exports_the_new_symbols(lib_built):
    lib = N.lib()
    assert hasattr(lib, "sb200_job_fetch_flac") and hasattr(lib, "sb200_flac_encode")


def test_flac_encode_refuses_a_rate_before_device_work(lib_built):
    import ctypes as C
    x = np.zeros(4, np.int16)
    out, n, err = C.POINTER(C.c_uint8)(), C.c_size_t(), N.sb200_error()
    rc = N.lib().sb200_flac_encode(0, x.ctypes.data_as(C.POINTER(C.c_int16)), 4, 12345, C.byref(out), C.byref(n),
                                   C.byref(err))
    assert rc == 19 and b"12345" in C.string_at(err.message)
    N.lib().sb200_string_free(err.message)
