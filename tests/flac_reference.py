"""FLAC (RFC 9639) restated in numpy / Python for the tests: CRC-8 and CRC-16, a decoder of native FLAC streams (every
subframe type, escape partitions and wasted bits included; mono), the optimal Rice cost of a residual by the library's
stated rule, and the fixed and LPC residuals.  Test infrastructure only: nothing here encodes."""
from dataclasses import dataclass, field
from typing import List

import numpy as np

BLOCK_SIZE = 4096
RATE_CODES = {8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10, 11025: 13}
_RATE_TABLE = {1: 88200, 2: 176400, 3: 192000, 4: 8000, 5: 16000, 6: 22050, 7: 24000, 8: 32000, 9: 44100, 10: 48000,
               11: 96000}
_BITS_TABLE = {1: 8, 2: 12, 4: 16, 5: 20, 6: 24, 7: 32}
FIXED_COEFS = {0: [], 1: [1], 2: [2, -1], 3: [3, -3, 1], 4: [4, -6, 4, -1]}


def crc8(data: bytes) -> int:
    """CRC-8, polynomial x^8 + x^2 + x + 1 (0x07), init 0, no reflection."""
    c = 0
    for b in data:
        c ^= b
        for _ in range(8):
            c = ((c << 1) ^ 0x07) & 0xFF if c & 0x80 else (c << 1) & 0xFF
    return c


def crc16(data: bytes) -> int:
    """CRC-16, polynomial x^16 + x^15 + x^2 + 1 (0x8005), init 0, no reflection."""
    c = 0
    for b in data:
        c ^= b << 8
        for _ in range(8):
            c = ((c << 1) ^ 0x8005) & 0xFFFF if c & 0x8000 else (c << 1) & 0xFFFF
    return c


class FlacError(Exception):
    pass


class _Bits:
    """MSB-first bit reader over `data`, with every position's next 32 bits precomputed for speed."""

    def __init__(self, data: bytes, byte_pos: int):
        self.data = data
        bits = np.unpackbits(np.frombuffer(data, np.uint8)).astype(np.uint64)
        padded = np.concatenate([bits, np.zeros(64, np.uint64)])
        win = np.zeros(len(bits) + 1, np.uint64)
        for j in range(32):
            win |= padded[j:j + len(bits) + 1] << np.uint64(31 - j)
        self.win = win.tolist()
        ones = np.flatnonzero(bits)
        nxt = np.full(len(bits) + 1, len(bits), np.int64)
        idx = np.searchsorted(ones, np.arange(len(bits) + 1))
        ok = idx < len(ones)
        nxt[ok] = ones[idx[ok]]
        self.next_one = nxt.tolist()
        self.nbits = len(bits)
        self.pos = 8 * byte_pos

    def read(self, n: int) -> int:
        if n == 0:
            return 0
        if self.pos + n > self.nbits:
            raise FlacError("read past the end of the stream")
        if n <= 32:
            v = self.win[self.pos] >> (32 - n)
        else:
            v = (self.win[self.pos] << (n - 32)) | (self.win[self.pos + 32] >> (64 - n))
        self.pos += n
        return int(v)

    def signed(self, n: int) -> int:
        v = self.read(n)
        return v - (1 << n) if n and v >> (n - 1) else v

    def unary(self) -> int:
        p = self.next_one[self.pos]
        if p >= self.nbits:
            raise FlacError("unterminated unary code")
        q = p - self.pos
        self.pos = p + 1
        return q

    def align(self) -> None:
        self.pos = (self.pos + 7) & ~7


@dataclass
class Frame:
    number: int
    offset: int                 # byte offset in the stream
    size: int                   # bytes, header to CRC-16
    block_size: int
    bs_code: int
    rate_code: int
    sample_rate: int
    header: bytes               # without the CRC-8
    type: str                   # "CONSTANT", "VERBATIM", "FIXED", "LPC"
    order: int = 0
    precision: int = 0
    shift: int = 0
    coefs: List[int] = field(default_factory=list)
    wasted: int = 0
    method: int = -1
    porder: int = -1
    params: List[int] = field(default_factory=list)
    escapes: int = 0
    subframe_bits: int = 0
    residual_bits: int = 0      # from the residual's method bits to its last code


@dataclass
class Stream:
    min_block: int
    max_block: int
    min_frame: int
    max_frame: int
    sample_rate: int
    channels: int
    bits: int
    total: int
    md5: bytes
    samples: np.ndarray
    frames: List[Frame]
    metadata: list


def _residual(r: _Bits, n: int, order: int, f: Frame) -> np.ndarray:
    start = r.pos
    f.method = r.read(2)
    if f.method > 1:
        raise FlacError(f"reserved residual coding method {f.method}")
    f.porder = r.read(4)
    pbits, esc = (4, 15) if f.method == 0 else (5, 31)
    parts = 1 << f.porder
    if n % parts or (n >> f.porder) < order:
        raise FlacError(f"partition order {f.porder} does not fit a block of {n} at order {order}")
    out = np.zeros(n - order, np.int64)
    i = 0
    for p in range(parts):
        m = (n >> f.porder) - (order if p == 0 else 0)
        k = r.read(pbits)
        f.params.append(k)
        if k == esc:
            f.escapes += 1
            w = r.read(5)
            for _ in range(m):
                out[i] = r.signed(w) if w else 0
                i += 1
            continue
        for _ in range(m):
            u = (r.unary() << k) | r.read(k)
            out[i] = (u >> 1) ^ -(u & 1)
            i += 1
    f.residual_bits = r.pos - start
    return out


def _restore(warm: List[int], res: np.ndarray, coefs: List[int], shift: int, n: int) -> List[int]:
    x = list(warm) + [0] * (n - len(warm))
    p = len(coefs)
    for i in range(p, n):
        acc = 0
        for j, q in enumerate(coefs):
            acc += q * x[i - 1 - j]
        x[i] = int(res[i - p]) + (acc >> shift)
    return x


def _frame(r: _Bits, data: bytes, pos: int, info: dict, number_expected: int) -> (Frame, np.ndarray, int):
    r.pos = 8 * pos
    if r.read(15) != 0x7FFC:
        raise FlacError(f"no frame sync at byte {pos}")
    if r.read(1) != 0:
        raise FlacError("variable blocking strategy")
    bs_code, rate_code, ch, bits_code, reserved = r.read(4), r.read(4), r.read(4), r.read(3), r.read(1)
    if reserved or ch != 0:
        raise FlacError(f"reserved bit {reserved} / channel assignment {ch} (mono only)")
    first = r.read(8)
    lead = 0
    while lead < 8 and first & (0x80 >> lead):
        lead += 1
    if lead == 1 or lead > 7:
        raise FlacError("bad coded frame number")
    number = first & (0x7F >> lead) if lead else first
    for _ in range(max(lead - 1, 0)):
        b = r.read(8)
        if b >> 6 != 2:
            raise FlacError("bad coded frame number continuation")
        number = (number << 6) | (b & 0x3F)
    if bs_code == 0:
        raise FlacError("reserved block size code")
    n = {1: 192}.get(bs_code)
    if 2 <= bs_code <= 5:
        n = 576 << (bs_code - 2)
    elif bs_code == 6:
        n = r.read(8) + 1
    elif bs_code == 7:
        n = r.read(16) + 1
    elif bs_code >= 8:
        n = 256 << (bs_code - 8)
    if rate_code == 0:
        rate = info["sample_rate"]
    elif rate_code in _RATE_TABLE:
        rate = _RATE_TABLE[rate_code]
    elif rate_code == 12:
        rate = r.read(8) * 1000
    elif rate_code == 13:
        rate = r.read(16)
    elif rate_code == 14:
        rate = r.read(16) * 10
    else:
        raise FlacError("invalid sample rate code 15")
    bps = info["bits"] if bits_code == 0 else _BITS_TABLE.get(bits_code)
    if bps is None:
        raise FlacError(f"reserved bit depth code {bits_code}")
    hlen = r.pos // 8 - pos
    header = data[pos:pos + hlen]
    if r.read(8) != crc8(header):
        raise FlacError(f"frame {number}: CRC-8 mismatch")
    f = Frame(number, pos, 0, n, bs_code, rate_code, rate, header, "")
    sub0 = r.pos
    if r.read(1):
        raise FlacError("subframe padding bit set")
    t = r.read(6)
    if r.read(1):
        f.wasted = r.unary() + 1
    w = bps - f.wasted
    if t == 0:
        f.type = "CONSTANT"
        x = [r.signed(w)] * n
    elif t == 1:
        f.type = "VERBATIM"
        x = [r.signed(w) for _ in range(n)]
    elif 8 <= t <= 12:
        f.type, f.order = "FIXED", t - 8
        warm = [r.signed(w) for _ in range(f.order)]
        res = _residual(r, n, f.order, f)
        f.coefs = FIXED_COEFS[f.order]
        x = _restore(warm, res, f.coefs, 0, n)
    elif t >= 32:
        f.type, f.order = "LPC", t - 31
        warm = [r.signed(w) for _ in range(f.order)]
        pc = r.read(4)
        if pc == 15:
            raise FlacError("invalid LPC precision")
        f.precision = pc + 1
        f.shift = r.signed(5)
        if f.shift < 0:
            raise FlacError("negative LPC shift")
        f.coefs = [r.signed(f.precision) for _ in range(f.order)]
        res = _residual(r, n, f.order, f)
        x = _restore(warm, res, f.coefs, f.shift, n)
    else:
        raise FlacError(f"reserved subframe type {t}")
    f.subframe_bits = r.pos - sub0
    r.align()
    end = r.pos // 8
    if r.read(16) != crc16(data[pos:end]):
        raise FlacError(f"frame {number}: CRC-16 mismatch")
    f.size = end + 2 - pos
    if number != number_expected:
        raise FlacError(f"frame number {number}, expected {number_expected}")
    return f, np.asarray(x, np.int64) << f.wasted, end + 2


def decode(data: bytes) -> Stream:
    """Parses a native FLAC stream: STREAMINFO, every metadata block header and every frame; checks every CRC."""
    if data[:4] != b"fLaC":
        raise FlacError("no fLaC marker")
    pos, meta, info = 4, [], None
    while True:
        last, btype = data[pos] >> 7, data[pos] & 0x7F
        length = int.from_bytes(data[pos + 1:pos + 4], "big")
        meta.append((btype, length))
        body = data[pos + 4:pos + 4 + length]
        if btype == 0:
            v = int.from_bytes(body[10:18], "big")
            info = dict(min_block=int.from_bytes(body[0:2], "big"), max_block=int.from_bytes(body[2:4], "big"),
                        min_frame=int.from_bytes(body[4:7], "big"), max_frame=int.from_bytes(body[7:10], "big"),
                        sample_rate=v >> 44, channels=((v >> 41) & 7) + 1, bits=((v >> 36) & 31) + 1,
                        total=v & ((1 << 36) - 1), md5=bytes(body[18:34]))
        pos += 4 + length
        if last:
            break
    if info is None:
        raise FlacError("no STREAMINFO")
    frames, parts = [], []
    r = _Bits(data, pos) if pos < len(data) else None
    while pos < len(data):
        f, x, pos = _frame(r, data, pos, info, len(frames))
        frames.append(f)
        parts.append(x)
    samples = np.concatenate(parts) if parts else np.zeros(0, np.int64)
    return Stream(samples=samples, frames=frames, metadata=meta, **info)


def zigzag(r: np.ndarray) -> np.ndarray:
    r = np.asarray(r, np.int64)
    return np.where(r >= 0, 2 * r, -2 * r - 1)


def rice_cost(residual: np.ndarray, order: int):
    """The exact Rice coding cost, in bits, of the residual of a predictor of `order` over a block of
    len(residual) + order samples: for every partition order 0..8 valid for the block (2^o divides it and each
    partition holds more than `order` samples), each partition's minimal-cost parameter k in 0..30 (smallest k on a
    tie), then the minimal total (smallest order on a tie).  The total counts the 2 method bits, 4 order bits, each
    partition's 4-bit parameter (5 bits, method 1, when some k > 14) and every code, (u >> k) + 1 + k bits.
    Returns (bits, partition order, parameters)."""
    u = zigzag(residual)
    n = len(u) + order
    uu = np.concatenate([np.zeros(order, np.int64), u])
    shifted = uu[:, None] >> np.arange(31)[None, :]           # [n, 31]
    best = None
    for o in range(0, 9):
        if n % (1 << o) or (n >> o) <= order:
            break
        size = n >> o
        sums = shifted.reshape(1 << o, size, 31).sum(axis=1)   # warm-up entries are 0
        counts = np.full(1 << o, size, np.int64)
        counts[0] -= order
        costs = sums + counts[:, None] * (np.arange(31)[None, :] + 1)
        ks = costs.argmin(axis=1)                             # first minimum: smallest k
        total = int(costs[np.arange(1 << o), ks].sum())
        pbits = 5 if ks.max() > 14 else 4
        bits = 6 + total + (1 << o) * pbits
        if best is None or bits < best[0]:
            best = (bits, o, [int(k) for k in ks])
    return best


def fixed_residual(x: np.ndarray, order: int) -> np.ndarray:
    return lpc_residual(x, FIXED_COEFS[order], 0)


def lpc_residual(x: np.ndarray, coefs, shift: int) -> np.ndarray:
    """x[i] - ((sum_j coefs[j] x[i-1-j]) >> shift) for i >= len(coefs), in int64."""
    x = np.asarray(x, np.int64)
    p = len(coefs)
    acc = np.zeros(len(x) - p, np.int64)
    for j, q in enumerate(coefs):
        acc += int(q) * x[p - 1 - j:len(x) - 1 - j]
    return x[p:] - (acc >> shift)


def subframe_cost(x: np.ndarray, kind: str, order: int = 0) -> int:
    """The exact bits of a VERBATIM or FIXED subframe of 16-bit samples x (header, warm-up, residual)."""
    if kind == "VERBATIM":
        return 8 + 16 * len(x)
    return 8 + 16 * order + rice_cost(fixed_residual(x, order), order)[0]
