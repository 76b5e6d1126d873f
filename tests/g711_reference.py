"""G.711 restated as two 65 536-entry tables, built value by value from ITU-T G.711's segment definition, for the
tests.  `encode(x, law)` maps int16 samples to their bytes by table lookup."""
import numpy as np


def _ulaw(x: int) -> int:
    v = x >> 2                         # 14-bit range
    mask = 0xFF if v >= 0 else 0x7F    # one's complement; a positive sample keeps bit 7 set
    v = min(abs(v), 8159) + 33         # biased magnitude, 33 .. 8192
    if v >= 8192:
        return 0x7F ^ mask
    seg = max(v.bit_length() - 6, 0)
    mant = (v >> (seg + 1)) & 0xF
    return ((seg << 4) | mant) ^ mask


def _alaw(x: int) -> int:
    v = x >> 3                         # 13-bit range
    if v >= 0:
        mask = 0xD5
    else:
        mask, v = 0x55, -v - 1
    seg = max(v.bit_length() - 5, 0)
    mant = (v >> (seg if seg >= 2 else 1)) & 0xF
    return ((seg << 4) | mant) ^ mask


VALUES = np.arange(-32768, 32768, dtype=np.int32)
TABLES = {
    "mulaw": np.array([_ulaw(int(x)) for x in VALUES], dtype=np.uint8),
    "alaw": np.array([_alaw(int(x)) for x in VALUES], dtype=np.uint8),
}
SILENCE = {"mulaw": 0xFF, "alaw": 0xD5}


def encode(x, law: str) -> np.ndarray:
    x = np.asarray(x, dtype=np.int16).astype(np.int32).reshape(-1)
    return TABLES[law][x + 32768]


def encode_bytes(x, law: str) -> bytes:
    return encode(x, law).tobytes()
