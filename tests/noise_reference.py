"""Host restatement of the engine's noise draws (kernels_misc.cu philox_normal4 / randn_seg_kernel) in numpy.

Philox4x32-10 runs in exact integer arithmetic; Box-Muller takes u = ((float)c + 0.5f) * 2^-32 in float32, as the
kernel does, the angle 2*pi*u as the kernel's float32 product, and log / sqrt / sin / cos in float64.  A seeded
utterance's eps_w is tag 0 with 2 columns per id, its eps_z tag 1 with `inter` columns per frame."""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: uint32 [..., 4], key: uint32 [..., 2] (broadcast) -> uint32 [..., 4]."""
    ctr = np.asarray(ctr, np.uint32)
    key = np.asarray(key, np.uint32)
    c = [ctr[..., i].astype(np.uint64) for i in range(4)]
    k0 = np.broadcast_to(key[..., 0], ctr.shape[:-1]).astype(np.uint32)
    k1 = np.broadcast_to(key[..., 1], ctr.shape[:-1]).astype(np.uint32)
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = M0 * c[0]
            p1 = M1 * c[2]
            c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0.astype(np.uint64), p1 & _LO,
                 (p0 >> np.uint64(32)) ^ c[3] ^ k1.astype(np.uint64), p0 & _LO]
            k0 = k0 + W0
            k1 = k1 + W1
    return np.stack([x.astype(np.uint32) for x in c], axis=-1)


def box_muller(bits):
    """uint32 [..., 4] -> float64 [..., 4]: the kernel's four normals, in float64 after the float32 u and angle."""
    u = (bits.astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -32)
    r0 = np.sqrt(-2.0 * np.log(u[..., 0].astype(np.float64)))
    r1 = np.sqrt(-2.0 * np.log(u[..., 2].astype(np.float64)))
    a0 = (np.float32(6.283185307179586) * u[..., 1]).astype(np.float64)
    a1 = (np.float32(6.283185307179586) * u[..., 3]).astype(np.float64)
    return np.stack([r0 * np.cos(a0), r0 * np.sin(a0), r1 * np.cos(a1), r1 * np.sin(a1)], axis=-1)


def seeded_bits(seed: int, tag: int, rows: int, cols: int):
    """Philox outputs of the quads of a seeded [rows][cols] tensor: uint32 [ceil(rows*cols/4)][4]."""
    nq = (rows * cols + 3) // 4
    q = np.arange(nq, dtype=np.uint64)
    ctr = np.stack([(q & _LO).astype(np.uint32), (q >> np.uint64(32)).astype(np.uint32),
                    np.full(nq, tag, np.uint32), np.zeros(nq, np.uint32)], axis=-1)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], np.uint32)
    return philox4x32_10(ctr, key)


def seeded_normals(seed: int, tag: int, rows: int, cols: int):
    """A seeded utterance's noise tensor [rows][cols] in float64 (tag 0: eps_w, cols 2; tag 1: eps_z, cols inter)."""
    return box_muller(seeded_bits(seed, tag, rows, cols)).reshape(-1)[:rows * cols].reshape(rows, cols)


def eps_w(seed: int, n_ids: int):
    return seeded_normals(seed, 0, n_ids, 2)


def eps_z(seed: int, n_frames: int, inter: int):
    return seeded_normals(seed, 1, n_frames, inter)
