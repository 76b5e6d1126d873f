"""Generates tests/golden/qualities/*.npz from the oracle for Piper's 16 kHz qualities (x_low, low):
    python tests/golden/qualities/make_quality_golden.py
Same contents as tests/golden/make_golden.py (ids, scales, injected noise, cumulative durations, y_len, logw, z, the
waveform, a checksum of the synthetic weights) plus the quality, which the file name cannot carry unambiguously."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(HERE))))
sys.path.insert(0, os.path.dirname(HERE))
from make_golden import weights_crc  # noqa: E402
from oracle import vits_oracle as vo  # noqa: E402
from sonata_b200 import voicegen  # noqa: E402

CASES = (("x_low", 8, False), ("x_low", 6, True), ("low", 7, False), ("low", 5, True))


def main():
    for q, n, noise in CASES:
        t = voicegen.make_tensors(q)
        W = vo.to_torch(t)
        a = vo.arch_of(W)
        ids = vo.synthetic_ids(n, utt=100 + n)
        scales = [0.667, 1.0, 0.8] if noise else [0.0, 1.0, 0.0]
        g = torch.Generator().manual_seed(2024)
        ew = ez = None
        if noise:
            ew = torch.randn(1, 2, len(ids), generator=g)
            st0 = {}
            vo.encode(W, ids, scales, eps_w=ew, stages=st0)
            ez = torch.randn(1, a["inter"], st0["y_len"], generator=g)
        st = {}
        wav = vo.infer(W, ids, scales, eps_w=ew, eps_z=ez, stages=st)
        out = dict(quality=np.array(q), ids=ids, scales=np.array(scales, np.float32),
                   cum=np.cumsum(st["w_ceil"].view(-1).numpy()).astype(np.int32), y_len=np.int32(st["y_len"]),
                   logw=st["logw"].view(-1).numpy(), z=st["z"][0].T.contiguous().numpy().astype(np.float32),
                   wav=wav.numpy().astype(np.float32), weights_crc=np.uint32(weights_crc(t)))
        if noise:
            out["eps_w"] = ew[0].T.contiguous().numpy()
            out["eps_z"] = ez[0].T.contiguous().numpy()
        name = f"{q}_n{n}_{'noise' if noise else 'det'}.npz"
        np.savez_compressed(os.path.join(HERE, name), **out)
        print(name, "samples", wav.numel(), "y_len", st["y_len"])


if __name__ == "__main__":
    main()
