"""Piper's 16 kHz qualities on the CPU: x_low (hidden = inter = 96, filter 384, 48-wide attention heads, the medium
decoder) and low (the medium architecture at 16 kHz).

* the oracle against transformers' `VitsModel` on x_low, up to the latent z (transformers has no ResBlock2 vocoder);
* the oracle against the committed goldens of tests/golden/qualities/ (generator alongside);
* the voice writer and the ONNX importer for both qualities, with architecture detection that does not depend on the
  order of `voicegen.ARCH`;
* the launch planners over every x_low conv layer, the zero-padded coupling layers included."""
import ctypes as C
import glob
import json
import os
import sys
import zlib
from collections import OrderedDict

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from oracle import vits_oracle as vo  # noqa: E402
from sonata_b200 import onnx_import, voicegen  # noqa: E402
from sonata_b200.svw import read_svw  # noqa: E402
from test_planner import two_stages_fit  # noqa: E402

QGOLD = sorted(glob.glob(os.path.join(HERE, "golden", "qualities", "*.npz")))


def _crc(t):
    c = 0
    for k in sorted(t):
        c = zlib.crc32(np.ascontiguousarray(t[k]).tobytes(), c)
    return c


def test_quality_goldens_present():
    assert {str(np.load(p)["quality"]) for p in QGOLD} == {"x_low", "low"} and len(QGOLD) == 4


@pytest.mark.parametrize("path", QGOLD, ids=[os.path.basename(p) for p in QGOLD])
def test_oracle_reproduces_quality_golden(path):
    g = np.load(path)
    q = str(g["quality"])
    t = voicegen.make_tensors(q)
    assert _crc(t) == int(g["weights_crc"]), "synthetic voice generator drifted"
    st = {}
    ew = torch.from_numpy(g["eps_w"].T[None].copy()) if "eps_w" in g else None
    ez = torch.from_numpy(g["eps_z"].T[None].copy()) if "eps_z" in g else None
    wav = vo.infer(vo.to_torch(t), g["ids"], [float(s) for s in g["scales"]], eps_w=ew, eps_z=ez, stages=st)
    assert st["y_len"] == int(g["y_len"])
    assert np.array_equal(np.cumsum(st["w_ceil"].view(-1).numpy()).astype(np.int32), g["cum"])
    assert wav.numel() == 256 * int(g["y_len"])
    assert float(np.abs(wav.numpy() - g["wav"]).max()) < 2e-5


def test_x_low_up_to_the_vocoder_against_live_transformers_run():
    """Text encoder (48-wide heads), duration predictor, alignment and flow of the x_low voice against
    `VitsModelOutput.spectrogram`: deterministic, and stochastic with transformers' own draws replayed."""
    pytest.importorskip("transformers")
    import hf_reference as hf
    a = voicegen.ARCH["x_low"]
    T = voicegen.make_tensors("x_low")
    m = hf.load_piper_tensors(hf.build_hf_model(a, decoder=False), T, a, decoder=False)
    W = vo.to_torch(T)
    ids = vo.synthetic_ids(40, utt=3)
    for scales, seed in (((0.0, 1.0, 0.0), 0), ((0.667, 1.1, 0.8), 9)):
        _, ew, ez = hf.hf_infer(m, ids, *scales, seed=seed)
        z_hf = hf.hf_infer.last_spectrogram
        st = {}
        vo.encode(W, ids, list(scales), eps_w=ew[None] if scales[2] else None, eps_z=ez[None] if scales[0] else None, stages=st)
        z = st["z"][0].numpy()
        assert z.shape == z_hf.shape, (scales, z.shape, z_hf.shape)           # identical frame count
        assert float(np.abs(z - z_hf).max()) < 5e-5, scales


def test_x_low_and_low_voices():
    """x_low has the stated shapes and ~5 M parameters (Piper's x_low files are ~20 MB of fp32); low is medium's tensors
    with a 16 kHz header and shares medium's gains; configs carry Piper's quality names and the voice's own rate; the
    medium and high generators are untouched (their goldens pin them bit for bit, tests/test_oracle.py)."""
    x = voicegen.make_tensors("x_low")
    n = sum(v.size for k, v in x.items() if not k.startswith("hp."))
    assert 4.9e6 < n < 5.2e6, n
    assert x["enc_p.emb.weight"].shape == (256, 96) and x["enc_p.proj.weight"].shape == (192, 96, 1)
    assert x["flow.flows.0.pre.weight"].shape == (96, 48, 1) and x["flow.flows.0.post.weight"].shape == (48, 96, 1)
    assert x["dec.conv_pre.weight"].shape == (256, 96, 7) and x["hp.arch"][-1] == 16000
    low, med = voicegen.make_tensors("low"), voicegen.make_tensors("medium")
    assert list(low) == list(med)
    for k in med:
        if k == "hp.arch":
            assert low[k][-1] == 16000 and med[k][-1] == 22050 and np.array_equal(low[k][:-1], med[k][:-1])
        else:
            assert np.array_equal(low[k], med[k]), k
    assert voicegen.load_gains("low") == voicegen.load_gains("medium")
    assert not os.path.exists(os.path.join(voicegen._DATA_DIR, "gains_low.json"))
    for q, sr in (("x_low", 16000), ("low", 16000), ("medium", 22050), ("high", 22050)):
        assert voicegen.make_config(q)["audio"] == {"sample_rate": sr, "quality": q}


def _onnx_voice(tmp_path, quality, seed=77):
    """An ONNX file of initialisers only (the importer reads nothing else) and its config, via the writer of
    tests/test_onnx_import.py's wire format."""
    from test_onnx_import import _model, _tensor
    tensors = voicegen.make_tensors(quality, seed)
    blobs = [_tensor(k, v, ("raw", "float_data", "packed_dims")[i % 3])
             for i, (k, v) in enumerate(tensors.items()) if not k.startswith("hp.")]
    onnx = tmp_path / f"v-{quality}.onnx"
    onnx.write_bytes(_model(blobs))
    cfg = tmp_path / f"v-{quality}.onnx.json"
    cfg.write_text(json.dumps(voicegen.make_config(quality)))
    return str(onnx), str(cfg), tensors


@pytest.mark.parametrize("quality", ["x_low", "low"])
def test_import_roundtrip_16k(tmp_path, quality):
    onnx, cfg, ref = _onnx_voice(tmp_path, quality)
    out_cfg = onnx_import.import_voice(onnx, cfg, str(tmp_path / "out"))
    got = read_svw(out_cfg[:-len(".onnx.json")] + ".svw")
    assert [k for k in got if not k.startswith("hp.")] == list(voicegen.tensor_specs(voicegen.ARCH[quality]))
    for name, a in ref.items():
        assert np.array_equal(got[name], a), name                # hp.* included: 16 kHz header
    c = json.load(open(cfg))
    assert onnx_import.detect_quality(onnx_import.read_initializers(onnx), c) == quality
    # low and medium share every tensor: without quality the sample rate decides, without either 22.05 kHz
    t = onnx_import.read_initializers(onnx)
    if quality == "low":
        assert onnx_import.detect_quality(t, {"audio": {"sample_rate": 16000}}) == "low"
        assert onnx_import.detect_quality(t) == "medium"
    else:
        assert onnx_import.detect_quality(t) == "x_low"


def test_detection_does_not_depend_on_arch_order(tmp_path, monkeypatch):
    files = {q: _onnx_voice(tmp_path, q) for q in ("x_low", "low", "medium", "high")}
    for order in (list(voicegen.ARCH), list(reversed(voicegen.ARCH))):
        monkeypatch.setattr(voicegen, "ARCH", OrderedDict((q, voicegen.ARCH[q]) for q in order))
        for q, (onnx, cfg, _) in files.items():
            assert onnx_import.detect_quality(onnx_import.read_initializers(onnx), json.load(open(cfg))) == q, (order, q)
    t = {"enc_p.emb.weight": np.zeros((256, 128), np.float32), "dec.conv_pre.weight": np.zeros((256, 96, 7), np.float32)}
    with pytest.raises(ValueError, match="encoder width 128.*known: .*x_low=96/256"):
        onnx_import.detect_quality(t)


# ------------------------------------------------------------------------------------------------ launch planners
ROWS = (100, 128, 700, 3000, 20_000, 300_000, 4_000_000)
SMEM_MAX = 227 * 1024
SMS = 132
ACT_NONE, ACT_RELU, ACT_GATE = 0, 1, 2


def _plan(backend, rows, cin, cout, k, dil, act=ACT_NONE, res=0, acc=0):
    from sonata_b200 import _native as N
    o = (C.c_int32 * 16)()
    return None if N.lib().sb200_debug_plan(backend, rows, cin, cout, k, dil, act, res, acc, o) else list(o)


def x_low_tc_layers():
    """(cin, cout, k, dil, act, res, acc) of every bf16x2 tensor-core layer of the x_low voice: the coupling layers with
    pre / post widened to all 96 channels of z (voice.cu), the WaveNet, conv_pre and the medium decoder."""
    a = voicegen.ARCH["x_low"]
    H, I = a["hidden"], a["inter"]
    L = {(I, H, 1, 1, ACT_NONE, 0, 0), (H, 2 * H, a["flow_kernel"], 1, ACT_GATE, 0, 0), (H, 2 * H, 1, 1, ACT_NONE, 0, 1),
         (H, H, 1, 1, ACT_NONE, 0, 1), (H, I, 1, 1, ACT_NONE, 0, 1), (I, a["up_init"], 7, 1, ACT_NONE, 0, 0)}
    ch = a["up_init"]
    for _ in a["up_rates"]:
        ch //= 2
        for k, dils in zip(a["res_kernels"], a["res_dils"]):
            L |= {(ch, ch, k, d, ACT_NONE, 1, acc) for d in dils for acc in (0, 1)}
    return sorted(L)


def x_low_tf_layers():
    """Every 3xTF32 layer: text encoder (qkv, o, ffn, proj) and duration predictor (pre, DDSConv 1x1, proj, the flows'
    29-column projections padded to 32)."""
    a = voicegen.ARCH["x_low"]
    H, F, k = a["hidden"], a["filter"], a["kernel"]
    return [(H, 3 * H, 1, 1, ACT_NONE, 0, 0), (H, H, 1, 1, ACT_NONE, 0, 0), (H, F, k, 1, ACT_RELU, 0, 0),
            (F, H, k, 1, ACT_NONE, 0, 0), (H, 2 * a["inter"], 1, 1, ACT_NONE, 0, 0), (H, 32, 1, 1, ACT_NONE, 0, 0)]


def test_x_low_layers_are_planned_on_tensor_cores():
    for lay in x_low_tc_layers():
        for rows in ROWS:
            p = _plan(1, rows, *lay)
            assert p is not None, (lay, rows)
            nt, wnt, mt, ntn, stages, smem, win = p[:7]
            assert smem <= SMEM_MAX and stages >= 2 and wnt % nt == 0 and nt % 32 == 0, (lay, rows, p)
            if nt < wnt:
                assert mt * ntn <= SMS or not two_stages_fit(win, lay[2], wnt, 1), (lay, rows, p)
    for lay in x_low_tf_layers():
        chunks = set()
        for rows in ROWS:
            p = _plan(2, rows, *lay)
            assert p is not None, (lay, rows)
            nth, wnth, mt, ntn, stages, chunk_kb, smem, win = p[:8]
            chunks.add(chunk_kb)
            assert smem <= SMEM_MAX and stages >= 2 and wnth % nth == 0 and nth in (32, 64, 96), (lay, rows, p)
            if nth < wnth:
                assert mt * (lay[1] // 32) <= SMS or not two_stages_fit(win, lay[2], wnth, 2), (lay, rows, p)
        assert len(chunks) == 1, (lay, chunks)          # the flush chunk follows from the shape alone
    # the unpadded 48-channel halves stay refused: widening them at load time is what puts them on tensor cores
    assert _plan(1, 1000, 48, 96, 1, 1) is None and _plan(1, 1000, 96, 48, 1, 1, acc=1) is None
