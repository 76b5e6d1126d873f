"""Piper voice import: ONNX initialisers -> the SVW weight container the library loads (SURVEY §8f row N1).

The reference loads a voice as `<name>.onnx` + `<name>.onnx.json` (crates/sonata/models/piper/src/lib.rs:88-110) and
hands the graph to onnxruntime.  This module reads only what the CUDA path needs from such a file -- the graph's
INITIALISERS (the trained tensors) -- with a small protobuf wire-format reader (no `onnx` package offline), maps them
onto the parameter names of Piper's `SynthesizerTrn` (the names `voicegen.tensor_specs` uses), folds weight
normalisation where the export kept it (`weight_g`, `weight_v` or `parametrizations.weight.original0/1`), checks every
shape against the architecture and writes `<name>.svw` next to a copy of the JSON config.

STATUS: verified on ONNX files produced by the test-suite's own writer (tests/test_onnx_import.py) -- there is no real
Piper voice offline, so the assumptions about upstream's export are listed here and fail loudly when they do not hold:
  * initialisers keep their state-dict names (constant-folded weights would appear as `onnx::Conv_123`: those are
    reported as missing parameters; graph-walking to recover them is not implemented);
  * multi-speaker voices carry `emb_g.weight` [n_speakers, gin] and the conditioning convs `dp.cond`,
    `flow.flows.<2f>.enc.cond_layer` (weight-normed) and `dec.cond` (voicegen.speaker_specs); n_speakers must agree
    with `num_speakers` of the JSON config;
  * fp32 / fp16 / fp64 tensor payloads in `raw_data`, `float_data` or `double_data`; external data is rejected.
"""
from __future__ import annotations

import json
import os
import shutil
import struct
import sys
from typing import Dict, Iterator, Tuple

import numpy as np

from collections import OrderedDict

from . import voicegen
from .svw import write_svw

# ----------------------------------------------------------------------------- protobuf wire format (reader)


def _varint(buf: bytes, i: int) -> Tuple[int, int]:
    shift = v = 0
    while True:
        b = buf[i]
        i += 1
        v |= (b & 0x7F) << shift
        if not b & 0x80:
            return v, i
        shift += 7


def _fields(buf: bytes) -> Iterator[Tuple[int, int, object]]:
    """(field number, wire type, value) for every field of one message; length-delimited values are memoryviews."""
    i, n = 0, len(buf)
    mv = memoryview(buf)
    while i < n:
        key, i = _varint(buf, i)
        fno, wt = key >> 3, key & 7
        if wt == 0:
            v, i = _varint(buf, i)
        elif wt == 1:
            v = bytes(mv[i:i + 8]); i += 8
        elif wt == 2:
            ln, i = _varint(buf, i)
            v = mv[i:i + ln]; i += ln
        elif wt == 5:
            v = bytes(mv[i:i + 4]); i += 4
        else:
            raise ValueError(f"unsupported protobuf wire type {wt}")
        yield fno, wt, v


_DTYPES = {1: np.float32, 10: np.float16, 11: np.float64, 7: np.int64, 6: np.int32}


def _tensor(buf: bytes) -> Tuple[str, np.ndarray]:
    """onnx.TensorProto: dims=1, data_type=2, float_data=4, int64_data=7, name=8, raw_data=9, double_data=10,
    external_data=13, data_location=14."""
    dims, dtype, name = [], 1, ""
    raw = None
    floats, doubles, int64s = [], [], []
    for fno, wt, v in _fields(buf):
        if fno == 1:
            if wt == 0:
                dims.append(int(v))
            else:                                   # packed
                b, i = bytes(v), 0
                while i < len(b):
                    d, i = _varint(b, i)
                    dims.append(d)
        elif fno == 2:
            dtype = int(v)
        elif fno == 8:
            name = bytes(v).decode("utf-8")
        elif fno == 9:
            raw = bytes(v)
        elif fno == 4:
            floats.append(np.frombuffer(bytes(v), dtype="<f4") if wt == 2 else np.frombuffer(v, dtype="<f4"))
        elif fno == 10:
            doubles.append(np.frombuffer(bytes(v), dtype="<f8") if wt == 2 else np.frombuffer(v, dtype="<f8"))
        elif fno == 7:
            if wt == 2:
                b, i = bytes(v), 0
                while i < len(b):
                    d, i = _varint(b, i)
                    int64s.append(d)
            else:
                int64s.append(int(v))
        elif fno in (13, 14) and (fno == 13 or int(v) == 1):
            raise ValueError(f"initialiser `{name}` uses external data: not supported")
    if dtype not in _DTYPES:
        return name, None                            # not a numeric parameter we care about
    if raw is not None:
        arr = np.frombuffer(raw, dtype=np.dtype(_DTYPES[dtype]).newbyteorder("<"))
    elif floats:
        arr = np.concatenate(floats)
    elif doubles:
        arr = np.concatenate(doubles)
    elif int64s:
        arr = np.array(int64s, dtype=np.int64)
    else:
        arr = np.zeros(0, dtype=_DTYPES[dtype])
    return name, np.array(arr).reshape(dims) if dims else np.array(arr).reshape(())


def read_initializers(onnx_path: str) -> Dict[str, np.ndarray]:
    """All numeric initialisers of ModelProto.graph (ModelProto.graph = 7, GraphProto.initializer = 5)."""
    with open(onnx_path, "rb") as f:
        model = f.read()
    out: Dict[str, np.ndarray] = {}
    graphs = [bytes(v) for fno, wt, v in _fields(model) if fno == 7 and wt == 2]
    if not graphs:
        raise ValueError(f"{onnx_path}: no GraphProto found (not an ONNX model?)")
    for fno, wt, v in _fields(graphs[0]):
        if fno == 5 and wt == 2:
            name, arr = _tensor(bytes(v))
            if arr is not None and name:
                out[name] = arr
    return out


# ----------------------------------------------------------------------------- name mapping / weight-norm folding


def _fold_weight_norm(t: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    """`w = g * v / ||v||` with the norm over every axis but 0 (torch.nn.utils.weight_norm, dim=0)."""
    out = dict(t)
    pairs = []
    for k in list(t):
        if k.endswith(".weight_g") and k[:-2] + "_v" in t:
            pairs.append((k[:-len("_g")], k, k[:-2] + "_v"))
        elif k.endswith(".parametrizations.weight.original0") and k[:-1] + "1" in t:
            pairs.append((k[:-len(".parametrizations.weight.original0")] + ".weight", k, k[:-1] + "1"))
    for name, kg, kv in pairs:
        g, v = t[kg].astype(np.float64), t[kv].astype(np.float64)
        nrm = np.sqrt((v * v).sum(axis=tuple(range(1, v.ndim)), keepdims=True))
        out[name] = (g.reshape((-1,) + (1,) * (v.ndim - 1)) * v / nrm).astype(np.float32)
        out.pop(kg, None); out.pop(kv, None)
    return out


def detect_quality(t: Dict[str, np.ndarray], cfg: dict | None = None) -> str:
    """The voice architecture from tensor shapes: the text encoder's width (`enc_p.emb.weight`), then the decoder's
    (`dec.conv_pre`).  Qualities with the same tensors (low and medium) are told apart by the config's
    `audio.quality`, then its `audio.sample_rate`; without a config the 22.05 kHz one is taken."""
    emb, pre = t.get("enc_p.emb.weight"), t.get("dec.conv_pre.weight")
    if emb is None or pre is None:
        raise ValueError("`enc_p.emb.weight` / `dec.conv_pre.weight` not found: initialisers do not carry Piper's "
                         "parameter names")
    shape = (int(emb.shape[-1]), int(pre.shape[0]))
    known = sorted(voicegen.ARCH.items())
    cands = [q for q, a in known if (a["hidden"], a["up_init"]) == shape]
    if not cands:
        raise ValueError(f"unsupported voice architecture: encoder width {shape[0]}, decoder width {shape[1]} (known: " +
                         ", ".join(f"{q}={a['hidden']}/{a['up_init']}" for q, a in known) + ")")
    audio = (cfg or {}).get("audio", {})
    for pick in (lambda q: q == audio.get("quality"),
                 lambda q: voicegen.ARCH[q]["sample_rate"] == audio.get("sample_rate", 22050)):
        hit = [q for q in cands if pick(q)]
        if len(hit) == 1:
            return hit[0]
    if len(cands) == 1:
        return cands[0]
    raise ValueError(f"tensors fit {', '.join(cands)}; the config's audio.quality / sample_rate do not pick one")


def convert_tensors(inits: Dict[str, np.ndarray], cfg: dict | None = None) -> Tuple[str, Dict[str, np.ndarray]]:
    """Initialisers -> exactly the tensors of `voicegen.tensor_specs(arch)`, fp32, shapes verified."""
    t = _fold_weight_norm(inits)
    quality = detect_quality(t, cfg)
    specs = voicegen.tensor_specs(voicegen.ARCH[quality])
    eg = t.get("emb_g.weight")
    if eg is not None:                               # multi-speaker voice
        if eg.ndim != 2 or eg.shape[1] != voicegen.GIN_CHANNELS:
            raise ValueError(f"emb_g.weight has shape {tuple(eg.shape)}; expected [n_speakers, {voicegen.GIN_CHANNELS}]")
        specs.update(voicegen.speaker_specs(voicegen.ARCH[quality], int(eg.shape[0])))
    out, missing, bad = {}, [], []
    for name, (shape, _kind) in specs.items():
        a = t.get(name)
        if a is None:
            missing.append(name)
            continue
        if tuple(a.shape) != tuple(shape):
            bad.append(f"{name}: {tuple(a.shape)} != {tuple(shape)}")
            continue
        out[name] = np.ascontiguousarray(a, dtype=np.float32)
    if missing or bad:
        anon = sum(1 for k in t if k.startswith("onnx::"))
        raise ValueError(f"{len(missing)} parameters missing (first: {missing[:4]}), {len(bad)} with unexpected shapes "
                         f"(first: {bad[:3]}); {anon} anonymous `onnx::*` initialisers present (constant-folded weights "
                         "cannot be mapped by name)")
    return quality, out


def import_voice(onnx_path: str, config_path: str, out_dir: str) -> str:
    """Writes `<out_dir>/<name>.onnx.json` (copy) + `<out_dir>/<name>.svw`; returns the config path to load."""
    with open(config_path) as f:
        cfg = json.load(f)
    quality, tensors = convert_tensors(read_initializers(onnx_path), cfg)
    n_spk = int(tensors["emb_g.weight"].shape[0]) if "emb_g.weight" in tensors else 1
    if int(cfg.get("num_speakers", 1)) > 1 and n_spk < int(cfg["num_speakers"]):
        raise ValueError(f"config says num_speakers = {cfg['num_speakers']} but the model embeds {n_spk} speaker(s)")
    os.makedirs(out_dir, exist_ok=True)
    base = os.path.basename(config_path)
    stem = base[:-len(".onnx.json")] if base.endswith(".onnx.json") else os.path.splitext(base)[0]
    dst_cfg = os.path.join(out_dir, stem + ".onnx.json")
    if os.path.abspath(dst_cfg) != os.path.abspath(config_path):
        shutil.copyfile(config_path, dst_cfg)
    arch = dict(voicegen.ARCH[quality])
    sr = int(cfg.get("audio", {}).get("sample_rate", arch["sample_rate"]))
    arch["sample_rate"] = sr
    blob = voicegen.hp_tensors(arch)                 # the container's hyper-parameter header the loader reads first
    blob.update(tensors)
    write_svw(os.path.join(out_dir, stem + ".svw"), blob)
    return dst_cfg


if __name__ == "__main__":
    if len(sys.argv) != 4:
        sys.exit("usage: python -m sonata_b200.onnx_import <voice.onnx> <voice.onnx.json> <out_dir>")
    print(import_voice(sys.argv[1], sys.argv[2], sys.argv[3]))
