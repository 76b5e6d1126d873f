"""Synthetic Piper-architecture voice writer (numpy only; no oracle, no torch).

The reference loads ``<voice>.onnx`` + ``<voice>.onnx.json`` (``piper/src/lib.rs:88-110``).
Real Piper voices are not available offline, so benchmarks and parity tests run on a
*synthetic* voice of the same architecture as en_US-lessac-medium / en_US-ryan-high:
seeded Gaussian weights, each tensor multiplied by a per-tensor gain.  The gains were
fitted once by ``oracle/calibrate.py`` (activations O(1) through all ~60 layers, mean
duration ~3 frames per id) and are committed as ``sonata_b200/data/gains_<quality>.json``
so the generator itself needs nothing but numpy and is bit-reproducible on any box.

Tensor names and shapes follow Piper's ``SynthesizerTrn`` state dict (weight-norm folded).
"""
from __future__ import annotations

import json
import os
import zlib
from collections import OrderedDict

import numpy as np

from .svw import write_svw

ARCH = {
    "medium": dict(
        hidden=192, inter=192, filter=768, heads=2, layers=6, kernel=3, window=4, n_vocab=256,
        resblock=2, res_kernels=(3, 5, 7), res_dils=((1, 2), (2, 6), (3, 12)),
        up_rates=(8, 8, 4), up_kernels=(16, 16, 8), up_init=256,
        flow_n=4, wn_layers=4, flow_kernel=5, dp_kernel=3, dp_bins=10,
        sample_rate=22050,
    ),
    "high": dict(
        hidden=192, inter=192, filter=768, heads=2, layers=6, kernel=3, window=4, n_vocab=256,
        resblock=1, res_kernels=(3, 7, 11), res_dils=((1, 3, 5), (1, 3, 5), (1, 3, 5)),
        up_rates=(8, 8, 2, 2), up_kernels=(16, 16, 4, 4), up_init=512,
        flow_n=4, wn_layers=4, flow_kernel=5, dp_kernel=3, dp_bins=10,
        sample_rate=22050,
    ),
}
# Piper's x_low: the medium decoder behind a 96-wide text encoder and flow (48-wide attention heads), at 16 kHz.
ARCH["x_low"] = dict(ARCH["medium"], hidden=96, inter=96, filter=384, sample_rate=16000)
# Piper's low: the medium architecture at 16 kHz.  Same tensors as medium, so it shares medium's gains.
ARCH["low"] = dict(ARCH["medium"], sample_rate=16000)
_GAINS_OF = {"low": "medium"}

_DATA_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data")


def tensor_specs(a: dict) -> "OrderedDict[str, tuple]":
    """name -> (shape, kind).  kind: 'w' conv/linear weight (fan-in scaled normal),
    'b' bias, 'g' LayerNorm gamma, 'bt' LayerNorm beta, 'emb', 'rel', 'ea'."""
    H, F, I = a["hidden"], a["filter"], a["inter"]
    s: "OrderedDict[str, tuple]" = OrderedDict()
    s["enc_p.emb.weight"] = ((a["n_vocab"], H), "emb")
    kc = H // a["heads"]
    for i in range(a["layers"]):
        p = f"enc_p.encoder.attn_layers.{i}."
        for c in ("conv_q", "conv_k", "conv_v", "conv_o"):
            s[p + c + ".weight"] = ((H, H, 1), "w")
            s[p + c + ".bias"] = ((H,), "b")
        s[p + "emb_rel_k"] = ((1, 2 * a["window"] + 1, kc), "rel")
        s[p + "emb_rel_v"] = ((1, 2 * a["window"] + 1, kc), "rel")
        s[f"enc_p.encoder.norm_layers_1.{i}.gamma"] = ((H,), "g")
        s[f"enc_p.encoder.norm_layers_1.{i}.beta"] = ((H,), "bt")
        p = f"enc_p.encoder.ffn_layers.{i}."
        s[p + "conv_1.weight"] = ((F, H, a["kernel"]), "w")
        s[p + "conv_1.bias"] = ((F,), "b")
        s[p + "conv_2.weight"] = ((H, F, a["kernel"]), "w")
        s[p + "conv_2.bias"] = ((H,), "b")
        s[f"enc_p.encoder.norm_layers_2.{i}.gamma"] = ((H,), "g")
        s[f"enc_p.encoder.norm_layers_2.{i}.beta"] = ((H,), "bt")
    s["enc_p.proj.weight"] = ((2 * I, H, 1), "w")
    s["enc_p.proj.bias"] = ((2 * I,), "b")

    def dds(prefix, ch, k):
        for j in range(3):
            s[f"{prefix}convs_sep.{j}.weight"] = ((ch, 1, k), "w")
            s[f"{prefix}convs_sep.{j}.bias"] = ((ch,), "b")
            s[f"{prefix}convs_1x1.{j}.weight"] = ((ch, ch, 1), "w")
            s[f"{prefix}convs_1x1.{j}.bias"] = ((ch,), "b")
            s[f"{prefix}norms_1.{j}.gamma"] = ((ch,), "g")
            s[f"{prefix}norms_1.{j}.beta"] = ((ch,), "bt")
            s[f"{prefix}norms_2.{j}.gamma"] = ((ch,), "g")
            s[f"{prefix}norms_2.{j}.beta"] = ((ch,), "bt")

    # stochastic duration predictor (inference subset: CF1 = dp.flows.1 is pruned by
    # `flows[:-2] + [flows[-1]]`, post_* are training-only)
    s["dp.pre.weight"] = ((H, H, 1), "w")
    s["dp.pre.bias"] = ((H,), "b")
    dds("dp.convs.", H, a["dp_kernel"])
    s["dp.proj.weight"] = ((H, H, 1), "w")
    s["dp.proj.bias"] = ((H,), "b")
    s["dp.flows.0.m"] = ((2, 1), "ea")
    s["dp.flows.0.logs"] = ((2, 1), "ea")
    nb = 3 * a["dp_bins"] - 1
    for fi in (3, 5, 7):
        p = f"dp.flows.{fi}."
        s[p + "pre.weight"] = ((H, 1, 1), "w")
        s[p + "pre.bias"] = ((H,), "b")
        dds(p + "convs.", H, a["dp_kernel"])
        s[p + "proj.weight"] = ((nb, H, 1), "w")
        s[p + "proj.bias"] = ((nb,), "b")

    # residual coupling flow
    half = I // 2
    for f in range(a["flow_n"]):
        p = f"flow.flows.{2 * f}."
        s[p + "pre.weight"] = ((H, half, 1), "w")
        s[p + "pre.bias"] = ((H,), "b")
        for l in range(a["wn_layers"]):
            s[p + f"enc.in_layers.{l}.weight"] = ((2 * H, H, a["flow_kernel"]), "w")
            s[p + f"enc.in_layers.{l}.bias"] = ((2 * H,), "b")
            rs = 2 * H if l < a["wn_layers"] - 1 else H
            s[p + f"enc.res_skip_layers.{l}.weight"] = ((rs, H, 1), "w")
            s[p + f"enc.res_skip_layers.{l}.bias"] = ((rs,), "b")
        s[p + "post.weight"] = ((half, H, 1), "w")
        s[p + "post.bias"] = ((half,), "b")

    # HiFi-GAN generator
    C = a["up_init"]
    s["dec.conv_pre.weight"] = ((C, I, 7), "w")
    s["dec.conv_pre.bias"] = ((C,), "b")
    nk = len(a["res_kernels"])
    for i, (u, k) in enumerate(zip(a["up_rates"], a["up_kernels"])):
        s[f"dec.ups.{i}.weight"] = ((C, C // 2, k), "wt")  # ConvTranspose1d: [C_in, C_out, k]
        s[f"dec.ups.{i}.bias"] = ((C // 2,), "b")
        C //= 2
        for j, (rk, rd) in enumerate(zip(a["res_kernels"], a["res_dils"])):
            p = f"dec.resblocks.{i * nk + j}."
            if a["resblock"] == 2:
                for m in range(len(rd)):
                    s[p + f"convs.{m}.weight"] = ((C, C, rk), "w")
                    s[p + f"convs.{m}.bias"] = ((C,), "b")
            else:
                for m in range(len(rd)):
                    s[p + f"convs1.{m}.weight"] = ((C, C, rk), "w")
                    s[p + f"convs1.{m}.bias"] = ((C,), "b")
                    s[p + f"convs2.{m}.weight"] = ((C, C, rk), "w")
                    s[p + f"convs2.{m}.bias"] = ((C,), "b")
    s["dec.conv_post.weight"] = ((1, C, 7), "w")
    return s


GIN_CHANNELS = 512      # Piper multi-speaker voices: gin_channels of SynthesizerTrn


def speaker_specs(a: dict, n_speakers: int) -> "OrderedDict[str, tuple]":
    """Extra tensors of a multi-speaker voice (`n_speakers > 1`, piper_train SynthesizerTrn): the speaker embedding and
    the 1x1 conditioning convs applied to g = emb_g(sid): duration predictor (`dp.cond`), every coupling layer's
    WaveNet (`enc.cond_layer`, all layers stacked: 2*hidden*n_layers rows) and the HiFi-GAN input (`dec.cond`)."""
    H, G = a["hidden"], GIN_CHANNELS
    s: "OrderedDict[str, tuple]" = OrderedDict()
    s["emb_g.weight"] = ((n_speakers, G), "embg")
    s["dp.cond.weight"] = ((H, G, 1), "wc")
    s["dp.cond.bias"] = ((H,), "b")
    for f in range(a["flow_n"]):
        p = f"flow.flows.{2 * f}.enc.cond_layer."
        s[p + "weight"] = ((2 * H * a["wn_layers"], G, 1), "wc")
        s[p + "bias"] = ((2 * H * a["wn_layers"],), "b")
    s["dec.cond.weight"] = ((a["up_init"], G, 1), "wc")
    s["dec.cond.bias"] = ((a["up_init"],), "b")
    return s


def _rng(seed: int, name: str) -> np.random.Generator:
    return np.random.Generator(np.random.PCG64([seed, zlib.crc32(name.encode("utf-8"))]))


def base_tensor(seed: int, name: str, shape, kind: str) -> np.ndarray:
    """Un-gained random tensor.  Deterministic in (seed, name) only."""
    r = _rng(seed, name)
    n = r.standard_normal(size=shape, dtype=np.float64)
    if kind == "w":
        fan_in = int(np.prod(shape[1:]))
        v = n / np.sqrt(fan_in)
    elif kind == "wt":  # ConvTranspose1d [C_in, C_out, k]: each output sees C_in * k/stride taps
        fan_in = shape[0] * 2
        v = n / np.sqrt(fan_in)
    elif kind == "b":
        v = 0.1 * n
    elif kind == "g":
        v = 1.0 + 0.1 * n
    elif kind == "bt":
        v = 0.1 * n
    elif kind == "emb":
        v = n / np.sqrt(shape[1])
    elif kind == "rel":
        v = n / np.sqrt(shape[2])
    elif kind == "ea":
        v = 0.1 * n
    elif kind == "embg":
        v = n
    elif kind == "wc":      # conditioning conv: shifts of ~0.4 standard deviations per speaker
        v = 0.4 * n / np.sqrt(shape[1])
    else:
        raise ValueError(kind)
    return v.astype(np.float32)


def hp_tensors(a: dict) -> "OrderedDict[str, np.ndarray]":
    t: "OrderedDict[str, np.ndarray]" = OrderedDict()
    t["hp.arch"] = np.array(
        [a["hidden"], a["inter"], a["filter"], a["heads"], a["layers"], a["kernel"], a["window"],
         a["n_vocab"], a["resblock"], a["up_init"], a["flow_n"], a["wn_layers"], a["flow_kernel"],
         a["dp_kernel"], a["dp_bins"], a["sample_rate"]], dtype=np.int32)
    t["hp.up_rates"] = np.array(a["up_rates"], dtype=np.int32)
    t["hp.up_kernels"] = np.array(a["up_kernels"], dtype=np.int32)
    t["hp.res_kernels"] = np.array(a["res_kernels"], dtype=np.int32)
    t["hp.res_dils"] = np.array(a["res_dils"], dtype=np.int32)
    return t


def load_gains(quality: str) -> dict:
    p = os.path.join(_DATA_DIR, f"gains_{_GAINS_OF.get(quality, quality)}.json")
    if not os.path.exists(p):
        return {}
    with open(p) as f:
        return json.load(f)


def make_tensors(quality: str, seed: int = 1234, gains: dict | None = None, n_speakers: int = 1):
    a = ARCH[quality]
    if gains is None:
        gains = load_gains(quality)
    out = hp_tensors(a)
    specs = tensor_specs(a)
    if n_speakers > 1:
        specs.update(speaker_specs(a, n_speakers))
    for name, (shape, kind) in specs.items():
        t = base_tensor(seed, name, shape, kind)
        g = gains.get(name)
        if g is not None:
            if isinstance(g, dict) and "value" in g:    # explicit override (tiny tensors)
                t = np.asarray(g["value"], dtype=np.float32).reshape(shape)
            elif isinstance(g, dict):                   # per-output-channel gains
                r = np.asarray(g["rows"], dtype=np.float32)
                t = (t * r.reshape((-1,) + (1,) * (t.ndim - 1))).astype(np.float32)
            else:
                t = (t * np.float32(g)).astype(np.float32)
        out[name] = t
    return out


# Piper phoneme_id_map convention: '_' pad = 0, '^' bos = 1, '$' eos = 2, then symbols.
_SYMBOLS = (
    " !\"#$%&'()*+,-./0123456789:;<=>?@ABCDEFGHIJKLMNOPQRSTUVWXYZ[\\]`abcdefghijklmnopqrstuvwxyz"
    "{|}~¡¢£¤¥¦§¨©ª«¬®¯°±²³´µ¶·¸¹º»¼½¾¿æçðøħŋœǀǁǂǃɐɑɒɓɔɕɖɗɘəɚɛɜɞɟɠɡɢɣɤɥɦɧɨɪɫɬɭɮɯɰɱɲɳɴɵɶɸɹɺɻɽɾʀʁʂʃʄʈʉʊʋʌʍʎʏʐʑʒʔʕʘʙʛʜʝʟʡʢˈˌːˑ˞βθχᵻⱱ"
)


def make_config(quality: str, num_symbols: int = 256, streaming: bool = False, n_speakers: int = 1) -> dict:
    """A Piper-style ``*.onnx.json`` (schema: ``piper/src/lib.rs:112-158``)."""
    a = ARCH[quality]
    idmap = {"_": [0], "^": [1], "$": [2]}
    nxt = 3
    for ch in _SYMBOLS:
        if ch in idmap:
            continue
        if nxt >= num_symbols:
            break
        idmap[ch] = [nxt]
        nxt += 1
    return {
        "key": f"synthetic-{quality}",
        "audio": {"sample_rate": a["sample_rate"], "quality": quality},
        "espeak": {"voice": "en-us"},
        "language": {"code": "en_US", "family": "en", "region": "US",
                     "name_native": "English", "name_english": "English"},
        "inference": {"noise_scale": 0.667, "length_scale": 1.0, "noise_w": 0.8},
        "num_symbols": num_symbols,
        "num_speakers": n_speakers,
        "speaker_id_map": {f"speaker_{i}": i for i in range(n_speakers)} if n_speakers > 1 else {},
        "streaming": streaming,
        "phoneme_map": {},
        "phoneme_id_map": idmap,
    }


def write_voice(dirpath: str, quality: str, seed: int = 1234, name: str | None = None,
                streaming: bool = False, n_speakers: int = 1) -> str:
    """Write ``<dir>/<name>.onnx.json`` + ``<dir>/<name>.svw``; returns the config path.

    The weight file sits where the reference expects ``<name>.onnx`` (config path minus
    ``.json``, ``piper/src/lib.rs:98-108``) with the extension swapped to ``.svw``.
    """
    os.makedirs(dirpath, exist_ok=True)
    name = name or (f"synthetic-{quality}" if n_speakers <= 1 else f"synthetic-{quality}-spk{n_speakers}")
    cfg_path = os.path.join(dirpath, name + ".onnx.json")
    svw_path = os.path.join(dirpath, name + ".svw")
    if not (os.path.exists(cfg_path) and os.path.exists(svw_path)):
        tmp = svw_path + f".tmp{os.getpid()}"
        write_svw(tmp, make_tensors(quality, seed, n_speakers=n_speakers))
        os.replace(tmp, svw_path)
        with open(cfg_path + f".tmp{os.getpid()}", "w", encoding="utf-8") as f:
            json.dump(make_config(quality, streaming=streaming, n_speakers=n_speakers), f, ensure_ascii=False)
        os.replace(cfg_path + f".tmp{os.getpid()}", cfg_path)
    return cfg_path


def default_voice_dir() -> str:
    d = os.environ.get("SONATA_B200_VOICE_DIR")
    if d:
        return d
    return os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", "voices")


if __name__ == "__main__":
    import sys
    q = sys.argv[1] if len(sys.argv) > 1 else "medium"
    print(write_voice(default_voice_dir(), q))
