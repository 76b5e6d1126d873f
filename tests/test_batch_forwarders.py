"""The narrower batch entry points of include/sonata_b200.h, which the Python package no longer calls: each forwards to
sb200_speak_batch_ids_blends / sb200_encode_batch_ids_blends with nulls in the places it does not take.

- CPU: on a config-only voice, each refuses a bad argument by name before any device work, or (the arguments the
  library checks only once the job exists) reaches the job and reports the config-only voice.
- GPU (-m gpu): for one small batch, seeded where the entry point takes seeds, each gives the same bits as the
  general entry point with the same arguments and nulls elsewhere: samples, rate, frames per id, delivered ends and
  loudness for the f32 route; frames per id and the decoded latent for the encoder."""
import ctypes as C

import numpy as np
import pytest

import sonata_b200
from sonata_b200 import PiperSynthesisConfig, voicegen, workload
from sonata_b200 import _native as N
from sonata_b200.core import OperationError
from sonata_b200.piper import EncoderOutputs, _check, _config_array, _take_audio

# the inputs of each entry point, in its argument order, and its outputs (after `outs`)
SPEAK_IN = ["cfgs", "scales", "frames", "seeds", "seeded", "rates", "lufs", "pitch", "tempo", "contour", "formants",
            "bs", "bw", "bo"]
SPEAK_OUT = ["id_frames", "bounds", "lufs_out", "gain_out"]
SPEAK = {"sb200_speak_batch_ids_configs": (SPEAK_IN[:1], []),
         "sb200_speak_batch_ids_durations": (SPEAK_IN[:3], SPEAK_OUT[:1]),
         "sb200_speak_batch_ids_seeded": (SPEAK_IN[:5], SPEAK_OUT[:1]),
         "sb200_speak_batch_ids_prosody": (SPEAK_IN[:9], SPEAK_OUT[:1] + SPEAK_OUT[2:]),
         "sb200_speak_batch_ids_contour": (SPEAK_IN[:10], SPEAK_OUT),
         "sb200_speak_batch_ids_formants": (SPEAK_IN[:11], SPEAK_OUT)}
ENCODE_IN = SPEAK_IN[:5] + SPEAK_IN[11:]
ENCODE = {"sb200_encode_batch_ids_seeded": ENCODE_IN[:5],
          "sb200_encode_batch_ids_durations": ENCODE_IN[:3],
          "sb200_encode_batch_ids_configs": ENCODE_IN[:1]}

IDS = [workload.synthetic_ids(5, utt=0)[:9], workload.synthetic_ids(7, utt=1)[:13]]
NAN = np.nan


def _inputs(seeded: bool = True):
    """C images of every option for IDS: utterance 0 with a pitch ratio, utterance 1 with a contour and a formant
    ratio; both seeded and scaled.  Unseeded noise moves on with every call of a voice, so without `seeded` the configs
    draw none."""
    n0, n1 = len(IDS[0]), len(IDS[1])
    scales = np.ones(n0 + n1, np.float32)
    scales[2], scales[n0 + 3] = 1.3, 0.7
    frames = np.full(n0 + n1, -1, np.int32)
    frames[n0 + 5] = 4
    contour = np.full(n0 + n1, NAN, np.float32)
    contour[n0 + 2:n0 + 8] = 1.25
    noise = (0.5, 0.6) if seeded else (0.0, 0.0)
    return {"cfgs": _config_array([PiperSynthesisConfig(1, noise[0], 1.1, noise[1]),
                                   PiperSynthesisConfig(None, noise[0], 1.0, noise[1])], 2),
            "scales": scales, "frames": frames, "seeds": np.array([11, 2**63 + 5], np.uint64),
            "seeded": np.array([1, 1], np.int32), "rates": np.array([16000, 0], np.uint32),
            "lufs": np.array([-20.0, -23.0], np.float32), "pitch": np.array([1.2, NAN], np.float32),
            "tempo": np.array([NAN, 1.1], np.float32), "contour": contour,
            "formants": np.array([NAN, 1.1], np.float32), "bs": np.array([0, 2], np.int64),
            "bw": np.array([0.25, 0.75], np.float32), "bo": np.array([0, 2, 2], np.uint64)}


def _c(x):
    if x is None or not isinstance(x, np.ndarray):
        return x
    return x.ctypes.data_as(C.POINTER(np.ctypeslib.as_ctypes_type(x.dtype)))


def _packed():
    ids = np.ascontiguousarray(np.concatenate([np.asarray(b, np.int64) for b in IDS]))
    offs = np.array([0, len(IDS[0]), len(IDS[0]) + len(IDS[1])], np.uint64)
    return ids, offs


def _speak(m, name, vals, outputs):
    """(rc, error, audio list, {output: array}) of one f32 entry point with `vals` in the places it takes."""
    ins = SPEAK[name][0] if name in SPEAK else SPEAK_IN
    ids, offs = _packed()
    total = ids.size
    outs = (N.sb200_audio * 2)()
    res = {"id_frames": np.zeros(total, np.int32), "bounds": np.zeros(total, np.int64),
           "lufs_out": np.zeros(2, np.float64), "gain_out": np.zeros(2, np.float32)}
    res = {k: v for k, v in res.items() if k in outputs}
    err = N.sb200_error()
    rc = getattr(m._lib, name)(m._h, _c(ids), _c(offs), 2, *[_c(vals.get(k)) for k in ins], outs,
                               *[_c(res.get(k)) for k in (SPEAK[name][1] if name in SPEAK else SPEAK_OUT)],
                               C.byref(err))
    return rc, err, outs, res


def _encode(m, name, vals):
    ins = ENCODE[name] if name in ENCODE else ENCODE_IN
    ids, offs = _packed()
    outs = (C.c_void_p * 2)()
    err = N.sb200_error()
    rc = getattr(m._lib, name)(m._h, _c(ids), _c(offs), 2, *[_c(vals.get(k)) for k in ins], outs, C.byref(err))
    return rc, err, outs


# ------------------------------------------------------------------------------------------------ CPU
@pytest.fixture(scope="module")
def config_only(lib_built):
    m = sonata_b200.VitsStreamingModel(voicegen.write_voice(voicegen.default_voice_dir(), "medium", n_speakers=4),
                                       device=-1)
    yield m
    m.close()


# the argument each entry point refuses by name before any device work; the others take none checked that early
BAD = {"sb200_speak_batch_ids_prosody": ("tempo", np.array([NAN, 9.0], np.float32), "utterance 1: tempo ratio 9"),
       "sb200_speak_batch_ids_contour": ("contour", None, "utterance 1, id 3: pitch ratio 3"),
       "sb200_speak_batch_ids_formants": ("formants", np.array([0.1, NAN], np.float32),
                                          "utterance 0: formant ratio 0.1")}


@pytest.mark.parametrize("name", list(SPEAK) + list(ENCODE))
def test_each_forwarder_refuses_by_name_on_a_config_only_voice(config_only, name):
    vals = {} if name in ENCODE else {k: v for k, v in _inputs().items() if k in SPEAK[name][0]}
    msg = "voice was loaded config-only"
    if name in BAD:
        key, bad, msg = BAD[name]
        if key == "contour":
            bad = vals["contour"].copy()
            bad[len(IDS[0]) + 3] = 3.0
        vals[key] = bad
    rc, err = (_encode(config_only, name, vals) if name in ENCODE else _speak(config_only, name, vals, []))[:2]
    with pytest.raises(OperationError, match=msg):
        _check(rc, err)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def voice(lib_built):
    m = sonata_b200.VitsStreamingModel(voicegen.write_voice(voicegen.default_voice_dir(), "medium", n_speakers=4),
                                       device=0)
    m.set_backend(1)
    yield m
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SPEAK) + list(ENCODE))
def test_each_forwarder_gives_the_general_entry_points_bits(voice, name):
    if name in ENCODE:
        vals = {k: v for k, v in _inputs("seeds" in ENCODE[name]).items() if k in ENCODE[name]}
        got, want = (_encode(voice, n, vals) for n in (name, "sb200_encode_batch_ids_blends"))
        _check(*got[:2])
        _check(*want[:2])
        for a, b in zip(got[2], want[2]):
            a, b = EncoderOutputs(voice, C.c_void_p(a)), EncoderOutputs(voice, C.c_void_p(b))
            assert np.array_equal(a.p_duration, b.p_duration)
            x, y = a.infer_decoder().as_slice(), b.infer_decoder().as_slice()
            assert x.shape == y.shape and np.array_equal(x.view(np.uint32), y.view(np.uint32))
        return
    ins, outputs = SPEAK[name]
    vals = {k: v for k, v in _inputs("seeds" in ins).items() if k in ins}
    got, want = _speak(voice, name, vals, outputs), _speak(voice, "sb200_speak_batch_ids_blends", vals, outputs)
    _check(*got[:2])
    _check(*want[:2])
    for a, b in zip(got[2], want[2]):
        a, b = _take_audio(a), _take_audio(b)
        assert a.info.sample_rate == b.info.sample_rate
        x, y = a.samples.as_slice(), b.samples.as_slice()
        assert x.shape == y.shape and np.array_equal(x.view(np.uint32), y.view(np.uint32))
    for k in outputs:
        assert np.array_equal(got[3][k], want[3][k], equal_nan=got[3][k].dtype.kind == "f"), k
