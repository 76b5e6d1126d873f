"""CPU: per-phoneme durations without a GPU.

The oracle's path with per-id duration controls (tests/durations_reference.py) equals the oracle's plain run when the
controls restate it; the phoneme-string -> id map
reports the source character of every id (dropped characters, multi-byte characters, multi-id map entries) on a
config-only voice; and the alignment grouping and argument checks of the Python layer run on a fake model."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import durations_reference as dr
import sonata_b200
from oracle import vits_oracle as vo
from sonata_b200 import OperationError, PhonemeAlignment, PiperSynthesisConfig
from sonata_b200.core import Audio
from sonata_b200.piper import _VitsCommons, _alignment, _duration_arrays


# ---------------------------------------------------------------- oracle
@pytest.mark.parametrize("quality", ["x_low", "medium"])
def test_oracle_controls_that_restate_the_plain_run_change_nothing(oracle_weights, quality):
    W = oracle_weights(quality)
    ids = vo.synthetic_ids(7, utt=11)
    eps_w = torch.from_numpy(np.random.default_rng(3).standard_normal((2, len(ids))).astype(np.float32)).view(1, 2, -1)
    plain = {}
    ref = vo.infer(W, ids, [0.0, 1.1, 0.8], eps_w=eps_w, stages=plain)
    for kw in ({}, {"w_ceil": plain["w_ceil"].clone()}, {"dur_scale": np.ones(len(ids), np.float32)},
               {"dur_scale": np.ones(len(ids), np.float32), "w_ceil": plain["w_ceil"].clone()}):
        st = {}
        got = dr.infer(W, ids, [0.0, 1.1, 0.8], eps_w=eps_w, stages=st, **kw)
        assert torch.equal(got, ref), kw.keys()
        for k in ("logw", "w_ceil", "z_p", "z"):
            assert torch.equal(st[k], plain[k]), (kw.keys(), k)


def test_oracle_fixed_and_scaled_durations(oracle_weights):
    W = oracle_weights("medium")
    ids = vo.synthetic_ids(4, utt=2)
    fixed = torch.tensor([0, 3, 0, 0, 5, 1, 0, 2, 0, 4], dtype=torch.float32)
    st = {}
    wav = dr.infer(W, ids, [0.0, 1.0, 0.0], stages=st, w_ceil=fixed)
    assert st["y_len"] == 15 and wav.numel() == 15 * 256
    assert torch.equal(st["tok"], torch.tensor([1] * 3 + [4] * 5 + [5] + [7] * 2 + [9] * 4))
    st0 = {}
    dr.infer(W, ids, [0.0, 1.0, 0.0], stages=st0, w_ceil=torch.zeros(len(ids)))
    assert st0["y_len"] == 1                                        # every id 0 frames: clamped to one frame
    s = np.array([0, 0.5, 1, 1.7, 3, 1, 1, 2, 0.25, 1], np.float32)
    st1 = {}
    dr.infer(W, ids, [0.0, 1.3, 0.0], stages=st1, dur_scale=s)
    want = torch.ceil((torch.exp(st1["logw"]) * 1.3) * torch.from_numpy(s).view(1, 1, -1))
    assert torch.equal(st1["w_ceil"], want)


# ---------------------------------------------------------------- id map of a config-only voice
@pytest.fixture(scope="module")
def map_model(voice_paths, tmp_path_factory):
    cfg = json.load(open(voice_paths["medium"], encoding="utf-8"))
    cfg["phoneme_id_map"]["a"] = [cfg["phoneme_id_map"]["a"][0], 7, 9]        # a multi-id entry: the first id is used
    d = tmp_path_factory.mktemp("idmap")
    path = d / "idmap.onnx.json"
    path.write_text(json.dumps(cfg), encoding="utf-8")
    m = sonata_b200.VitsModel(str(path), device=-1)
    yield m, cfg["phoneme_id_map"]
    m.close()


def test_id_map_reports_each_ids_source_character(map_model):
    m, idmap = map_model
    ph = "a\U0001F600tˈɛ☃s"                # 😀 and ☃ are not in the map and are dropped
    ids, src = m.phonemes_to_input_ids_map(ph)
    assert ids == m.phonemes_to_input_ids(ph)
    kept = [0, 2, 3, 4, 6]                      # character indices (not bytes) of a, t, ˈ, ɛ, s
    assert src == [-1] + [c for c in kept for _ in (0, 1)] + [-1]
    assert ids[0] == idmap["^"][0] and ids[-1] == idmap["$"][0]
    for k, c in enumerate(kept):
        assert ids[1 + 2 * k] == idmap[ph[c]][0] and ids[2 + 2 * k] == idmap["_"][0]
    assert m.phonemes_to_input_ids_map("") == ([idmap["^"][0], idmap["$"][0]], [-1, -1])
    assert m.phonemes_to_input_ids_map("☃") == ([idmap["^"][0], idmap["$"][0]], [-1, -1])


def test_config_only_voice_checks_duration_arguments_before_any_device_call(map_model):
    m, _ = map_model
    with pytest.raises(OperationError, match="utterance 1: 2 duration scales for 3 ids"):
        m.infer_batch_with_durations([[1, 5, 2], [1, 6, 2]], duration_scales=[None, [1.0, 1.0]])
    with pytest.raises(OperationError, match="utterance 0, id 1: duration scale nan"):
        m.infer_batch_with_durations([[1, 5, 2]], duration_scales=[[1.0, float("nan"), 1.0]])
    with pytest.raises(OperationError, match="utterance 0, character 1: duration scale -1.0"):
        m.speak_batch_with_alignment(["at"], duration_scales=[[1.0, -1.0]])
    with pytest.raises(OperationError, match="no CPU path"):
        m.infer_batch_with_durations([[1, 5, 2]], durations=[[0, 3, -1]])


# ---------------------------------------------------------------- argument checks
def test_duration_arrays_pack_and_fill_the_plain_utterances():
    sc, fr = _duration_arrays([3, 2, 1], [None, [0.5, 2], None], [[-1, 0, 7], None, None])
    assert sc.dtype == np.float32 and sc.tolist() == [1, 1, 1, 0.5, 2, 1]
    assert fr.dtype == np.int32 and fr.tolist() == [-1, 0, 7, -1, -1, -1]
    assert _duration_arrays([3], None, None) == (None, None)
    sc, fr = _duration_arrays([2], [np.array([1.0, 3.0], np.float32)], [np.array([4, -1])])
    assert sc.tolist() == [1, 3] and fr.tolist() == [4, -1]


@pytest.mark.parametrize("scales,frames,msg", [
    ([[1.0]], None, "1 duration scales for 2 ids"),
    ([[1.0, 1.0]] * 2, None, "2 entries for 1 utterances"),
    ([[1.0, math.inf]], None, "utterance 0, id 1: duration scale inf"),
    ([[-0.5, 1.0]], None, "utterance 0, id 0: duration scale -0.5"),
    ([[1.0, "x"]], None, "utterance 0, id 1: duration scale 'x' is not a number"),
    ("ab", None, "one entry"),
    (None, [[0, -2]], "utterance 0, id 1: fixed duration -2"),
    (None, [[0, 1.5]], "utterance 0, id 1: fixed duration 1.5 is not an integer"),
    (None, [[3]], "1 durations for 2 ids"),
    (None, [[2**31, 0]], "utterance 0, id 0: fixed duration 2147483648"),
])
def test_duration_argument_errors(scales, frames, msg):
    with pytest.raises(OperationError, match=msg):
        _duration_arrays([2], scales, frames)


# ---------------------------------------------------------------- alignment on a fake model
class FakeModel:
    """Ids: bos 1, (ord(ch) % 50 + 3, pad 0) per character except '~' (dropped), eos 2; every id lasts
    ceil(scale * (id % 4)) frames, or the fixed count."""

    def __init__(self):
        self.calls = []

    def phonemes_to_input_ids_map(self, ph):
        ids, src = [1], [-1]
        for c, ch in enumerate(ph):
            if ch != "~":
                ids += [ord(ch) % 50 + 3, 0]
                src += [c, c]
        return ids + [2], src + [-1]

    def _speak_ids(self, batches, o, frames=False):
        offs = np.cumsum([0] + [len(ids) for ids in batches])
        scales = None if o.scales is None else [o.scales[offs[b]:offs[b + 1]].tolist() for b in range(len(batches))]
        self.calls.append((batches, o.cfgs, scales))
        out = []
        for b, ids in enumerate(batches):
            s = scales[b] if scales else [1.0] * len(ids)
            f = np.array([math.ceil(x * (i % 4)) for i, x in zip(ids, s)], np.int32)
            n = max(int(f.sum()), 1) * 256
            out.append((Audio(np.zeros(n, np.float32), 22050), f, None))
        return out


def test_alignment_groups_ids_by_character_through_the_f32_route():
    fake = FakeModel()
    ph = "ab~c"
    res = _VitsCommons.speak_batch_with_alignment(fake, [ph, "~"], duration_scales=[[2.0, 1.0, float("nan"), 0.5], None])
    (audio, al), (audio2, al2) = res
    ids, src = fake.phonemes_to_input_ids_map(ph)
    assert fake.calls[0][2][0] == [1.0, 2.0, 2.0, 1.0, 1.0, 0.5, 0.5, 1.0]      # the NaN of a dropped character is ignored
    assert fake.calls[0][2][1] == [1.0, 1.0]                                     # bos and eos of "~": no scales
    assert [a.phoneme for a in al] == ["^", "a", "b", "c", "$"]
    assert al[0].start_sample == 0 and all(x.start_sample + x.num_samples == y.start_sample for x, y in zip(al, al[1:]))
    assert al[-1].start_sample + al[-1].num_samples == len(audio)
    frames = [math.ceil(s * (i % 4)) for i, s in zip(ids, fake.calls[0][2][0])]
    assert [a.num_samples for a in al] == [256 * x for x in (frames[0], frames[1] + frames[2], frames[3] + frames[4],
                                                             frames[5] + frames[6], frames[7])]
    assert [a.phoneme for a in al2] == ["^", "$"] and al2[-1].start_sample + al2[-1].num_samples == len(audio2)


def test_alignment_of_an_all_zero_utterance_ends_at_its_one_frame():
    al = _alignment("ab", [-1, 0, 0, 1, 1, -1], [0] * 6, 256)
    assert al == [PhonemeAlignment("^", 0, 0), PhonemeAlignment("a", 0, 0), PhonemeAlignment("b", 0, 0),
                  PhonemeAlignment("$", 0, 256)]
    al = _alignment("ab", [-1, 0, 0, 1, 1, -1], [1, 2, 0, 0, 3, 1], 7 * 512)       # a 512-sample hop is read off
    assert [(a.start_sample, a.num_samples) for a in al] == [(0, 512), (512, 1024), (1536, 1536), (3072, 512)]


def test_alignment_argument_errors_come_before_the_model():
    fake = FakeModel()
    with pytest.raises(OperationError, match="utterance 0: 1 duration scales for 2 characters"):
        _VitsCommons.speak_batch_with_alignment(fake, ["ab"], duration_scales=[[1.0]])
    with pytest.raises(OperationError, match="1 configs for 2 utterances"):
        _VitsCommons.speak_batch_with_alignment(fake, ["a", "b"], configs=[PiperSynthesisConfig()])
    with pytest.raises(OperationError, match="2 entries for 1 utterances"):
        _VitsCommons.speak_batch_with_alignment(fake, ["a"], duration_scales=[None, None])
    assert fake.calls == []
