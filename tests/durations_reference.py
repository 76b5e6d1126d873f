"""The oracle's whole path with per-id duration controls.

`infer` restates `oracle.vits_oracle.infer` stage for stage, calling the oracle's own functions, and changes only the
rounding step: `dur_scale` multiplies the predicted durations before their ceil, and `w_ceil` replaces the rounded
durations outright.  Without controls it computes exactly what the oracle computes
(tests/test_durations_host.py checks that, bit for bit)."""
import numpy as np
import torch

from oracle import vits_oracle as vo


def durations(logw, length_scale, dur_scale=None, w_ceil=None):
    w = torch.exp(logw) * length_scale
    if dur_scale is not None:
        w = w * torch.as_tensor(dur_scale, dtype=w.dtype).view_as(w)
    w_ceil = torch.ceil(w) if w_ceil is None else torch.as_tensor(w_ceil, dtype=w.dtype).view_as(w)
    y_len = int(torch.clamp_min(torch.sum(w_ceil), 1).item())
    return w, w_ceil, y_len


def encode(W, ids, scales, eps_w=None, eps_z=None, stages=None, sid=None, dur_scale=None, w_ceil=None):
    """vo.encode with the controls; scales = [noise_scale, length_scale, noise_w]."""
    a = vo.arch_of(W)
    noise_scale, length_scale, noise_w = (float(s) for s in scales)
    ids = torch.as_tensor(np.asarray(ids, dtype=np.int64)).view(1, -1)
    T = ids.shape[1]
    dt = W["enc_p.emb.weight"].dtype
    x, m_p, logs_p = vo.text_encoder(W, ids, a, None, stages)
    eps_w = torch.zeros(1, 2, T, dtype=dt) if eps_w is None else torch.as_tensor(eps_w).to(dt).view(1, 2, T)
    g = vo.speaker_embedding(W, sid)
    logw = vo.sdp_reverse(W, x, eps_w, noise_w, a, None, stages, g=g)
    w, w_ceil, y_len = durations(logw, length_scale, dur_scale, w_ceil)
    if eps_z is not None:
        eps_z = torch.as_tensor(eps_z).to(dt).view(1, a["inter"], y_len)
    z_p, tok = vo.expand(m_p, logs_p, w_ceil, y_len, eps_z, noise_scale)
    z = vo.flow_reverse(W, z_p, a, None, stages, g=g)
    if stages is not None:
        stages.update({"x": x, "m_p": m_p, "logs_p": logs_p, "logw": logw, "w": w,
                       "w_ceil": w_ceil, "y_len": y_len, "z_p": z_p, "z": z, "tok": tok})
    return z


def infer(W, ids, scales, eps_w=None, eps_z=None, stages=None, sid=None, dur_scale=None, w_ceil=None):
    """vo.infer with the controls: the waveform as a flat tensor."""
    with torch.inference_mode():
        z = encode(W, ids, scales, eps_w, eps_z, stages, sid=sid, dur_scale=dur_scale, w_ceil=w_ceil)
        wav = vo.decode(W, z, None, stages, sid=sid)
        if stages is not None:
            stages["wav"] = wav
    return wav.reshape(-1)
