"""The emission rule of a stream with a formant ratio (include/sonata_b200.h, sb200_prosody_stream_create_formant) in
Python: what each chunk emits and how many inputs the formant stage holds between chunks, on top of the pitch stage's
rule (prosody_stream_reference, prosody_contour_stream_reference)."""
import math

import numpy as np

import formant_reference as fr
import prosody_contour_reference as pcr
import prosody_contour_stream_reference as pcs
import prosody_stream_reference as psr

N, H = fr.N, fr.H


def rule(inputs):
    """[dict(emitted, inputs, held)] of the formant stage fed inputs[k] new samples per chunk, the last chunk ending
    it: a chunk before the last emits every hop whose 4 frames lie inside its G inputs, the last one everything."""
    G = E = 0
    out = []
    for i, g in enumerate(inputs):
        last = i + 1 == len(inputs)
        G += int(g)
        E0 = E
        if last:
            E, held = G, 0
        else:
            E = H * max(0, (G - (N - H)) // H)
            held = G - max(0, E - 3 * H)
        out.append(dict(emitted=E - E0, inputs=G, held=held))
    return out


def _asked(v):
    return v is not None and not math.isnan(float(v)) and float(v) != 1.0


def stream(rate, pitch, tempo, phi, chunk_lens, ends=None, ratios=None):
    """[dict(emitted, ...)] per chunk of a stream with a pitch ratio and a tempo, or (ends, ratios) a contour over
    n = sum chunk_lens inputs and the tempo, and formant ratio phi.  Without the stage (formant_reference.asks false)
    the pitch stage's counts; a formant-only stream's pitch stage passes its chunks through."""
    lens = [int(c) for c in chunk_lens]
    Q = P = None
    p = pitch
    if ratios is not None:
        n = sum(lens)
        pl = pcr.plan(rate, n, np.asarray(ends, np.int64), np.asarray(ratios, np.float32), tempo)
        if pl["one"] is None:
            Q, P, n2 = pl["Q"], pl["p"], pl["n2"]
            warped = pcs.stream(rate, n, ends, ratios, tempo, lens)
        else:
            p = float(pl["p"][0])
            p = None if p == 1.0 else p
    if Q is None:
        n2 = 1                          # a single ratio runs the stage on every frame or on none
        warped = psr.stream(rate, p, tempo, lens) if _asked(p) or _asked(tempo) else [dict(emitted=c) for c in lens]
    pitch_out = [r["emitted"] for r in warped]
    if not fr.asks(n2, phi, p, Q, P):
        return [dict(emitted=e) for e in pitch_out]
    return rule(pitch_out)


def hold_back_ms(rate):
    """(least, most) formant hold-back in ms at `rate`: G - E is 768 .. 1023 samples."""
    return 1000.0 * (N - H) / rate, 1000.0 * (N - 1) / rate
