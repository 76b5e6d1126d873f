"""Live loudness on K realtime streams served by one StreamBatch: what the meter costs and what level it holds.

Workload: a synthetic `streaming: true` medium voice; K in {1, 8, 32, 128} streams admitted at t = 0, each one
256-phoneme sentence (workload.synthetic_ids); chunk 55, padding 3.  Arms, alternated in every round: no meter;
-16 LUFS; -16 LUFS at 48 kHz; -16 LUFS with pitch 1.25.  Per arm and K, one JSON line with bench_streams' figures
(wall to drain, audio-s/s, first-chunk p50 / p99, underruns) and:
  loudness_ms_per_step   the "loudness" device ms of the metered passes, summed per step, averaged over the steps
  last3s_lu_p50 / max    per metered stream: |BS.1770 loudness of its last 3 s - T|, median and worst (LU)
  clipped                samples at full scale (|y| = 1) in the metered streams, over all streams
The device name and power limit are printed first, read in the same run.

  python tools/bench_live_loudness.py [--ks 1,8,32,128] [--reps 1]
"""
import argparse
import atexit
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_streams import CHUNK, PAD, PHONEMES, _summary    # noqa: E402

TARGET = -16.0
ARMS = {"none": {}, "lufs_-16": {"live_loudness": TARGET},
        "lufs_-16_48k": {"live_loudness": TARGET, "output_rate": 48000},
        "lufs_-16_pitch_1.25": {"live_loudness": TARGET, "pitch": 1.25}}


def run(model, batches, kw):
    import loudness_reference as lr
    from sonata_b200 import StreamBatch
    decode = model.infer_decoder_batch
    prof = {"ms": 0.0}

    def timed(chunks, **k):
        out = decode(chunks, **k)
        m = next((m for m in k.get("meters") or [] if m is not None), None)
        if m is not None:
            prof["ms"] += m.last_pass_ms
        return out
    model.infer_decoder_batch = timed
    steps = 0
    try:
        sb = StreamBatch(model, CHUNK, PAD)
        t0 = time.perf_counter()
        keys = [sb.add(ids, **kw) for ids in batches]
        arrivals = {k: [] for k in keys}
        chunks = {k: [] for k in keys}
        while len(sb):
            out = sb.step()
            steps += 1
            t = time.perf_counter() - t0
            for key, a in out:
                if isinstance(a, Exception):
                    raise a
                arrivals[key].append(t)
                chunks[key].append(a.as_slice())
        wall = time.perf_counter() - t0
    finally:
        del model.infer_decoder_batch
    sr = kw.get("output_rate") or model.audio_output_info().sample_rate
    extra = {"steps": steps}
    if "live_loudness" in kw:
        dev, clipped = [], 0
        for k in keys:
            y = np.concatenate(chunks[k])
            dev.append(abs(lr.integrated(y[-3 * sr:], sr) - kw["live_loudness"]))
            clipped += int(np.count_nonzero(np.abs(y) >= 1.0))
        extra.update(loudness_ms_per_step=round(prof["ms"] / max(steps, 1), 4),
                     last3s_lu_p50=round(float(np.median(dev)), 3), last3s_lu_max=round(float(np.max(dev)), 3),
                     clipped=clipped)
    return wall, [arrivals[k] for k in keys], [[len(c) for c in chunks[k]] for k in keys], sr, extra


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,8,32,128")
    ap.add_argument("--reps", type=int, default=1, help="rounds over the arms per K (each line is one run)")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_live_loudness: no CUDA device visible")
    from bench_voices import device_info
    from sonata_b200 import _native, voicegen, workload, from_config_path
    if not os.path.exists(_native.LIB_PATH):
        from sonata_b200 import build
        build.build()
    if not os.environ.get("SONATA_B200_VOICE_DIR"):        # generated voices never go into the tree
        os.environ["SONATA_B200_VOICE_DIR"] = tempfile.mkdtemp(prefix="sonata_voices_")
        atexit.register(shutil.rmtree, os.environ["SONATA_B200_VOICE_DIR"], True)
    print(json.dumps(device_info()), flush=True)
    path = voicegen.write_voice(voicegen.default_voice_dir(), "medium", streaming=True, name="medium_streaming")
    model = from_config_path(path, device=0)
    assert model.supports_streaming_output()
    ks = [int(k) for k in args.ks.split(",")]
    batches = [[int(i) for i in workload.synthetic_ids(PHONEMES, utt=u)] for u in range(max(ks))]
    for k in ks:
        for kw in ARMS.values():                  # warm-up: modules, arenas and pinned blocks at this K
            run(model, batches[:k], kw)
        torch.cuda.synchronize()
        for _ in range(args.reps):
            for name, kw in ARMS.items():
                wall, arrivals, lens, sr, extra = run(model, batches[:k], kw)
                print(json.dumps(_summary(name, k, wall, arrivals, lens, sr, extra)), flush=True)
    model.close()


if __name__ == "__main__":
    main()
