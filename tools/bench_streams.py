"""Serving K realtime streams at once: StreamBatch (one encoder pass for new streams, one decoder pass per chunk step)
against K host threads that each iterate their own `stream_synthesis`, as a server does with one B = 1 stream per
request.

Workload: a synthetic `streaming: true` medium voice; K requests admitted at t = 0, each one 256-phoneme sentence
(workload.synthetic_ids); chunk 55, padding 3 (the gRPC realtime path's values); the voice's default noise.  Per arm and
K, one JSON line:
  wall_s            time until every stream has delivered its last chunk
  audio_s_per_s     audio seconds delivered (at the voice's rate) over wall_s
  first_chunk_ms    p50 / p99 over the streams of the time from admission to the first chunk
  underruns         chunks i+1 that arrived after the audio of chunks 0..i, played from the first chunk's arrival, ran
                    out (and how many streams had at least one)
  pad_frac          StreamBatch only: padding rows of the decoder passes' frame levels over all their rows (each chunk
                    occupies whole 128-frame granules)
The device name and power limit are printed first, read in the same run.  With --ratios the arms are StreamBatch runs
with every stream at one pair of pitch / tempo ratios (none, pitch 1.25, tempo 1.5, pitch 0.8 with tempo 2), whose lines
add the "stretch" and "pitch" device ms per step; audio_s_per_s is then at the delivered length.

  python tools/bench_streams.py [--ks 1,8,32,128] [--reps 1] [--ratios]
"""
import argparse
import atexit
import json
import os
import shutil
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

CHUNK, PAD, PHONEMES = 55, 3, 256
GY, HY = 128, 8                  # frame granule and least gap of the engine's frame level (engine.cu)


def _summary(arm, k, wall, arrivals, lens, sr, extra=None):
    """arrivals[s]: host times of stream s's chunks (from admission); lens[s]: their sample counts."""
    first = np.array([a[0] for a in arrivals]) * 1e3
    under, streams_under = 0, 0
    for a, n in zip(arrivals, lens):
        play_end = a[0] + np.cumsum(n) / sr                 # the audio of chunks 0..i has played out at play_end[i]
        u = int(np.sum(np.asarray(a[1:]) > play_end[:-1]))
        under += u
        streams_under += u > 0
    line = {"arm": arm, "K": k, "wall_s": round(wall, 4),
            "audio_s_per_s": round(sum(sum(n) for n in lens) / sr / wall, 1),
            "first_chunk_ms_p50": round(float(np.percentile(first, 50)), 2),
            "first_chunk_ms_p99": round(float(np.percentile(first, 99)), 2),
            "chunks": sum(len(n) for n in lens), "underruns": under, "streams_with_underrun": streams_under}
    line.update(extra or {})
    return line


def run_batch(model, batches, sr):
    from sonata_b200 import StreamBatch
    rows = {"valid": 0, "all": 0}
    decode = model.infer_decoder_batch

    def counted(chunks, **kw):
        for _, lo, hi in chunks:
            rows["valid"] += hi - lo
            rows["all"] += (hi - lo + HY + GY - 1) // GY * GY
        return decode(chunks, **kw)
    model.infer_decoder_batch = counted
    try:
        sb = StreamBatch(model, CHUNK, PAD)
        t0 = time.perf_counter()
        keys = [sb.add(ids) for ids in batches]
        arrivals = {k: [] for k in keys}
        lens = {k: [] for k in keys}
        while len(sb):
            out = sb.step()
            t = time.perf_counter() - t0
            for key, a in out:
                if isinstance(a, Exception):
                    raise a
                arrivals[key].append(t)
                lens[key].append(len(a))
        wall = time.perf_counter() - t0
    finally:
        del model.infer_decoder_batch
    pad = 1.0 - rows["valid"] / rows["all"]
    return wall, [arrivals[k] for k in keys], [lens[k] for k in keys], {"pad_frac": round(pad, 4)}


RATIO_ARMS = {"none": {}, "pitch_1.25": {"pitch": 1.25}, "tempo_1.5": {"tempo": 1.5},
              "pitch_0.8_tempo_2": {"pitch": 0.8, "tempo": 2.0}}


def run_ratios(model, batches, sr, ratios):
    """StreamBatch with every stream at `ratios`: the batch arm's figures plus the "stretch" and "pitch" device ms per
    step (each warped pass's regions, summed over the passes of a step, averaged over the steps)."""
    from sonata_b200 import StreamBatch
    decode = model.infer_decoder_batch
    prof = {"stretch": 0.0, "pitch": 0.0}

    def timed(chunks, **kw):
        out = decode(chunks, **kw)
        w = next((w for w in kw.get("warps") or [] if w is not None), None)
        if w is not None:
            s, p = w.last_pass_ms()
            prof["stretch"] += s
            prof["pitch"] += p
        return out
    model.infer_decoder_batch = timed
    steps = 0
    try:
        sb = StreamBatch(model, CHUNK, PAD)
        t0 = time.perf_counter()
        keys = [sb.add(ids, **ratios) for ids in batches]
        arrivals = {k: [] for k in keys}
        lens = {k: [] for k in keys}
        while len(sb):
            out = sb.step()
            steps += 1
            t = time.perf_counter() - t0
            for key, a in out:
                if isinstance(a, Exception):
                    raise a
                arrivals[key].append(t)
                lens[key].append(len(a))
        wall = time.perf_counter() - t0
    finally:
        del model.infer_decoder_batch
    return wall, [arrivals[k] for k in keys], [lens[k] for k in keys], {
        "stretch_ms_per_step": round(prof["stretch"] / max(steps, 1), 3),
        "pitch_ms_per_step": round(prof["pitch"] / max(steps, 1), 3), "steps": steps}


def run_threads(model, batches, sr):
    from sonata_b200 import SpeechStreamer
    k = len(batches)
    arrivals, lens = [[] for _ in range(k)], [[] for _ in range(k)]
    errors = []
    start = threading.Barrier(k + 1)
    t0 = [0.0]

    def client(s):
        start.wait()
        try:
            for a in SpeechStreamer(model.infer_encoder(batches[s]), CHUNK, PAD):   # stream_synthesis on ids
                arrivals[s].append(time.perf_counter() - t0[0])
                lens[s].append(len(a))
        except Exception as e:             # noqa: BLE001
            errors.append(e)
    th = [threading.Thread(target=client, args=(s,)) for s in range(k)]
    for t in th:
        t.start()
    t0[0] = time.perf_counter()
    start.wait()
    for t in th:
        t.join()
    wall = time.perf_counter() - t0[0]
    if errors:
        raise errors[0]
    return wall, arrivals, lens, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,8,32,128")
    ap.add_argument("--reps", type=int, default=1, help="timed runs per arm and K (each line is one run)")
    ap.add_argument("--ratios", action="store_true",
                    help="StreamBatch arms with pitch / tempo ratios instead (no ratios, pitch 1.25, tempo 1.5, pitch "
                         "0.8 with tempo 2), alternated in each rep; audio_s_per_s is at the delivered length")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_streams: no CUDA device visible")
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
    sr = model.audio_output_info().sample_rate
    ks = [int(k) for k in args.ks.split(",")]
    batches = [[int(i) for i in workload.synthetic_ids(PHONEMES, utt=u)] for u in range(max(ks))]
    arms = {"stream_batch": run_batch, "threads": run_threads}
    if args.ratios:
        arms = {name: (lambda m, b, s, r=r: run_ratios(m, b, s, r)) for name, r in RATIO_ARMS.items()}
    for k in ks:
        for name, fn in arms.items():            # warm-up: modules, arenas and pinned blocks at this K
            fn(model, batches[:k], sr)
        torch.cuda.synchronize()
        for _ in range(args.reps):
            for name, fn in arms.items():
                wall, arrivals, lens, extra = fn(model, batches[:k], sr)
                print(json.dumps(_summary(name, k, wall, arrivals, lens, sr, extra)), flush=True)
    model.close()


if __name__ == "__main__":
    main()
