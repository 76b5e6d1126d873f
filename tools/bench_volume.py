"""Cost of the volume stage, for batches at the C2 shape and for realtime streams.

Batches: 32 utterances x 256 phonemes on the medium voice (22 050 Hz), its default noise scales, every utterance seeded.
Each step synthesises the batch as a job and fetches the f32 result to the host.  Four arms:

  (a) none              : no contour;
  (b) span_+6           : +6 dB on 10 % of each utterance's ids (one run a third of the way in);
  (c) mixed             : each id's level drawn from {-6, 0, +6} dB (seeded);
  (d) mixed_pitch_1.25  : (c) with pitch 1.25.

The arms alternate over --rounds rounds of --steps steps each.  One JSON line per arm: wall and device ms per step
(medians over rounds) and the "volume" region's ms and bytes (8 per delivered sample it scales, plus its piece tables)
with the bandwidth that implies against 3.35 TB/s (the H100 SXM's HBM3 data sheet figure).

Streams (--streams): StreamBatch runs of K = --ks streams at the same shape, with and without the mixed contour.  One
JSON line per arm and K: the first-chunk p50 / p99, underruns (tools/bench_streams.py's measures) and the "volume" device
ms summed over each step's passes and averaged over the steps.

The device name and power limit are printed first, read in the same run.

  python tools/bench_volume.py --steps 5 --warmup 2 --rounds 3 --streams
"""
import argparse
import atexit
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM_BYTES_PER_S = 3.35e12


def levels(batches, kind, seed=1234):
    rng = np.random.default_rng(seed)
    out = []
    for b in batches:
        n = len(b)
        if kind == "span":
            v = [None] * n
            a = n // 3
            v[a:a + max(1, n // 10)] = [6.0] * max(1, n // 10)
        else:
            v = [float(x) for x in rng.choice([-6.0, 0.0, 6.0], n)]
        out.append(v)
    return out


def run_batches(args, torch):
    import sonata_b200
    from sonata_b200 import voicegen, workload
    from sonata_b200.job import SynthesisJob
    model = sonata_b200.from_config_path(voicegen.write_voice(voicegen.default_voice_dir(), "medium"), device=0)
    n = args.utts
    batches = [workload.synthetic_ids(args.phonemes, utt=u) for u in range(n)]
    seeds = [1000 + b for b in range(n)]
    mixed = levels(batches, "mixed")
    arms = {"a_none": {}, "b_span_+6": dict(volume_contours=levels(batches, "span")),
            "c_mixed": dict(volume_contours=mixed), "d_mixed_pitch_1.25": dict(volume_contours=mixed, pitches=[1.25] * n)}

    def step(arm):
        job = SynthesisJob(model, batches, seeds=seeds, **arm)
        ms = job.run()
        job.fetch()
        reg = next((r for r in job.profile() if r["name"] == "volume"), None)
        job.close()
        return ms, reg

    for arm in arms.values():
        for _ in range(max(args.warmup, 1)):
            step(arm)
    torch.cuda.synchronize()
    res = {name: {"wall": [], "dev": [], "vol": [], "reg": None} for name in arms}
    for _ in range(args.rounds):
        for name, arm in arms.items():
            dev = vol = 0.0
            t0 = time.perf_counter()
            for _ in range(args.steps):
                ms, reg = step(arm)
                dev += ms
                if reg:
                    vol += reg["ms"]
                    res[name]["reg"] = reg
            torch.cuda.synchronize()
            r = res[name]
            r["wall"].append((time.perf_counter() - t0) * 1e3 / args.steps)
            r["dev"].append(dev / args.steps)
            r["vol"].append(vol / args.steps)
    for name, r in res.items():
        out = {"arm": name, "wall_ms": round(statistics.median(r["wall"]), 2),
               "device_ms": round(statistics.median(r["dev"]), 2),
               "device_ms_spread": round(max(r["dev"]) - min(r["dev"]), 2)}
        if r["reg"]:
            ms = statistics.median(r["vol"])
            out["volume"] = {"ms": round(ms, 4), "bytes": r["reg"]["bytes"],
                             "tb_per_s": round(r["reg"]["bytes"] / (ms * 1e-3) / 1e12, 3) if ms > 0 else None,
                             "share_of_3.35_tb_per_s": round(r["reg"]["bytes"] / (ms * 1e-3) / HBM_BYTES_PER_S, 3)
                             if ms > 0 else None}
        print(json.dumps(out), flush=True)
    model.close()


def run_streams(args, torch):
    from bench_streams import _summary
    from sonata_b200 import StreamBatch, from_config_path, voicegen, workload
    path = voicegen.write_voice(voicegen.default_voice_dir(), "medium", streaming=True, name="medium_streaming")
    model = from_config_path(path, device=0)
    sr = model.audio_output_info().sample_rate
    ks = [int(k) for k in args.ks.split(",")]
    batches = [[int(i) for i in workload.synthetic_ids(args.phonemes, utt=u)] for u in range(max(ks))]
    mixed = levels(batches, "mixed")
    decode = model.infer_decoder_batch

    def run(k, contour):
        prof = {"volume": 0.0, "steps": 0}

        def timed(chunks, **kw):
            out = decode(chunks, **kw)
            w = next((w for w in kw.get("warps") or [] if w is not None), None)
            if w is not None:
                prof["volume"] += w.last_volume_ms()
            return out
        model.infer_decoder_batch = timed
        try:
            sb = StreamBatch(model, 55, 3)
            t0 = time.perf_counter()
            keys = [sb.add(batches[s], volume_contour=mixed[s] if contour else None) for s in range(k)]
            arrivals, lens = {q: [] for q in keys}, {q: [] for q in keys}
            while len(sb):
                out = sb.step()
                prof["steps"] += 1
                t = time.perf_counter() - t0
                for key, a in out:
                    if isinstance(a, Exception):
                        raise a
                    arrivals[key].append(t)
                    lens[key].append(len(a))
            wall = time.perf_counter() - t0
        finally:
            del model.infer_decoder_batch
        extra = {"volume_ms_per_step": round(prof["volume"] / max(prof["steps"], 1), 4)} if contour else {}
        return _summary("volume_mixed" if contour else "none", k, wall, [arrivals[q] for q in keys],
                        [lens[q] for q in keys], sr, extra)

    for k in ks:
        for contour in (False, True):
            run(k, contour)                         # warm-up at this K
        torch.cuda.synchronize()
        for _ in range(args.reps):
            for contour in (False, True):
                print(json.dumps(run(k, contour)), flush=True)
    model.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--utts", type=int, default=32)
    ap.add_argument("--phonemes", type=int, default=256)
    ap.add_argument("--streams", action="store_true", help="also run the StreamBatch arms")
    ap.add_argument("--ks", default="1,8,32,128")
    ap.add_argument("--reps", type=int, default=1)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_volume: no CUDA device visible")
    from bench_voices import device_info
    from sonata_b200 import _native
    if not os.path.exists(_native.LIB_PATH):
        from sonata_b200 import build
        build.build()
    if not os.environ.get("SONATA_B200_VOICE_DIR"):        # generated voices never go into the tree
        os.environ["SONATA_B200_VOICE_DIR"] = tempfile.mkdtemp(prefix="sonata_voices_")
        atexit.register(shutil.rmtree, os.environ["SONATA_B200_VOICE_DIR"], True)
    print(json.dumps(device_info()), flush=True)
    run_batches(args, torch)
    if args.streams:
        run_streams(args, torch)


if __name__ == "__main__":
    main()
