"""Cost and strength of the watermark, for batches at the C2 shape.

Batches: 32 utterances x 256 phonemes on the medium voice (22 050 Hz), its default noise scales, every utterance seeded.
Each step synthesises the batch as a job and fetches the result to the host.  Four arms, alternated over --rounds
rounds of --steps steps each:

  (a) unmarked;
  (b) marked             : key, payload 1234, -26 dB;
  (c) marked_48k_-16LUFS : (b) delivered at 48 kHz with a -16 LUFS target;
  (d) marked_mulaw_8k    : (b) delivered at 8 kHz and fetched as G.711 mu-law.

One JSON line per arm: wall and device ms per step (medians over rounds) and the "watermark" region's ms and bytes (8
per delivered sample) with the bandwidth that implies against 3.35 TB/s (the H100 SXM's HBM3 data sheet figure).

Detection: clips per second of core.watermark_detect (host to device copy included) for the 32 C2 utterances and for
1 024 clips of 5 s, against tests/watermark_reference.py's numpy detector on one host thread (over a sample of clips).

Strength: for each route (f32 and i16 at 22.05 kHz, mu-law and A-law at 8 kHz, -16 LUFS at 48 kHz) and strength (-20,
-26, -32 dB), the shortest crop from the middle of each utterance, on a grid of lengths, that the detector finds with its
payload in at least 95 % of the 32 utterances.

Streams (--streams): StreamBatch runs of K = --ks streams of the same shape (chunk 55, padding 3), unmarked and
marked.  One JSON line per arm and K: the first-chunk p50 / p99 and underruns (tools/bench_streams.py's measures) and
the "watermark" device ms summed over each step's passes and averaged over the steps.

The device name, power limit and maximum SM clock are printed first, read in the same run.

  python tools/bench_watermark.py --steps 5 --warmup 2 --rounds 3 --streams
"""
import argparse
import atexit
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BYTES_PER_S = 3.35e12
KEY, PAYLOAD = 0x5EC12E70DDBA11, 1234
CROPS_S = (0.25, 0.5, 0.75, 1.0, 1.5, 2.0, 3.0, 4.0, 5.0, 7.5, 10.0)


def device_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = (s.strip() for s in q[0].split(",")) if q else ("?", "?", "?")
    return {"device": name, "power_limit": power, "max_sm_clock": clock}


def _g711_decode(b, law):
    u = np.frombuffer(bytes(b), np.uint8).astype(np.int32)
    if law == "mulaw":
        u = ~u & 0xFF
        t = (((u & 0x0F) << 3) + 0x84) << ((u & 0x70) >> 4)
        return np.where(u & 0x80, 0x84 - t, t - 0x84).astype(np.int16)
    a = u ^ 0x55
    seg = (a & 0x70) >> 4
    t = (a & 0x0F) << 4
    t = np.where(seg == 0, t + 8, (t + 0x108) << np.maximum(seg - 1, 0))
    return np.where(a & 0x80, t, -t).astype(np.int16)


def run_batches(args, torch, model, batches, seeds):
    from sonata_b200.job import SynthesisJob
    n = len(batches)
    arms = {"a_unmarked": (None, {}, None), "b_marked": (-26.0, {}, None),
            "c_marked_48k_-16LUFS": (-26.0, dict(output_rates=[48000] * n, loudness=[-16.0] * n), None),
            "d_marked_mulaw_8k": (-26.0, dict(output_rates=[8000] * n), "mulaw")}

    def step(arm):
        db, kw, law = arm
        model.set_watermark(None if db is None else KEY, PAYLOAD, -26.0 if db is None else db)
        job = SynthesisJob(model, batches, seeds=seeds, **kw)
        ms = job.run()
        job.fetch_g711(law) if law else job.fetch()
        reg = next((r for r in job.profile() if r["name"] == "watermark"), None)
        job.close()
        return ms, reg

    for arm in arms.values():
        for _ in range(max(args.warmup, 1)):
            step(arm)
    torch.cuda.synchronize()
    res = {name: {"wall": [], "dev": [], "wm": [], "reg": None} for name in arms}
    for _ in range(args.rounds):
        for name, arm in arms.items():
            dev = wm = 0.0
            t0 = time.perf_counter()
            for _ in range(args.steps):
                ms, reg = step(arm)
                dev += ms
                if reg:
                    wm += reg["ms"]
                    res[name]["reg"] = reg
            torch.cuda.synchronize()
            r = res[name]
            r["wall"].append((time.perf_counter() - t0) * 1e3 / args.steps)
            r["dev"].append(dev / args.steps)
            r["wm"].append(wm / args.steps)
    model.set_watermark(None)
    for name, r in res.items():
        out = {"arm": name, "wall_ms": round(statistics.median(r["wall"]), 2),
               "device_ms": round(statistics.median(r["dev"]), 2),
               "device_ms_spread": round(max(r["dev"]) - min(r["dev"]), 2)}
        if r["reg"]:
            ms = statistics.median(r["wm"])
            out["watermark"] = {"ms": round(ms, 4), "bytes": r["reg"]["bytes"],
                                "tb_per_s": round(r["reg"]["bytes"] / (ms * 1e-3) / 1e12, 3) if ms > 0 else None,
                                "share_of_3.35_tb_per_s": round(r["reg"]["bytes"] / (ms * 1e-3) / HBM_BYTES_PER_S, 3)
                                if ms > 0 else None}
        print(json.dumps(out), flush=True)


def routes(model, batches, seeds, db):
    """{route: (clips, rate)} of the marked C2 batch at strength db."""
    from sonata_b200.job import SynthesisJob
    n = len(batches)
    model.set_watermark(KEY, PAYLOAD, db)
    try:
        j = SynthesisJob(model, batches, seeds=seeds)
        j.run()
        out = {"f32": ([a.samples.as_slice().copy() for a in j.fetch()], 22050), "i16": (j.fetch_i16(), 22050)}
        j8 = SynthesisJob(model, batches, seeds=seeds, output_rates=[8000] * n)
        j8.run()
        out["mulaw_8k"] = ([_g711_decode(x, "mulaw") for x in j8.fetch_g711("mulaw")], 8000)
        out["alaw_8k"] = ([_g711_decode(x, "alaw") for x in j8.fetch_g711("alaw")], 8000)
        j48 = SynthesisJob(model, batches, seeds=seeds, output_rates=[48000] * n, loudness=[-16.0] * n)
        j48.run()
        out["-16LUFS_48k"] = ([a.samples.as_slice().copy() for a in j48.fetch()], 48000)
    finally:
        model.set_watermark(None)
    return out


def run_detection(model, batches, seeds):
    import watermark_reference as wr
    from sonata_b200.core import watermark_detect
    clips = routes(model, batches, seeds, -26.0)["f32"][0]
    rng = np.random.default_rng(5)
    five = []
    while len(five) < 1024:
        x = clips[len(five) % len(clips)]
        lo = int(rng.integers(0, max(1, x.size - 5 * 22050)))
        five.append(x[lo:lo + 5 * 22050])
    c = wr.chips(KEY)
    for name, cl in (("c2_utterances", clips), ("5s_clips_x1024", five)):
        watermark_detect(cl, KEY)
        t0 = time.perf_counter()
        reps = 5
        for _ in range(reps):
            got = watermark_detect(cl, KEY)
        dev = reps * len(cl) / (time.perf_counter() - t0)
        sample = cl[:16]
        t0 = time.perf_counter()
        for x in sample:
            wr.detect(x, KEY, c)
        host = len(sample) / (time.perf_counter() - t0)
        print(json.dumps({"detector": name, "clips": len(cl), "device_clips_per_s": round(dev, 1),
                          "numpy_one_thread_clips_per_s": round(host, 1),
                          "detected": sum(g.marked and g.payload == PAYLOAD for g in got)}), flush=True)


def run_strength(model, batches, seeds):
    from sonata_b200.core import watermark_detect
    for db in (-20.0, -26.0, -32.0):
        for route, (clips, rate) in routes(model, batches, seeds, db).items():
            shortest, z_full = None, [round(g.z0, 1) for g in watermark_detect(clips, KEY)]
            for s in CROPS_S:
                n = int(s * rate)
                crops = [x[max(0, x.size // 2 - n // 2):max(0, x.size // 2 - n // 2) + n] for x in clips]
                got = watermark_detect(crops, KEY)
                if sum(g.marked and g.payload == PAYLOAD for g in got) >= 0.95 * len(clips):
                    shortest = s
                    break
            print(json.dumps({"strength_db": db, "route": route, "shortest_crop_s_95pct": shortest,
                              "whole_utterance_z0_median": float(np.median(z_full)),
                              "whole_utterance_z0_min": float(np.min(z_full))}), flush=True)


def run_streams(args, torch):
    from bench_streams import _summary
    from sonata_b200 import StreamBatch, from_config_path, voicegen, workload
    path = voicegen.write_voice(voicegen.default_voice_dir(), "medium", streaming=True, name="medium_streaming")
    model = from_config_path(path, device=0)
    sr = model.audio_output_info().sample_rate
    ks = [int(k) for k in args.ks.split(",")]
    batches = [[int(i) for i in workload.synthetic_ids(args.phonemes, utt=u)] for u in range(max(ks))]
    decode = model.infer_decoder_batch

    def run(k, marked):
        prof = {"watermark": 0.0, "steps": 0}

        def timed(chunks, **kw):
            out = decode(chunks, **kw)
            w = next((w for w in kw.get("marks") or [] if w is not None), None)
            if w is not None:
                prof["watermark"] += w.last_pass_ms
            return out
        model.infer_decoder_batch = timed
        model.set_watermark(KEY if marked else None, PAYLOAD, -26.0)
        try:
            sb = StreamBatch(model, 55, 3)
            t0 = time.perf_counter()
            keys = [sb.add(batches[s]) for s in range(k)]
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
            model.set_watermark(None)
        extra = {"watermark_ms_per_step": round(prof["watermark"] / max(prof["steps"], 1), 4)} if marked else {}
        return _summary("marked" if marked else "unmarked", k, wall, [arrivals[q] for q in keys],
                        [lens[q] for q in keys], sr, extra)

    for k in ks:
        for marked in (False, True):
            run(k, marked)                          # warm-up at this K
        torch.cuda.synchronize()
        for marked in (False, True):
            print(json.dumps(run(k, marked)), flush=True)
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
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_watermark: no CUDA device visible")
    import sonata_b200
    from sonata_b200 import _native, voicegen, workload
    if not os.path.exists(_native.LIB_PATH):
        from sonata_b200 import build
        build.build()
    if not os.environ.get("SONATA_B200_VOICE_DIR"):        # generated voices never go into the tree
        os.environ["SONATA_B200_VOICE_DIR"] = tempfile.mkdtemp(prefix="sonata_voices_")
        atexit.register(shutil.rmtree, os.environ["SONATA_B200_VOICE_DIR"], True)
    print(json.dumps(device_info()), flush=True)
    model = sonata_b200.from_config_path(voicegen.write_voice(voicegen.default_voice_dir(), "medium"), device=0)
    batches = [workload.synthetic_ids(args.phonemes, utt=u) for u in range(args.utts)]
    seeds = [1000 + b for b in range(args.utts)]
    run_batches(args, torch, model, batches, seeds)
    run_detection(model, batches, seeds)
    run_strength(model, batches, seeds)
    model.close()
    if args.streams:
        run_streams(args, torch)


if __name__ == "__main__":
    main()
