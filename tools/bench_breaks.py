"""Cost of the break stage (pauses), for batches at the C2 shape and for realtime streams.

Batches: 32 utterances x 256 phonemes on the medium voice (22 050 Hz), its default noise scales, every utterance seeded.
Each step synthesises the batch as a job and fetches the f32 result to the host.  Four arms:

  (a) none                  : no breaks;
  (b) every10_250ms         : 250 ms after every 10th character (on its pad id);
  (c) every10_pitch_1.25    : (b) with pitch 1.25;
  (d) every10_48k_-16lufs   : (b) delivered at 48 kHz with a -16 LUFS loudness target.

The arms alternate over --rounds rounds of --steps steps each.  One JSON line per arm: wall and device ms per step
(medians over rounds), audio seconds per wall second at the delivered length, and the "break" region's ms and bytes (4
per input sample and 4 per output sample, plus its tables) with the bandwidth that implies against 3.35 TB/s (the H100
SXM's HBM3 data sheet figure).

Streams (--streams): StreamBatch runs of K = --ks streams at the same shape (chunk 55, padding 3), with and without the
breaks of (b).  One JSON line per arm and K: the first-chunk p50 / p99, underruns (tools/bench_streams.py's measures) and
the "break" device ms summed over each step's passes and averaged over the steps.

The device name, power limit and max SM clock are printed first, read in the same run.

  python tools/bench_breaks.py --steps 5 --warmup 2 --rounds 3 --streams
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

HBM_BYTES_PER_S = 3.35e12


def every10(batches, ms=250.0):
    """ms after every 10th character: ids are bos, then (id, pad) per character, then eos, so character c's pad is id
    2 + 2 c and every 10th character's (c = 9, 19, ..) is an id i > 0 with i % 20 == 0."""
    return [[ms if i > 0 and i % 20 == 0 and i < len(b) - 1 else None for i in range(len(b))] for b in batches]


def run_batches(args, torch):
    import sonata_b200
    from sonata_b200 import voicegen, workload
    from sonata_b200.job import SynthesisJob
    model = sonata_b200.from_config_path(voicegen.write_voice(voicegen.default_voice_dir(), "medium"), device=0)
    n = args.utts
    batches = [workload.synthetic_ids(args.phonemes, utt=u) for u in range(n)]
    seeds = [1000 + b for b in range(n)]
    bk = every10(batches)
    arms = {"a_none": {}, "b_every10_250ms": dict(breaks=bk), "c_every10_pitch_1.25": dict(breaks=bk, pitches=[1.25] * n),
            "d_every10_48k_-16lufs": dict(breaks=bk, output_rates=[48000] * n, loudness=[-16.0] * n)}
    seconds = {}

    def step(arm):
        job = SynthesisJob(model, batches, seeds=seeds, **arm)
        ms = job.run()
        audio = job.fetch()
        reg = next((r for r in job.profile() if r["name"] == "break"), None)
        job.close()
        return ms, reg, sum(len(a.samples.as_slice()) / a.info.sample_rate for a in audio)

    for name, arm in arms.items():
        for _ in range(max(args.warmup, 1)):
            seconds[name] = step(arm)[2]
    torch.cuda.synchronize()
    res = {name: {"wall": [], "dev": [], "brk": [], "reg": None} for name in arms}
    for _ in range(args.rounds):
        for name, arm in arms.items():
            dev = brk = 0.0
            t0 = time.perf_counter()
            for _ in range(args.steps):
                ms, reg, _ = step(arm)
                dev += ms
                if reg:
                    brk += reg["ms"]
                    res[name]["reg"] = reg
            torch.cuda.synchronize()
            r = res[name]
            r["wall"].append((time.perf_counter() - t0) * 1e3 / args.steps)
            r["dev"].append(dev / args.steps)
            r["brk"].append(brk / args.steps)
    for name, r in res.items():
        out = {"arm": name, "wall_ms": round(statistics.median(r["wall"]), 2),
               "device_ms": round(statistics.median(r["dev"]), 2),
               "device_ms_spread": round(max(r["dev"]) - min(r["dev"]), 2),
               "audio_s": round(seconds[name], 2),
               "audio_s_per_s": round(seconds[name] / (statistics.median(r["wall"]) * 1e-3), 1)}
        if r["reg"]:
            ms = statistics.median(r["brk"])
            out["break"] = {"ms": round(ms, 4), "bytes": r["reg"]["bytes"],
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
    bk = every10(batches)
    decode = model.infer_decoder_batch

    def run(k, contour):
        prof = {"break": 0.0, "steps": 0}

        def timed(chunks, **kw):
            out = decode(chunks, **kw)
            w = next((w for w in kw.get("warps") or [] if w is not None), None)
            if w is not None:
                prof["break"] += w.last_break_ms()
            return out
        model.infer_decoder_batch = timed
        try:
            sb = StreamBatch(model, 55, 3)
            t0 = time.perf_counter()
            keys = [sb.add(batches[s], breaks=bk[s] if contour else None) for s in range(k)]
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
        extra = {"break_ms_per_step": round(prof["break"] / max(prof["steps"], 1), 4)} if contour else {}
        return _summary("every10_250ms" if contour else "none", k, wall, [arrivals[q] for q in keys],
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
        sys.exit("bench_breaks: no CUDA device visible")
    from bench_voices import device_info
    from sonata_b200 import _native
    if not os.path.exists(_native.LIB_PATH):
        from sonata_b200 import build
        build.build()
    if not os.environ.get("SONATA_B200_VOICE_DIR"):        # generated voices never go into the tree
        os.environ["SONATA_B200_VOICE_DIR"] = tempfile.mkdtemp(prefix="sonata_voices_")
        atexit.register(shutil.rmtree, os.environ["SONATA_B200_VOICE_DIR"], True)
    info = device_info()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["max_sm_clock_mhz"] = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        info["max_sm_clock_mhz"] = None
    print(json.dumps(info), flush=True)
    run_batches(args, torch)
    if args.streams:
        run_streams(args, torch)


if __name__ == "__main__":
    main()
