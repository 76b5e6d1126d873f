"""Cost of target durations at the C2 shape, against the host two-pass workaround.

Batches: 32 utterances x 256 phonemes on the medium voice (22 050 Hz), its default noise scales, every utterance seeded.
Each step synthesises the batch as a job and fetches the f32 result to the host.  Arms:

  (a) none          : no targets;
  (b) whole_0.8x    : every utterance fitted to 0.8x its natural length (arm (a)'s);
  (c) whole_1.25x   : the same at 1.25x;
  (d) words         : spans of 8 ids (about 4 characters: each is an id and a pad) at 0.9x their natural length;
  (e) two_pass_0.8x : the host workaround for (b): synthesise, read the frames per id, scale every id's duration by
                      target / natural, synthesise again.  Its wall time covers both passes.

The arms alternate over --rounds rounds of --steps steps each.  One JSON line per arm: wall and device ms per step
(medians over rounds) and, for the fitted arms, the "fit" profile region's ms; (b), (c) and (e) also give how far the
delivered lengths land from their targets (mean and worst, in samples; a fitted utterance never passes its slot, and
sits below it by less than one step of its durations).

The device name, power limit and max SM clock are printed first, read in the same run.

  python tools/bench_fit.py --steps 5 --warmup 2 --rounds 3
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


def run(args, torch):
    import sonata_b200
    from sonata_b200 import voicegen, workload
    from sonata_b200.job import SynthesisJob
    model = sonata_b200.from_config_path(voicegen.write_voice(voicegen.default_voice_dir(), "medium"), device=0)
    rate = model.audio_output_info().sample_rate
    n = args.utts
    batches = [workload.synthetic_ids(args.phonemes, utt=u) for u in range(n)]
    seeds = [1000 + b for b in range(n)]
    job = SynthesisJob(model, batches, seeds=seeds)
    job.run()
    natural = [np.asarray(f, np.int64) for f in job.id_frames()]
    job.close()
    ms_of = lambda frames: 1000.0 * 256 * float(frames) / rate
    whole = lambda r: [r * ms_of(f.sum()) for f in natural]
    words = [[(a, min(a + 7, len(f) - 1), 0.9 * ms_of(f[a:a + 8].sum())) for a in range(0, len(f), 8)
              if f[a:a + 8].sum() > 0] for f in natural]
    arms = {"a_none": None, "b_whole_0.8x": whole(0.8), "c_whole_1.25x": whole(1.25), "d_words": words,
            "e_two_pass_0.8x": "two_pass"}
    target_ms = {"b_whole_0.8x": whole(0.8), "c_whole_1.25x": whole(1.25), "e_two_pass_0.8x": whole(0.8)}

    def step(name, arm):
        if arm == "two_pass":
            j = SynthesisJob(model, batches, seeds=seeds)
            dev = j.run()
            frames = j.id_frames()
            j.close()
            t = target_ms[name]
            scales = [np.full(len(f), t[b] / max(ms_of(f.sum()), 1e-9), np.float32) for b, f in enumerate(frames)]
            j = SynthesisJob(model, batches, seeds=seeds)
            j.set_durations(scales=scales)
            dev += j.run()
            audio = j.fetch()
            j.close()
            return dev, None, audio
        j = SynthesisJob(model, batches, seeds=seeds, target_durations=arm)
        dev = j.run()
        audio = j.fetch()
        reg = next((r for r in j.profile() if r["name"] == "fit"), None)
        j.close()
        return dev, reg, audio

    miss = {}
    for name, arm in arms.items():
        for _ in range(max(args.warmup, 1)):
            _, _, audio = step(name, arm)
        if name in target_ms:
            d = [len(a.samples.as_slice()) - int(np.floor(t * rate / 1000.0 + 0.5))
                 for a, t in zip(audio, target_ms[name])]
            miss[name] = {"mean_samples": round(float(np.mean(d)), 1), "worst_over": int(max(d)),
                          "worst_under": int(min(d))}
    torch.cuda.synchronize()
    res = {name: {"wall": [], "dev": [], "fit": []} for name in arms}
    for _ in range(args.rounds):
        for name, arm in arms.items():
            dev = fit = 0.0
            t0 = time.perf_counter()
            for _ in range(args.steps):
                ms, reg, _ = step(name, arm)
                dev += ms
                if reg:
                    fit += reg["ms"]
            torch.cuda.synchronize()
            r = res[name]
            r["wall"].append((time.perf_counter() - t0) * 1e3 / args.steps)
            r["dev"].append(dev / args.steps)
            r["fit"].append(fit / args.steps)
    for name, r in res.items():
        out = {"arm": name, "wall_ms": round(statistics.median(r["wall"]), 2),
               "wall_ms_spread": round(max(r["wall"]) - min(r["wall"]), 2),
               "device_ms": round(statistics.median(r["dev"]), 2)}
        if arms[name] not in (None, "two_pass"):
            out["fit_ms"] = round(statistics.median(r["fit"]), 4)
        if name in miss:
            out["vs_target"] = miss[name]
        print(json.dumps(out), flush=True)
    model.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--utts", type=int, default=32)
    ap.add_argument("--phonemes", type=int, default=256)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_fit: no CUDA device visible")
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
    run(args, torch)


if __name__ == "__main__":
    main()
