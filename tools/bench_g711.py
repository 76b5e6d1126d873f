"""Cost of delivering G.711 telephony audio at the C2 shape.

32 utterances x 256 phonemes on the medium voice, its default noise scales, every utterance seeded, at the voice's
rate (22 050 Hz) and at 8 kHz.  Each step synthesises the batch and fetches the result to the host in one of four
ways:

  f32        : job.fetch() (4 bytes per sample);
  i16        : job.fetch_i16() (2 bytes per sample, converted on the device);
  mulaw_dev  : job.fetch_g711("mulaw") (1 byte per sample, encoded on the device in the i16 conversion's launches);
  mulaw_host : job.fetch_i16(), then encoded on the host with a 65 536-entry numpy table.

The arms alternate over --rounds rounds of --steps steps each.  Prints the device name and power limit, then one JSON
line per arm: wall ms per step and of the fetch alone (medians over rounds, and the spread), the run's device ms per
step, the device->host bytes and the kernel launches of the fetch.

  python tools/bench_g711.py --steps 10 --warmup 3 --rounds 5
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--utts", type=int, default=32)
    ap.add_argument("--phonemes", type=int, default=256)
    args = ap.parse_args()

    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_g711: no CUDA device visible")
    import sonata_b200
    from bench_voices import device_info
    from sonata_b200 import _native, voicegen, workload
    from sonata_b200.core import g711_encode
    from sonata_b200.job import SynthesisJob
    if not os.path.exists(_native.LIB_PATH):
        from sonata_b200 import build
        build.build()
    if not os.environ.get("SONATA_B200_VOICE_DIR"):        # generated voices never go into the tree
        os.environ["SONATA_B200_VOICE_DIR"] = tempfile.mkdtemp(prefix="sonata_voices_")
        atexit.register(shutil.rmtree, os.environ["SONATA_B200_VOICE_DIR"], True)

    lib = _native.lib()
    model = sonata_b200.from_config_path(voicegen.write_voice(voicegen.default_voice_dir(), "medium"), device=0)
    batches = [workload.synthetic_ids(args.phonemes, utt=u) for u in range(args.utts)]
    seeds = [1000 + b for b in range(args.utts)]
    n = args.utts
    table = g711_encode(np.arange(-32768, 32768, dtype=np.int16), "mulaw")

    def host_mulaw(job):
        return [table[x.astype(np.int32) + 32768].tobytes() for x in job.fetch_i16()]

    fetches = {"f32": (lambda job: job.fetch(), 4), "i16": (lambda job: job.fetch_i16(), 2),
               "mulaw_dev": (lambda job: job.fetch_g711("mulaw"), 1), "mulaw_host": (host_mulaw, 2)}
    arms = {f"{name}@{rate or 'voice'}": (rate, fn, bps) for rate in (None, 8000)
            for name, (fn, bps) in fetches.items()}

    def step(arm):
        rate, fetch, bps = arm
        job = SynthesisJob(model, batches, seeds=seeds, output_rates=None if rate is None else [rate] * n)
        ms = job.run()
        samples = sum(job.lengths()[1])
        l0 = lib.sb200_launch_count()
        t0 = time.perf_counter()
        fetch(job)
        fetch_ms = (time.perf_counter() - t0) * 1e3
        launches = lib.sb200_launch_count() - l0
        job.close()
        return ms, fetch_ms, samples * bps, launches

    print(json.dumps(device_info()), flush=True)
    for arm in arms.values():
        for _ in range(max(args.warmup, 1)):
            step(arm)
    torch.cuda.synchronize()
    res = {name: {"wall": [], "dev": [], "fetch": [], "d2h": 0, "launches": 0} for name in arms}
    for _ in range(args.rounds):
        for name, arm in arms.items():
            dev_ms = fetch_ms = 0.0
            t0 = time.perf_counter()
            for _ in range(args.steps):
                ms, f_ms, d2h, launches = step(arm)
                dev_ms += ms
                fetch_ms += f_ms
                res[name]["d2h"], res[name]["launches"] = d2h, launches
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            r = res[name]
            r["wall"].append(wall * 1e3 / args.steps)
            r["dev"].append(dev_ms / args.steps)
            r["fetch"].append(fetch_ms / args.steps)
    for name, r in res.items():
        med = lambda k: statistics.median(r[k])
        print(json.dumps({
            "arm": name, "shape": f"{args.utts}x{args.phonemes}", "steps": args.steps, "rounds": args.rounds,
            "wall_ms_per_step": round(med("wall"), 3), "wall_ms_range": [round(min(r["wall"]), 3), round(max(r["wall"]), 3)],
            "fetch_ms_per_step": round(med("fetch"), 3),
            "fetch_ms_range": [round(min(r["fetch"]), 3), round(max(r["fetch"]), 3)],
            "device_ms_per_step": round(med("dev"), 3), "device_ms_range": [round(min(r["dev"]), 3), round(max(r["dev"]), 3)],
            "d2h_bytes": r["d2h"], "fetch_launches": r["launches"]}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
