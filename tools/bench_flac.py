"""Cost and ratio of FLAC output.

Part 1, the C2 shape: 32 utterances x 256 phonemes on the medium voice, its default noise scales, every utterance
seeded, at the voice's rate (22 050 Hz) and at 8 kHz.  Each step synthesises the batch and fetches the result to the
host in one of three ways, the arms alternating over --rounds rounds of --steps steps:

  f32  : job.fetch() (4 bytes per sample);
  i16  : job.fetch_i16() (2 bytes per sample, converted on the device);
  flac : job.fetch_flac() (one FLAC stream per utterance, encoded on the device).

One JSON line per arm: wall ms per step and of the fetch alone (medians over rounds, and the spread), the run's device
ms per step, the device->host bytes, bits per sample and the fetch's kernel launches.

Part 2, in a run of its own: the device time of the FLAC fetch's kernels (torch.profiler's CUDA kernel records, summed
per kernel over --steps fetches of one finished job).

Part 3: flac_encode on a SYNTHETIC compressible signal generated here (a seeded harmonic source with vibrato through
three resonators, 60 s at 22 050 Hz): ratio, bits per sample and encoder throughput.  The synthetic voices produce
near-white noise, which FLAC hardly compresses; this signal shows what the encoder does with a predictable one.

Prints the device name and power limit first.

  python tools/bench_flac.py --steps 10 --warmup 3 --rounds 5
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


def synthetic_signal(rate=22050, seconds=60, seed=1234):
    """A seeded harmonic source (f0 around 120 Hz with vibrato, 1/h harmonics) through three two-pole resonators."""
    import numpy as np
    from scipy.signal import lfilter
    rng = np.random.default_rng(seed)
    n = rate * seconds
    t = np.arange(n) / rate
    f0 = 120.0 * (1.0 + 0.03 * np.sin(2 * np.pi * 5.0 * t)) * (1.0 + 0.1 * np.sin(2 * np.pi * 0.2 * t))
    phase = 2 * np.pi * np.cumsum(f0) / rate
    x = sum(np.sin(h * phase) / h for h in range(1, 30))
    x = x + 0.01 * rng.standard_normal(n)
    for fc, bw in ((500.0, 80.0), (1500.0, 120.0), (2500.0, 160.0)):
        r = np.exp(-np.pi * bw / rate)
        x = lfilter([1.0 - r], [1.0, -2.0 * r * np.cos(2 * np.pi * fc / rate), r * r], x)
    x = x / np.abs(x).max() * 0.5
    return (x * 32767).astype(np.int16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--utts", type=int, default=32)
    ap.add_argument("--phonemes", type=int, default=256)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_flac: no CUDA device visible")
    import sonata_b200
    from bench_voices import device_info
    from sonata_b200 import _native, voicegen, workload
    from sonata_b200.core import flac_encode
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

    def flac_fetch(job):
        streams = job.fetch_flac()
        # frame bytes plus the size table (4 x 8 bytes per stream); STREAMINFO is built on the host
        return sum(len(s) - 42 for s in streams) + 32 * len(streams), 8.0 * sum(len(s) for s in streams)

    fetches = {"f32": lambda job: (4 * sum(job.lengths()[1]), None),
               "i16": lambda job: (2 * sum(job.lengths()[1]), None),
               "flac": flac_fetch}
    calls = {"f32": lambda job: job.fetch(), "i16": lambda job: job.fetch_i16()}
    arms = {f"{name}@{rate or 'voice'}": (rate, name) for rate in (None, 8000) for name in fetches}

    def step(arm):
        rate, name = arm
        job = SynthesisJob(model, batches, seeds=seeds, output_rates=None if rate is None else [rate] * n)
        ms = job.run()
        samples = sum(job.lengths()[1])
        l0 = lib.sb200_launch_count()
        t0 = time.perf_counter()
        if name == "flac":
            d2h, bits = flac_fetch(job)
        else:
            calls[name](job)
            d2h, bits = fetches[name](job)
        fetch_ms = (time.perf_counter() - t0) * 1e3
        launches = lib.sb200_launch_count() - l0
        job.close()
        return ms, fetch_ms, d2h, launches, (bits / samples if bits else 8.0 * d2h / samples)

    print(json.dumps(device_info()), flush=True)
    for arm in arms.values():
        for _ in range(max(args.warmup, 1)):
            step(arm)
    torch.cuda.synchronize()
    res = {name: {"wall": [], "dev": [], "fetch": [], "d2h": 0, "launches": 0, "bps": 0.0} for name in arms}
    for _ in range(args.rounds):
        for name, arm in arms.items():
            dev_ms = fetch_ms = 0.0
            t0 = time.perf_counter()
            for _ in range(args.steps):
                ms, f_ms, d2h, launches, bps = step(arm)
                dev_ms += ms
                fetch_ms += f_ms
                res[name]["d2h"], res[name]["launches"], res[name]["bps"] = d2h, launches, bps
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
            "d2h_bytes": r["d2h"], "bits_per_sample": round(r["bps"], 4), "fetch_launches": r["launches"]}), flush=True)

    # Part 2: the FLAC fetch's kernels alone
    from torch.profiler import ProfilerActivity, profile
    for rate in (None, 8000):
        job = SynthesisJob(model, batches, seeds=seeds, output_rates=None if rate is None else [rate] * n)
        job.run()
        job.fetch_flac()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                job.fetch_flac()
        per = {}
        for e in prof.events():
            if e.device_type.name == "CUDA" and ("flac" in e.name or "i16_" in e.name):
                key = ("flac_" + e.name.split("flac_")[1].split("_kernel")[0]) if "flac_" in e.name else \
                      e.name.split("(")[0].split("<")[0]
                per[key] = per.get(key, 0.0) + e.device_time / 1e3 / args.steps
        print(json.dumps({"flac_fetch_kernels_ms": {k: round(v, 4) for k, v in sorted(per.items())},
                          "rate": rate or "voice", "samples": sum(job.lengths()[1])}), flush=True)
        job.close()

    # Part 3: a synthetic compressible signal
    x = synthetic_signal()
    flac_encode(x, 22050)
    times = []
    for _ in range(max(args.steps, 3)):
        t0 = time.perf_counter()
        data = flac_encode(x, 22050)
        times.append(time.perf_counter() - t0)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        flac_encode(x, 22050)
    kern = sum(e.device_time for e in prof.events() if e.device_type.name == "CUDA" and "flac" in e.name) / 1e3
    t = statistics.median(times)
    print(json.dumps({"signal": "synthetic harmonic source through resonators (not speech)", "rate": 22050,
                      "samples": int(x.size), "flac_bytes": len(data), "ratio_vs_i16": round(len(data) / (2 * x.size), 4),
                      "bits_per_sample": round(8 * len(data) / x.size, 3), "encode_wall_ms": round(t * 1e3, 3),
                      "encode_wall_ms_range": [round(min(times) * 1e3, 3), round(max(times) * 1e3, 3)],
                      "encode_kernel_ms": round(kern, 3),
                      "msamples_per_s_wall": round(x.size / t / 1e6, 2)}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
