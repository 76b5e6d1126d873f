"""Cost of output-rate resampling at the C2 shape.

32 utterances x 256 phonemes on the medium voice (22 050 Hz), its default noise scales, every utterance seeded.  Each
step synthesises the batch and fetches the f32 result to the host.  Four arms:

  (a) none      : no output rate;
  (b) dev_48k   : every utterance at 48 kHz, resampled on the device;
  (c) dev_8k    : every utterance at 8 kHz, resampled on the device;
  (d) host_48k  : arm (a)'s result resampled to 48 kHz on the host, one thread, with scipy.signal.resample_poly.

The arms alternate over --rounds rounds of --steps steps each, so drift in the card's clocks reaches every arm alike.
Prints the device name and power limit, then one JSON line per arm: wall and device ms per step (medians over rounds,
and the spread), audio-s/s, the device time of the "resample" region and its achieved bytes/s (the bytes it must move:
input and output samples once, plus the tap tables) against the H100 SXM's 3.35 TB/s of HBM3.

  python tools/bench_resample.py --steps 10 --warmup 3 --rounds 5
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

HBM_BYTES_PER_S = 3.35e12


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
        sys.exit("bench_resample: no CUDA device visible")
    from scipy.signal import resample_poly
    import sonata_b200
    from bench_voices import device_info
    from sonata_b200 import _native, voicegen, workload
    from sonata_b200.job import SynthesisJob
    if not os.path.exists(_native.LIB_PATH):
        from sonata_b200 import build
        build.build()
    if not os.environ.get("SONATA_B200_VOICE_DIR"):        # generated voices never go into the tree
        os.environ["SONATA_B200_VOICE_DIR"] = tempfile.mkdtemp(prefix="sonata_voices_")
        atexit.register(shutil.rmtree, os.environ["SONATA_B200_VOICE_DIR"], True)

    model = sonata_b200.from_config_path(voicegen.write_voice(voicegen.default_voice_dir(), "medium"), device=0)
    sr = model.audio_output_info().sample_rate
    batches = [workload.synthetic_ids(args.phonemes, utt=u) for u in range(args.utts)]
    seeds = [1000 + b for b in range(args.utts)]
    arms = {"a_none": None, "b_dev_48k": 48000, "c_dev_8k": 8000, "d_host_48k": "host"}

    def step(rate):
        job = SynthesisJob(model, batches, seeds=seeds,
                           output_rates=[rate] * args.utts if isinstance(rate, int) else None)
        ms = job.run()
        audio = job.fetch()
        if rate == "host":
            audio = [resample_poly(a.samples.as_slice(), 320, 147) for a in audio]
        audio_s = sum(job.lengths()[0]) * 256 / sr
        rs = [r for r in job.profile() if r["name"] == "resample"]
        job.close()
        return audio_s, ms, sum(r["ms"] for r in rs), sum(r["bytes"] for r in rs)

    print(json.dumps(device_info()), flush=True)
    for rate in arms.values():
        for _ in range(max(args.warmup, 1)):
            step(rate)
    torch.cuda.synchronize()
    res = {name: {"wall": [], "dev": [], "rs": [], "audio": [], "bytes": 0.0} for name in arms}
    for _ in range(args.rounds):
        for name, rate in arms.items():
            audio_s = dev_ms = rs_ms = 0.0
            t0 = time.perf_counter()
            for _ in range(args.steps):
                a, ms, r_ms, r_bytes = step(rate)
                audio_s += a
                dev_ms += ms
                rs_ms += r_ms
                res[name]["bytes"] = r_bytes
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            r = res[name]
            r["wall"].append(wall * 1e3 / args.steps)
            r["dev"].append(dev_ms / args.steps)
            r["rs"].append(rs_ms / args.steps)
            r["audio"].append(audio_s / args.steps)
    for name, r in res.items():
        med = lambda k: statistics.median(r[k])
        rs_ms = med("rs")
        bps = r["bytes"] / (rs_ms / 1e3) if rs_ms > 0 else None
        print(json.dumps({
            "arm": name, "shape": f"{args.utts}x{args.phonemes}", "steps": args.steps, "rounds": args.rounds,
            "wall_ms_per_step": round(med("wall"), 3), "wall_ms_range": [round(min(r["wall"]), 3), round(max(r["wall"]), 3)],
            "device_ms_per_step": round(med("dev"), 3), "device_ms_range": [round(min(r["dev"]), 3), round(max(r["dev"]), 3)],
            "resample_ms_per_step": round(rs_ms, 4), "resample_bytes": r["bytes"],
            "resample_bytes_per_s": None if bps is None else round(bps / 1e9, 1) * 1e9,
            "resample_share_of_hbm_peak": None if bps is None else round(bps / HBM_BYTES_PER_S, 4),
            "audio_s_per_s_wall": round(med("audio") / (med("wall") / 1e3), 1),
            "audio_s_per_s_device": round(med("audio") / (med("dev") / 1e3), 1)}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
