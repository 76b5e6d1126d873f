"""Cost of loudness normalisation at the C2 shape.

32 utterances x 256 phonemes on the medium voice (22 050 Hz), its default noise scales, every utterance seeded.  Each
step synthesises the batch and fetches the f32 result to the host.  Four arms:

  (a) none        : no loudness target;
  (b) dev         : every utterance at -16 LUFS, measured and scaled on the device;
  (c) dev_48k     : every utterance at -16 LUFS at a 48 kHz output rate (resampled, then measured at 48 kHz);
  (d) host        : arm (a)'s result measured and scaled on the host, one thread, with the float64 reference meter
                    (tests/loudness_reference.py, scipy.signal.lfilter).

The arms alternate over --rounds rounds of --steps steps each, so drift in the card's clocks reaches every arm alike.
Prints the device name and power limit, then one JSON line per arm: wall and device ms per step (medians over rounds,
and the spread), audio-s/s, and the device time and algorithmic bytes of the "loudness" region.

  python tools/bench_loudness.py --steps 10 --warmup 3 --rounds 5
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

TARGET = -16.0


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
        sys.exit("bench_loudness: no CUDA device visible")
    import loudness_reference as lr
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
    n = args.utts
    arms = {"a_none": (None, None), "b_dev": ([TARGET] * n, None), "c_dev_48k": ([TARGET] * n, [48000] * n),
            "d_host": ("host", None)}

    def step(arm):
        targets, rates = arm
        job = SynthesisJob(model, batches, seeds=seeds, output_rates=rates,
                           loudness=targets if isinstance(targets, list) else None)
        ms = job.run()
        audio = job.fetch()
        if targets == "host":
            out = []
            for a in audio:
                x = a.samples.as_slice()
                out.append(x * lr.gain(x, TARGET, lr.integrated(x, sr)))
        audio_s = sum(job.lengths()[0]) * 256 / sr
        ld = [r for r in job.profile() if r["name"] == "loudness"]
        job.close()
        return audio_s, ms, sum(r["ms"] for r in ld), sum(r["bytes"] for r in ld)

    print(json.dumps(device_info()), flush=True)
    for arm in arms.values():
        for _ in range(max(args.warmup, 1)):
            step(arm)
    torch.cuda.synchronize()
    res = {name: {"wall": [], "dev": [], "ld": [], "audio": [], "bytes": 0.0} for name in arms}
    for _ in range(args.rounds):
        for name, arm in arms.items():
            audio_s = dev_ms = ld_ms = 0.0
            t0 = time.perf_counter()
            for _ in range(args.steps):
                a, ms, l_ms, l_bytes = step(arm)
                audio_s += a
                dev_ms += ms
                ld_ms += l_ms
                res[name]["bytes"] = l_bytes
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            r = res[name]
            r["wall"].append(wall * 1e3 / args.steps)
            r["dev"].append(dev_ms / args.steps)
            r["ld"].append(ld_ms / args.steps)
            r["audio"].append(audio_s / args.steps)
    for name, r in res.items():
        med = lambda k: statistics.median(r[k])
        print(json.dumps({
            "arm": name, "shape": f"{args.utts}x{args.phonemes}", "steps": args.steps, "rounds": args.rounds,
            "wall_ms_per_step": round(med("wall"), 3), "wall_ms_range": [round(min(r["wall"]), 3), round(max(r["wall"]), 3)],
            "device_ms_per_step": round(med("dev"), 3), "device_ms_range": [round(min(r["dev"]), 3), round(max(r["dev"]), 3)],
            "loudness_ms_per_step": round(med("ld"), 4), "loudness_bytes": r["bytes"],
            "audio_s_per_s_wall": round(med("audio") / (med("wall") / 1e3), 1),
            "audio_s_per_s_device": round(med("audio") / (med("dev") / 1e3), 1)}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
