"""Cost of per-utterance noise seeds at the C2 shape.

32 utterances x 256 phonemes on the medium voice, its default noise scales (0.667 / 0.8), device-resident results.
Three arms run the same batch:

  (a) unseeded : positional Philox noise (randn_kernel), what bench.py times;
  (b) seeded   : every utterance seeded (randn_seg_kernel writes both noise tensors);
  (c) half     : the even utterances seeded, the odd ones positional.

The arms alternate (a, b, c, a, b, c, ...) over --rounds rounds of --steps steps each, so drift in the card's clocks
reaches every arm alike.  Prints the device name and power limit, then one JSON line per arm: wall and device ms per
step and audio-s/s (medians over rounds, and the spread), plus the device time of the "align" region, where eps_z is
drawn.

  python tools/bench_seeds.py --steps 10 --warmup 3 --rounds 5
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

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_seeds: no CUDA device visible")
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
    arms = {"a_unseeded": None,
            "b_seeded": [1000 + b for b in range(args.utts)],
            "c_half": [1000 + b if b % 2 == 0 else None for b in range(args.utts)]}

    def step(seeds):
        job = SynthesisJob(model, batches, seeds=seeds)
        ms = job.run()
        audio = sum(job.lengths()[1]) / sr
        align = sum(r["ms"] for r in job.profile() if r["name"] == "align")
        job.close()
        return audio, ms, align

    print(json.dumps(device_info()), flush=True)
    for seeds in arms.values():
        for _ in range(max(args.warmup, 1)):
            step(seeds)
    torch.cuda.synchronize()
    res = {name: {"wall": [], "dev": [], "align": [], "audio": []} for name in arms}
    for _ in range(args.rounds):
        for name, seeds in arms.items():
            audio_s = dev_ms = align_ms = 0.0
            t0 = time.perf_counter()
            for _ in range(args.steps):
                a, ms, al = step(seeds)
                audio_s += a
                dev_ms += ms
                align_ms += al
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            r = res[name]
            r["wall"].append(wall * 1e3 / args.steps)
            r["dev"].append(dev_ms / args.steps)
            r["align"].append(align_ms / args.steps)
            r["audio"].append(audio_s / args.steps)
    for name, r in res.items():
        med = lambda k: statistics.median(r[k])
        print(json.dumps({
            "arm": name, "shape": f"{args.utts}x{args.phonemes}", "steps": args.steps, "rounds": args.rounds,
            "wall_ms_per_step": round(med("wall"), 3), "wall_ms_range": [round(min(r["wall"]), 3), round(max(r["wall"]), 3)],
            "device_ms_per_step": round(med("dev"), 3), "device_ms_range": [round(min(r["dev"]), 3), round(max(r["dev"]), 3)],
            "align_ms_per_step": round(med("align"), 4),
            "audio_s_per_s_wall": round(med("audio") / (med("wall") / 1e3), 1),
            "audio_s_per_s_device": round(med("audio") / (med("dev") / 1e3), 1)}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
