"""Cost of per-phoneme duration control and timings.

At the C2 shape (32 utterances x 256 phonemes, medium voice, the voice's default noise scales with on-device Philox
noise, device-resident waveforms) three arms are timed:

  (a) plain   : no controls (a job that never calls sb200_job_set_durations);
  (b) neutral : all-1.0 scales and all -1 frames, plus the frames per id fetched after every step (sb200_job_id_frames);
  (c) scaled  : per-id scales drawn from {0.8, 1.0, 1.25}.

The arms alternate, `--runs` times over, so each arm's run-to-run spread can be compared with the others.  Audio seconds
are counted at the voice's sample rate from what each arm produced.  Prints the device name and power limit, then one
JSON line per arm and run (audio-s/s by wall clock and by device time, ms per step).

  python tools/bench_durations.py --steps 10 --warmup 3 --runs 3
"""
import argparse
import atexit
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--utts", type=int, default=32)
    ap.add_argument("--phonemes", type=int, default=256)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_durations: no CUDA device visible")
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
    lens = [len(b) for b in batches]
    rng = np.random.default_rng(5)
    ones = [np.ones(n, np.float32) for n in lens]
    predicted = [np.full(n, -1, np.int32) for n in lens]
    scaled = [rng.choice(np.array([0.8, 1.0, 1.25], np.float32), size=n) for n in lens]

    def step(kind):
        job = SynthesisJob(model, batches)
        if kind == "b_neutral":
            job.set_durations(ones, predicted)
        elif kind == "c_scaled":
            job.set_durations(scaled, None)
        ms = job.run()
        if kind == "b_neutral":
            job.id_frames()
        audio = sum(job.lengths()[1]) / sr
        job.close()
        return audio, ms

    print(json.dumps(device_info()), flush=True)
    arms = ("a_plain", "b_neutral", "c_scaled")
    for kind in arms:
        for _ in range(max(args.warmup, 1)):
            step(kind)
    for run in range(args.runs):
        for kind in arms:
            torch.cuda.synchronize()
            audio_s, dev_ms = 0.0, 0.0
            t0 = time.perf_counter()
            for _ in range(args.steps):
                a, ms = step(kind)
                audio_s += a
                dev_ms += ms
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            print(json.dumps({
                "arm": kind, "run": run, "shape": f"{args.utts}x{args.phonemes}", "sample_rate": sr, "steps": args.steps,
                "audio_s_per_s_wall": round(audio_s / wall, 1), "audio_s_per_s_device": round(audio_s / (dev_ms / 1e3), 1),
                "wall_ms_per_step": round(wall * 1e3 / args.steps, 3), "device_ms_per_step": round(dev_ms / args.steps, 3),
                "audio_s_per_step": round(audio_s / args.steps, 3)}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
