"""Throughput of the synthetic x_low, low and medium voices at one shape, each at its own sample rate.

bench.py measures the medium / high workloads at 22.05 kHz; this script puts the 16 kHz qualities beside medium at
the C2 shape: 32 utterances x 256 phonemes in one device-resident pass (results stay in HBM), the voice's own
inference scales with on-device Philox noise.  Audio seconds are samples / the voice's sample rate.  Prints one JSON
line per voice (audio-s/s, device ms per step, per-region ms of the last profiled step from sb200_job_profile) and the
device name and power limit, read in the same run.

  python tools/bench_voices.py --steps 10 --warmup 3 [--voices x_low,low,medium]
"""
import argparse
import atexit
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def device_info():
    import torch
    info = {"device": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--voices", default="x_low,low,medium")
    ap.add_argument("--utts", type=int, default=32)
    ap.add_argument("--phonemes", type=int, default=256)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_voices: no CUDA device visible")
    import sonata_b200
    from sonata_b200 import _native, voicegen, workload
    from sonata_b200.job import SynthesisJob
    if not os.path.exists(_native.LIB_PATH):
        from sonata_b200 import build
        build.build()
    if not os.environ.get("SONATA_B200_VOICE_DIR"):        # generated voices never go into the tree
        os.environ["SONATA_B200_VOICE_DIR"] = tempfile.mkdtemp(prefix="sonata_voices_")
        atexit.register(shutil.rmtree, os.environ["SONATA_B200_VOICE_DIR"], True)

    batches = [workload.synthetic_ids(args.phonemes, utt=u) for u in range(args.utts)]
    print(json.dumps(device_info()), flush=True)
    for q in args.voices.split(","):
        model = sonata_b200.from_config_path(voicegen.write_voice(voicegen.default_voice_dir(), q), device=0)
        sr = model.audio_output_info().sample_rate
        for _ in range(max(args.warmup, 1)):
            job = SynthesisJob(model, batches)
            job.run()
            job.close()
        torch.cuda.synchronize()
        audio_s, dev_ms, regions = 0.0, 0.0, []
        t0 = time.perf_counter()
        for _ in range(args.steps):
            job = SynthesisJob(model, batches)
            dev_ms += job.run()
            audio_s += sum(job.lengths()[1]) / sr
            regions = job.profile()
            job.close()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        print(json.dumps({
            "voice": q, "sample_rate": sr, "shape": f"{args.utts}x{args.phonemes}", "steps": args.steps,
            "audio_s_per_s_wall": round(audio_s / wall, 1), "audio_s_per_s_device": round(audio_s / (dev_ms / 1e3), 1),
            "device_ms_per_step": round(dev_ms / args.steps, 3), "audio_s_per_step": round(audio_s / args.steps, 3),
            "regions_ms": {r["name"]: round(r["ms"], 3) for r in regions},
        }), flush=True)
        model.close()


if __name__ == "__main__":
    main()
