"""Throughput of batches whose utterances speak with blends of a multi-speaker voice's speakers.

At the C2 shape (32 utterances x 256 phonemes, device-resident results, the voice's default noise scales with seeded
on-device noise) on a synthetic 32-speaker medium voice, four arms run the same utterances:

  (a) speakers : utterance b speaks as speaker b (per-utterance configs, today's path);
  (b) blend2   : utterance b speaks with its own 2-speaker blend {b: 0.7, b + 1: 0.3};
  (c) blend32  : utterance b speaks with its own 32-speaker blend (weights rotated by b);
  (d) shared32 : every utterance speaks with one 32-speaker blend.

Forming g costs gin * n fused multiply-adds per slot and the biases cost what they cost with plain speakers, so the arms
are expected to agree within run-to-run spread.  The arms are alternated round by round; each round times --steps
steps of each arm after its warm-up.  Prints the device name and power limit, then one JSON line per arm with the
median and range over rounds of wall and device ms per step and of audio-s/s.

With --profile, one separate run of each blended arm under torch.profiler reports the device time of the blend-table
and bias kernels (blend_g_kernel, cond_bias_kernel) per step.

  python tools/bench_blends.py --steps 5 --warmup 2 --rounds 5
  python tools/bench_blends.py --profile
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

N_SPEAKERS = 32


def arms(n_utts):
    rot = lambda b: {(b + k) % N_SPEAKERS: 1.0 + k for k in range(N_SPEAKERS)}
    return {"a_speakers": (True, None),
            "b_blend2": (False, [{b % N_SPEAKERS: 0.7, (b + 1) % N_SPEAKERS: 0.3} for b in range(n_utts)]),
            "c_blend32": (False, [rot(b) for b in range(n_utts)]),
            "d_shared32": (False, [rot(0)] * n_utts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--utts", type=int, default=32)
    ap.add_argument("--phonemes", type=int, default=256)
    ap.add_argument("--profile", action="store_true", help="time the blend and bias kernels with torch.profiler")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_blends: no CUDA device visible")
    import sonata_b200
    from bench_voices import device_info
    from sonata_b200 import PiperSynthesisConfig, _native, voicegen, workload
    from sonata_b200.job import SynthesisJob
    if not os.path.exists(_native.LIB_PATH):
        from sonata_b200 import build
        build.build()
    if not os.environ.get("SONATA_B200_VOICE_DIR"):        # generated voices never go into the tree
        os.environ["SONATA_B200_VOICE_DIR"] = tempfile.mkdtemp(prefix="sonata_voices_")
        atexit.register(shutil.rmtree, os.environ["SONATA_B200_VOICE_DIR"], True)

    model = sonata_b200.from_config_path(
        voicegen.write_voice(voicegen.default_voice_dir(), "medium", n_speakers=N_SPEAKERS), device=0)
    sr = model.audio_output_info().sample_rate
    base = model.get_fallback_synthesis_config()
    batches = [workload.synthetic_ids(args.phonemes, utt=u) for u in range(args.utts)]
    seeds = [7000 + b for b in range(args.utts)]
    speakers = [PiperSynthesisConfig(b % N_SPEAKERS, base.noise_scale, base.length_scale, base.noise_w)
                for b in range(args.utts)]
    plan = arms(args.utts)

    def step(name):
        plain, blends = plan[name]
        job = SynthesisJob(model, batches, configs=speakers if plain else None, seeds=seeds, speaker_blends=blends)
        ms = job.run()
        audio = sum(job.lengths()[1]) / sr
        job.close()
        return audio, ms

    print(json.dumps(device_info()), flush=True)
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for name in plan:
            for _ in range(max(args.warmup, 1)):
                step(name)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    step(name)
                torch.cuda.synchronize()
            us = {}
            for e in prof.key_averages():
                for k in ("blend_g_kernel", "cond_bias_kernel"):
                    if k in e.key:
                        us[k] = us.get(k, 0.0) + e.device_time_total
            print(json.dumps({"arm": name, "profile_steps": args.steps,
                              "us_per_step": {k: round(v / args.steps, 2) for k, v in us.items()}}), flush=True)
        model.close()
        return

    for name in plan:
        for _ in range(max(args.warmup, 1)):
            step(name)
    rec = {name: [] for name in plan}
    for _ in range(args.rounds):
        for name in plan:
            torch.cuda.synchronize()
            audio_s, dev_ms = 0.0, 0.0
            t0 = time.perf_counter()
            for _ in range(args.steps):
                a, ms = step(name)
                audio_s += a
                dev_ms += ms
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            rec[name].append((wall * 1e3 / args.steps, dev_ms / args.steps, audio_s / wall))
    for name, rows in rec.items():
        col = lambda i: [r[i] for r in rows]
        summ = lambda v: {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}
        print(json.dumps({"arm": name, "shape": f"{args.utts}x{args.phonemes}", "rounds": args.rounds,
                          "steps": args.steps, "wall_ms_per_step": summ(col(0)), "device_ms_per_step": summ(col(1)),
                          "audio_s_per_s_wall": summ(col(2))}), flush=True)
    model.close()


if __name__ == "__main__":
    main()
