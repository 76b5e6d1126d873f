"""Throughput of a batch whose utterances have different speakers and length scales.

A server fed by many users, or synthetic-data generation for speech-recognition training, draws a speaker and scales
per utterance.  At the C2 shape (32 utterances x 256 phonemes, device-resident results, the voice's default noise
scales with on-device Philox noise) on a synthetic 32-speaker medium voice, utterance b speaks as speaker b with a
length_scale from {0.8, 1.0, 1.25}.  Three ways to synthesise that batch are timed:

  (a) mixed   : one pass with per-utterance configs (sb200_job_set_configs);
  (b) split   : what a caller without per-utterance configs has to do: one pass per distinct config, back to back;
  (c) uniform : the same 32 utterances in one pass with one shared config (speaker 0, length_scale 1.0).

Audio seconds are counted at the voice's sample rate from what each arm produced.  Prints the device name and power
limit, then one JSON line per arm (audio-s/s by wall clock and by device time, ms per step) and for (a) and (c) the
per-region device times of the last step.

  python tools/bench_mixed.py --steps 10 --warmup 3
"""
import argparse
import atexit
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

LENGTH_SCALES = (0.8, 1.0, 1.25)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--utts", type=int, default=32)
    ap.add_argument("--phonemes", type=int, default=256)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_mixed: no CUDA device visible")
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

    model = sonata_b200.from_config_path(voicegen.write_voice(voicegen.default_voice_dir(), "medium", n_speakers=32),
                                         device=0)
    sr = model.audio_output_info().sample_rate
    base = model.get_fallback_synthesis_config()
    batches = [workload.synthetic_ids(args.phonemes, utt=u) for u in range(args.utts)]
    mixed = [PiperSynthesisConfig(b % 32, base.noise_scale, LENGTH_SCALES[b % 3], base.noise_w) for b in range(args.utts)]
    uniform = [PiperSynthesisConfig(0, base.noise_scale, 1.0, base.noise_w)] * args.utts

    def step_one_pass(configs):
        job = SynthesisJob(model, batches, configs=configs)
        ms = job.run()
        audio = sum(job.lengths()[1]) / sr
        prof = job.profile()
        job.close()
        return audio, ms, prof

    def step_split(configs):
        # one pass per distinct config (every utterance here has its own speaker, so one pass each), back to back
        groups = {}
        for b, c in enumerate(configs):
            groups.setdefault((c.speaker, c.noise_scale, c.length_scale, c.noise_w), []).append(b)
        audio, ms = 0.0, 0.0
        for idx in groups.values():
            job = SynthesisJob(model, [batches[b] for b in idx], configs=[configs[b] for b in idx])
            ms += job.run()
            audio += sum(job.lengths()[1]) / sr
            job.close()
        return audio, ms, []

    arms = [("a_mixed", lambda: step_one_pass(mixed)), ("b_split", lambda: step_split(mixed)),
            ("c_uniform", lambda: step_one_pass(uniform))]
    print(json.dumps(device_info()), flush=True)
    for name, step in arms:
        for _ in range(max(args.warmup, 1)):
            step()
        torch.cuda.synchronize()
        audio_s, dev_ms, prof = 0.0, 0.0, []
        t0 = time.perf_counter()
        for _ in range(args.steps):
            a, ms, prof = step()
            audio_s += a
            dev_ms += ms
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        line = {"arm": name, "shape": f"{args.utts}x{args.phonemes}", "sample_rate": sr, "steps": args.steps,
                "audio_s_per_s_wall": round(audio_s / wall, 1), "audio_s_per_s_device": round(audio_s / (dev_ms / 1e3), 1),
                "wall_ms_per_step": round(wall * 1e3 / args.steps, 3), "device_ms_per_step": round(dev_ms / args.steps, 3),
                "audio_s_per_step": round(audio_s / args.steps, 3)}
        if prof:
            line["regions_ms"] = {r["name"]: round(r["ms"], 3) for r in prof}
        print(json.dumps(line), flush=True)
    model.close()


if __name__ == "__main__":
    main()
