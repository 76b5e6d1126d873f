"""Cost of pitch and tempo shifting at the C2 shape.

32 utterances x 256 phonemes on the medium voice (22 050 Hz), its default noise scales, every utterance seeded.  Each
step synthesises the batch and fetches the f32 result to the host.  Six arms:

  (a) none        : no ratios;
  (b) pitch       : every utterance at pitch 1.25 (stretch by 1.25, then resample by 1.25);
  (c) tempo       : every utterance at tempo 1.5 (stretch only);
  (d) both        : pitch 0.8 and tempo 2.0;
  (e) chain       : pitch 1.25, then a 48 kHz output rate, then -16 LUFS;
  (f) host        : arm (a)'s result put through the numpy specification (tests/prosody_reference.py) at pitch 1.25,
                    one thread.

The arms alternate over --rounds rounds of --steps steps each, so drift in the card's clocks reaches every arm alike.
Prints the device name and power limit, then one JSON line per arm: wall and device ms per step (medians over rounds,
and the spread), the device time, algorithmic bytes and operations of the "stretch" and "pitch" regions, and the
"stretch" region's time per frame step of its longest utterance (the offset chain is sequential per utterance, so the
region lasts as long as the utterance with the most frames).

  python tools/bench_prosody.py --steps 5 --warmup 2 --rounds 3
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--utts", type=int, default=32)
    ap.add_argument("--phonemes", type=int, default=256)
    ap.add_argument("--no-host", action="store_true", help="skip the host arm")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_prosody: no CUDA device visible")
    import prosody_reference as pr
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
    n = args.utts
    batches = [workload.synthetic_ids(args.phonemes, utt=u) for u in range(n)]
    seeds = [1000 + b for b in range(n)]
    arms = {"a_none": {}, "b_pitch_1.25": dict(pitches=[1.25] * n), "c_tempo_1.5": dict(tempos=[1.5] * n),
            "d_pitch_0.8_tempo_2": dict(pitches=[0.8] * n, tempos=[2.0] * n),
            "e_pitch_48k_lufs": dict(pitches=[1.25] * n, output_rates=[48000] * n, loudness=[-16.0] * n)}
    if not args.no_host:
        arms["f_host_pitch_1.25"] = "host"

    def step(arm):
        job = SynthesisJob(model, batches, seeds=seeds, **({} if arm == "host" else arm))
        ms = job.run()
        audio = job.fetch()
        if arm == "host":
            for a in audio:
                pr.process(a.samples.as_slice(), sr, 1.25, None)
        audio_s = sum(job.lengths()[0]) * 256 / sr
        reg = {r["name"]: r for r in job.profile() if r["name"] in ("stretch", "pitch")}
        frames = int(job.prosody()[2].max()) if reg else 0
        job.close()
        return audio_s, ms, reg, frames

    print(json.dumps(device_info()), flush=True)
    for arm in arms.values():
        for _ in range(max(args.warmup, 1) if arm != "host" else 1):
            step(arm)
    torch.cuda.synchronize()
    res = {name: {"wall": [], "dev": [], "stretch": [], "pitch": [], "audio": [], "reg": {}, "frames": 0} for name in arms}
    for _ in range(args.rounds):
        for name, arm in arms.items():
            steps = 1 if arm == "host" else args.steps
            audio_s = dev_ms = st_ms = pi_ms = 0.0
            t0 = time.perf_counter()
            for _ in range(steps):
                a, ms, reg, frames = step(arm)
                audio_s += a
                dev_ms += ms
                st_ms += reg.get("stretch", {}).get("ms", 0.0)
                pi_ms += reg.get("pitch", {}).get("ms", 0.0)
                res[name]["reg"], res[name]["frames"] = reg, frames
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            r = res[name]
            r["wall"].append(wall * 1e3 / steps)
            r["dev"].append(dev_ms / steps)
            r["stretch"].append(st_ms / steps)
            r["pitch"].append(pi_ms / steps)
            r["audio"].append(audio_s / steps)
    for name, r in res.items():
        med = lambda k: statistics.median(r[k])
        rng = lambda k, d=3: [round(min(r[k]), d), round(max(r[k]), d)]
        out = {"arm": name, "shape": f"{args.utts}x{args.phonemes}", "steps": args.steps, "rounds": args.rounds,
               "wall_ms_per_step": round(med("wall"), 3), "wall_ms_range": rng("wall"),
               "device_ms_per_step": round(med("dev"), 3), "device_ms_range": rng("dev"),
               "stretch_ms_per_step": round(med("stretch"), 4), "stretch_ms_range": rng("stretch", 4),
               "pitch_ms_per_step": round(med("pitch"), 4), "pitch_ms_range": rng("pitch", 4),
               "audio_s_per_s_wall": round(med("audio") / (med("wall") / 1e3), 1)}
        for k, v in r["reg"].items():
            out[k + "_bytes"], out[k + "_ops"] = v["bytes"], v["flops"]
        if r["frames"] > 1:
            out["longest_utterance_frames"] = r["frames"]
            out["stretch_us_per_frame_step"] = round(med("stretch") * 1e3 / (r["frames"] - 1), 3)
        print(json.dumps(out), flush=True)
    model.close()


if __name__ == "__main__":
    main()
