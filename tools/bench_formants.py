"""Cost of the formant stage at the C2 shape.

32 utterances x 256 phonemes on the medium voice (22 050 Hz), its default noise scales, every utterance seeded.  Each
step synthesises the batch as a job and fetches the f32 result to the host.  Five arms:

  (a) none              : no ratios;
  (b) pitch             : every utterance at pitch 1.25;
  (c) pitch_formant     : pitch 1.25 with formant ratio 1 (a formant-preserving pitch shift);
  (d) formant           : formant ratio 1.2 alone (a timbre shift at the same pitch and duration);
  (e) question_formant  : a question contour (1 on the first 75 % of each utterance's ids, then rising in five steps
                          to 1.3) with formant ratio 1.

The arms alternate over --rounds rounds of --steps steps each.  Prints the device name and power limit, then one JSON
line per arm: wall and device ms per step (medians over rounds), and the "stretch", "pitch" and "formant" regions' ms,
algorithmic bytes and FP64 operations (computed from the shapes).

  python tools/bench_formants.py --steps 5 --warmup 2 --rounds 3
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
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--utts", type=int, default=32)
    ap.add_argument("--phonemes", type=int, default=256)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_formants: no CUDA device visible")
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
    n = args.utts
    batches = [workload.synthetic_ids(args.phonemes, utt=u) for u in range(n)]
    seeds = [1000 + b for b in range(n)]

    def question(k):
        c = [1.0] * k
        rise = k - int(0.75 * k)
        for i in range(int(0.75 * k), k):
            c[i] = 1.0 + 0.06 * (1 + (i - int(0.75 * k)) * 5 // rise)
        return c
    arms = {"a_none": {}, "b_pitch_1.25": dict(pitches=[1.25] * n),
            "c_pitch_1.25_formant_1": dict(pitches=[1.25] * n, formants=[1.0] * n),
            "d_formant_1.2": dict(formants=[1.2] * n),
            "e_question_formant_1": dict(pitch_contours=[question(len(b)) for b in batches], formants=[1.0] * n)}
    names = ("stretch", "pitch", "formant")

    def step(arm):
        job = SynthesisJob(model, batches, seeds=seeds, **arm)
        ms = job.run()
        job.fetch()
        reg = {r["name"]: r for r in job.profile() if r["name"] in names}
        job.close()
        return ms, reg

    print(json.dumps(device_info()), flush=True)
    for arm in arms.values():
        for _ in range(max(args.warmup, 1)):
            step(arm)
    torch.cuda.synchronize()
    res = {name: {"wall": [], "dev": [], "reg_ms": {k: [] for k in names}, "reg": {}} for name in arms}
    for _ in range(args.rounds):
        for name, arm in arms.items():
            dev = 0.0
            reg_ms = {k: 0.0 for k in names}
            t0 = time.perf_counter()
            for _ in range(args.steps):
                ms, reg = step(arm)
                dev += ms
                for k in names:
                    reg_ms[k] += reg.get(k, {}).get("ms", 0.0)
                res[name]["reg"] = reg
            torch.cuda.synchronize()
            r = res[name]
            r["wall"].append((time.perf_counter() - t0) * 1e3 / args.steps)
            r["dev"].append(dev / args.steps)
            for k in names:
                r["reg_ms"][k].append(reg_ms[k] / args.steps)
    for name, r in res.items():
        out = {"arm": name, "wall_ms": round(statistics.median(r["wall"]), 2),
               "device_ms": round(statistics.median(r["dev"]), 2),
               "device_ms_spread": round(max(r["dev"]) - min(r["dev"]), 2)}
        for k in names:
            if k in r["reg"]:
                out[k] = {"ms": round(statistics.median(r["reg_ms"][k]), 3), "bytes": r["reg"][k]["bytes"],
                          "flops": r["reg"][k]["flops"]}
        print(json.dumps(out), flush=True)
    model.close()


if __name__ == "__main__":
    main()
