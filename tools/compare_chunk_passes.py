"""Compares two builds of the library on every chunk entry point and on batch jobs with output rates: each build runs
the same calls in a process of its own, and every result must be byte-identical and every call must add the same
number of kernel launches (sb200_launch_count).

Calls, on a 4-speaker medium voice with zero noise over the chunk set of tests/test_stream_batch_gpu.py:
  sb200_decode_chunk and sb200_decode_chunks;
  sb200_decode_chunks_i16 with trims and gains, fade 0 and 42;
  sb200_decode_chunks_resampled with trims and gains, fade 0 and 42, f32 and i16, null resamplers mixed with ones to
  8000 and 48000 Hz, over three consecutive calls per resampler (the last flushing some streams), then the errors of a
  flushed resampler, a resampler twice in one call, a bad last flag and a bad trim, and a call after them;
  libsonataSpeak in realtime mode (its i16 events);
and SynthesisJob with mixed output rates on medium and high: fetch, fetch_i16 and profile() minus its times.

  python tools/compare_chunk_passes.py PARENT_LIB CHILD_LIB
"""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _record(out_path):
    from sonata_b200 import OperationError, PiperSynthesisConfig, voicegen, workload
    from sonata_b200 import _native as N
    from sonata_b200.job import SynthesisJob
    from sonata_b200.piper import Resampler, VitsModel, VitsStreamingModel
    from test_stream_batch_gpu import _chunk_latents, _chunk_set
    from test_libsonata_facade import CALLBACK, ExternError, PiperSynthConfig, SynthesisEvent, SynthesisParams

    res = {}
    lib = N.lib()

    def call(name, f):
        n0 = lib.sb200_launch_count()
        try:
            out = f()
        except OperationError as e:
            out = [np.frombuffer(str(e).encode(), np.uint8)]
        res[name + "/launches"] = np.array([lib.sb200_launch_count() - n0])
        for k, a in enumerate(out):
            res[f"{name}/{k}"] = np.asarray(a.as_slice() if hasattr(a, "as_slice") else a)

    d = voicegen.default_voice_dir()
    m = VitsStreamingModel(voicegen.write_voice(d, "medium", n_speakers=4), device=0)
    chunks = _chunk_set(_chunk_latents(m))
    n = len(chunks)
    trimmed = [c + ((3, 3) if c[2] - c[1] > 6 else (0, 0)) for c in chunks]
    gains = [1.0 if k % 3 else 0.8 for k in range(n)]

    def bad_last(r, pcm16):
        """A last flag of 2, which the Python layer cannot pass."""
        e, lo, hi = chunks[1]
        p64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))  # noqa: E731
        lo_a, hi_a, fl = np.array([lo], np.int64), np.array([hi], np.int64), np.array([2], np.int32)
        outs, lens, err = (C.c_void_p * 1)(), (C.c_size_t * 1)(), N.sb200_error()
        rc = lib.sb200_decode_chunks_resampled(m._h, (C.c_void_p * 1)(e._h.value), p64(lo_a), p64(hi_a), None, None, 1,
                                               0, None, (C.c_void_p * 1)(r._h.value),
                                               fl.ctypes.data_as(C.POINTER(C.c_int32)), int(pcm16), outs, lens,
                                               C.byref(err))
        return [np.array([rc]), np.frombuffer(C.string_at(err.message), np.uint8)]

    call("chunks", lambda: m.infer_decoder_batch(chunks))
    call("chunk", lambda: [e.infer_decoder(lo, hi) for e, lo, hi in chunks[:4]])
    for fade in (0, 42):
        call(f"i16/{fade}", lambda: m.infer_decoder_batch(trimmed, pcm16=True, fade=fade, gains=gains))
        call(f"i16-one/{fade}", lambda: m.infer_decoder_batch([trimmed[1]], pcm16=True, fade=fade))
        for pcm16 in (False, True):
            tag = f"rs/{fade}/{int(pcm16)}"
            rs = [Resampler(m, (8000, 48000)[k % 2]) if k % 3 else None for k in range(n)]
            run = lambda cs, last=None, r=rs: m.infer_decoder_batch(cs, pcm16=pcm16, fade=fade, gains=gains,  # noqa
                                                                   resamplers=r, last=last)
            for step in range(3):
                call(f"{tag}/{step}", lambda: run(trimmed, [step == 2 and k % 2 == 1 for k in range(n)]))
            call(f"{tag}/flushed", lambda: run(trimmed))
            live = [r if k % 2 == 0 else None for k, r in enumerate(rs)]
            call(f"{tag}/twice", lambda: run(trimmed[:3], r=[live[2], None, live[2]]))
            call(f"{tag}/badtrim", lambda: run([trimmed[0], chunks[5] + (1, 1)], r=[live[2], None]))
            call(f"{tag}/badlast", lambda: bad_last(live[2], pcm16))
            call(f"{tag}/after", lambda: run(trimmed, r=live))
    m.close()

    # the facade's realtime mode
    lib.libsonataLoadVoiceFromConfigPath.restype = C.c_void_p
    lib.libsonataLoadVoiceFromConfigPath.argtypes = [C.c_char_p, C.POINTER(ExternError)]
    lib.libsonataSpeak.argtypes = [C.c_void_p, C.c_char_p, SynthesisParams, C.POINTER(ExternError)]
    lib.libsonataSetPiperSynthConfig.argtypes = [C.c_void_p, PiperSynthConfig, C.POINTER(ExternError)]
    lib.libsonataFreeSynthesisEvent.argtypes = [SynthesisEvent]
    lib.libsonataUnloadSonataVoice.argtypes = [C.c_void_p]
    err = ExternError()
    v = lib.libsonataLoadVoiceFromConfigPath(voicegen.write_voice(d, "medium").encode(), C.byref(err))
    lib.libsonataSetPiperSynthConfig(v, PiperSynthConfig(0, 1.0, 0.0, 0.0), C.byref(err))
    events = []

    def cb(ev):
        events.append(np.ctypeslib.as_array(ev.data, shape=(max(ev.len, 1),))[:ev.len].copy())
        lib.libsonataFreeSynthesisEvent(ev)
        return 0
    cb_c = CALLBACK(cb)
    text = ("ðɪs ɪz ə tɛst əv ðə riːəltaɪm moʊd wɪð ə lɔŋɡɚ sɛntəns ðæt niːdz mɔːɹ ðæn wʌn tʃʌŋk ænd sʌm mɔːɹ. "
            "ʃɔːɹt wʌn.")
    call("facade", lambda: (lib.libsonataSpeak(v, text.encode(), SynthesisParams(2, 10, 100, 50, 20, cb_c, 0),
                                                C.byref(err)), events)[1])
    lib.libsonataUnloadSonataVoice(v)

    # batch jobs with mixed output rates
    for q in ("medium", "high"):
        mb = VitsModel(voicegen.write_voice(d, q), device=0)
        mb.set_fallback_synthesis_config(PiperSynthesisConfig(None, 0.667, 1.0, 0.8))
        batches = [list(workload.synthetic_ids(n_ids, utt=90 + i)) for i, n_ids in enumerate((40, 7, 120, 64, 13, 90))]
        job = SynthesisJob(mb, batches, seeds=list(range(len(batches))),
                           output_rates=[0, 8000, 48000, 16000, 44100, mb.audio_output_info().sample_rate])

        def run_job():
            job.run()
            prof = [np.array([r["flops"], r["bytes"], r["launches"]], np.float64) for r in job.profile()]
            names = [np.frombuffer(r["name"].encode(), np.uint8) for r in job.profile()]
            return [a.samples.as_slice() for a in job.fetch()] + job.fetch_i16() + prof + names
        call(f"job/{q}", run_job)
        job.close()
        mb.close()
    np.savez(out_path, **res)


def main():
    if len(sys.argv) == 3 and sys.argv[1] == "--record":
        _record(sys.argv[2])
        return
    libs = sys.argv[1:]
    if len(libs) != 2:
        raise SystemExit(__doc__)
    with tempfile.TemporaryDirectory() as tmp:
        env = dict(os.environ, SONATA_B200_VOICE_DIR=os.path.join(tmp, "voices"))
        outs = []
        for i, lib in enumerate(libs):
            out = os.path.join(tmp, f"{i}.npz")
            subprocess.run([sys.executable, os.path.abspath(__file__), "--record", out],
                           env=dict(env, SB200_LIB=os.path.abspath(lib)), check=True)
            outs.append(dict(np.load(out)))
    a, b = outs
    bad = sorted(k for k in a.keys() | b.keys()
                 if k not in a or k not in b or a[k].dtype != b[k].dtype or a[k].tobytes() != b[k].tobytes())
    launches = {k: int(a[k][0]) for k in sorted(a) if k.endswith("/launches")}
    print(f"{len(a)} arrays compared, {len(bad)} differ; launches per call: {launches}")
    for k in bad:
        print("differs:", k)
    raise SystemExit(1 if bad else 0)


if __name__ == "__main__":
    main()
