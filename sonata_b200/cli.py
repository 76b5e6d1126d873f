"""`sonata` command-line frontend (SURVEY §8f row N4): the argument set and the JSON-lines protocol of the reference
CLI (crates/frontends/cli/src/main.rs:32-260) over the H100 engine.

    python -m sonata_b200.cli voice.onnx.json -f phonemes.txt -o out.wav --mode parallel
    echo '{"text": "hɛloʊ", "mode": "realtime", "chunk_size": 100}' | python -m sonata_b200.cli voice.onnx.json > pcm.raw

Without `-f`, one JSON request per stdin line (fields of `SynthesisRequest`, main.rs:78-92); without `-o`, raw 16-bit
LE PCM (peak-normalised per sentence / chunk like `as_wave_bytes`) goes to stdout; with `-o` and stdin requests the
files are numbered `<stem>-<n>.<ext>` (main.rs:243-256).  `text` is phonemes, one sentence per line.  With
`--encoding mulaw|alaw` (or a JSON "encoding") the output is G.711 instead, encoded on the GPU: raw bytes on stdout,
or an 8-bit G.711 WAV with `-o`.  With `--encoding flac` each request is one lossless FLAC stream, encoded on the GPU:
on stdout, or as the `-o` file (the same bytes either way); realtime mode refuses it.  With `--speaker-blend
"speaker_3=0.7,speaker_12=0.3"` (or a JSON "speaker_blend": {"speaker_3": 0.7, "12": 0.3}) a multi-speaker voice speaks
with a blend of its speakers, in every mode; a key made of digits is a speaker id, any other a speaker name.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from typing import Optional

from . import from_config_path
from .core import ENCODINGS, FLAC, OperationError, check_encoding
from .piper import (PiperSynthesisConfig, VitsStreamingModel, _check_live_loudness, refuse_formants,
                    refuse_live_loudness, refuse_prosody)
from .synth import AudioOutputConfig, SonataSpeechSynthesizer, _check_loudness, _check_prosody

MODES = ("lazy", "parallel", "realtime")


def _blend_key(key: str):
    key = key.strip()
    return int(key) if key.isdigit() else key


def parse_speaker_blend(text: str) -> dict:
    """The blend of a --speaker-blend value, "name_or_id=weight,...": {speaker id (digits) or name: weight}."""
    out = {}
    for part in text.split(","):
        key, eq, w = part.partition("=")
        if not eq or not key.strip():
            raise OperationError(f"speaker blend: {part.strip()!r} is not speaker=weight")
        try:
            out[_blend_key(key)] = float(w)
        except ValueError:
            raise OperationError(f"speaker blend: the weight {w.strip()!r} of speaker {key.strip()} is not a number")
    return out


def speaker_blend_of(value):
    """A request's speaker blend: None, a --speaker-blend string, or a JSON object {speaker: weight}, whose keys made of
    digits are speaker ids."""
    if value is None:
        return None
    if isinstance(value, str):
        return parse_speaker_blend(value)
    if isinstance(value, dict):
        return {_blend_key(k) if isinstance(k, str) else k: w for k, w in value.items()}
    raise OperationError(f"speaker blend: {value!r} is not an object of speakers and weights")


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="sonata", description="H100-native Piper/VITS synthesis (phoneme input)")
    ap.add_argument("config", help="Model config (<voice>.onnx.json)")
    ap.add_argument("-f", "--input-file", help="Input text file (default stdin: one JSON request per line)")
    ap.add_argument("-o", "--output-file", help="Output WAV file (default stdout: raw i16 PCM)")
    ap.add_argument("--mode", choices=MODES, help="Synthesis mode (default lazy)")
    ap.add_argument("--speaker-id", type=int)
    ap.add_argument("--length-scale", type=float)
    ap.add_argument("--noise-scale", type=float)
    ap.add_argument("--noise-w", type=float)
    ap.add_argument("--rate", type=int, help="Speaking rate [0 - 100] (10 = 1.0x; other values need Sonic, not part of this path)")
    ap.add_argument("--pitch", type=int, help="Speech pitch [0 - 100] (50 = 1.0x)")
    ap.add_argument("--volume", type=int, help="Speech volume [0 - 100]")
    ap.add_argument("--silence", type=int, help="Extra silence (ms) appended to each sentence")
    ap.add_argument("--chunk-size", type=int)
    ap.add_argument("--chunk-padding", type=int)
    ap.add_argument("--seed", type=int, help="Noise seed [0, 2^64): sentence i uses seed + i, so the same input and seed "
                                          "give the same samples (default: positional noise)")
    ap.add_argument("--output-rate", type=int, help="Output sample rate in Hz (8000, 11025, 16000, 22050, 24000, 32000, "
                                                  "44100 or 48000; default the voice's), resampled on the GPU")
    ap.add_argument("--loudness", type=float, metavar="LUFS",
                    help="Target integrated loudness of every sentence in LUFS, [-70, 0] (ITU-R BS.1770-4; e.g. -23 "
                         "EBU R128, -16 podcasts), measured and applied on the GPU; output is then written at a fixed "
                         "scale instead of peak-normalised.  Not in realtime mode")
    ap.add_argument("--live-loudness", type=float, metavar="LUFS",
                    help="Realtime mode only (streaming voices): hold the stream at this loudness in LUFS, [-70, 0], "
                         "with a causal BS.1770 meter of everything delivered so far driving a gain ramped over each "
                         "100 ms, on the GPU, adding no latency; output is then written at a fixed scale.  The first "
                         "100 ms play at gain 1 and peaks are clamped, not limited.  Other modes: use --loudness")
    ap.add_argument("--max-gain-db", type=float, metavar="DB",
                    help="The most gain --live-loudness may apply, in dB, [0, 40] (default 20)")
    ap.add_argument("--pitch-ratio", type=float, metavar="RATIO",
                    help="Multiply every frequency of the speech by RATIO, [0.5, 2], at the same duration, on the GPU.  "
                         "Not in realtime mode")
    ap.add_argument("--tempo", type=float, metavar="RATIO",
                    help="Play the speech RATIO times faster, [0.25, 4], at the same pitch, on the GPU (a waveform time "
                         "stretch: unlike --length-scale it keeps the model's articulation).  Not in realtime mode")
    ap.add_argument("--formant-ratio", type=float, metavar="RATIO",
                    help="Give the speech the voice's own formants (spectral envelope) with every frequency multiplied "
                         "by RATIO, [0.5, 2], on the GPU after --pitch-ratio: 1 with a pitch ratio keeps the speaker's "
                         "timbre, another value without one changes it at the same pitch.  In realtime mode (streaming "
                         "voices only) it holds back 35 - 64 ms more audio")
    ap.add_argument("--encoding", choices=("pcm16",) + ENCODINGS + (FLAC,),
                    help="Output encoding: pcm16 (default), G.711 mulaw / alaw at one byte per sample (telephony: "
                         "PCMU / PCMA), or lossless flac (one FLAC stream per request, on stdout or in the -o file; "
                         "not in realtime mode), encoded on the GPU")
    ap.add_argument("--speaker-blend", metavar="SPEAKER=WEIGHT,...",
                    help="Speak with a blend of a multi-speaker voice's speakers, e.g. \"speaker_3=0.7,speaker_12=0.3\" "
                         "(names or ids; weights >= 0, normalised to sum 1), in place of --speaker-id")
    ap.add_argument("--watermark-key", type=_watermark_key, metavar="KEY",
                    help="Mark all audio with this key's watermark (decimal or 0x-hex, [0, 2^64)), added on the GPU at "
                         "the delivered rate, in every mode; core.watermark_detect finds it")
    ap.add_argument("--watermark-payload", type=int, metavar="N", help="The mark's payload, [0, 4096) (default 0)")
    ap.add_argument("--watermark-strength-db", type=float, metavar="DB",
                    help="The mark's level relative to the local envelope, [-40, -10] dB (default -26)")
    ap.add_argument("--device", type=int, default=int(os.environ.get("SONATA_B200_DEVICE", "0")))
    return ap


def _watermark_key(s: str) -> int:
    return int(s, 16) if s.strip().lower().startswith("0x") else int(s, 10)


def set_watermark_of(model, args) -> None:
    """Mark `model` with the --watermark-* options, if a key is given; a payload or strength without a key is an
    error."""
    if args.watermark_key is None:
        if args.watermark_payload is not None or args.watermark_strength_db is not None:
            raise OperationError("--watermark-payload and --watermark-strength-db need --watermark-key")
        return
    model.set_watermark(args.watermark_key,
                        0 if args.watermark_payload is None else args.watermark_payload,
                        -26.0 if args.watermark_strength_db is None else args.watermark_strength_db)


def process_request(synth: SonataSpeechSynthesizer, default_cfg: PiperSynthesisConfig, req: dict,
                    output_file: Optional[str], out=None) -> None:
    """process_synthesis_request (main.rs:126-165).  `seed` (optional): the request's noise seed, see
    synth.sentence_seed.  `output_rate` (optional): the sample rate of the WAV or raw PCM written.  `loudness`
    (optional): every sentence's target loudness in LUFS; the PCM is then written at the fixed scale.  `pitch_ratio` /
    `tempo` (optional): the ratios every sentence is shifted and played by, in lazy and parallel modes.
    `formant_ratio` (optional): the ratio every sentence's formants are moved by after the pitch stage, in every mode
    (realtime mode carries it as a stream on this library's streaming voices).  `speaker_blend` (optional): an object
    {speaker name or id: weight} (see speaker_blend_of) every sentence speaks with, in every mode.  `live_loudness` /
    `max_gain_db` (optional, realtime mode only): the request's live loudness target in LUFS and the meter's maximum
    gain (see SonataSpeechSynthesizer.synthesize_streamed); the PCM is then written at the fixed scale."""
    out = out or sys.stdout.buffer
    mode = (req.get("mode") or "lazy").lower()
    loudness = req.get("loudness")
    encoding = req.get("encoding")
    if encoding == FLAC:
        if mode == "realtime" and not output_file:
            raise OperationError("FLAC output is not available in realtime mode: a FLAC stream is one whole file whose "
                                 "header holds its length, and realtime mode hands out a sentence's first chunk before "
                                 "its last one is decoded (use lazy or parallel mode)")
    else:
        encoding = None if encoding == "pcm16" else check_encoding(encoding, "request: ")
    if loudness is not None:
        _check_loudness(loudness)
        if mode == "realtime" and not output_file:
            raise OperationError("loudness normalisation is not available in realtime mode: integrated loudness needs "
                                 "the whole sentence, and realtime mode hands out a sentence's first chunk before its "
                                 "last one is decoded (use lazy or parallel mode)")
    live = {k: req[k] for k in ("live_loudness", "max_gain_db") if req.get(k) is not None}
    if live:
        if "live_loudness" not in live:
            raise OperationError("request: a maximum gain is the cap of a live loudness meter: give live_loudness")
        if mode != "realtime" or output_file:
            raise OperationError("live loudness is a realtime mode meter of a stream as it is delivered: for lazy, "
                                 "parallel and file output use loudness (--loudness), which normalises each whole "
                                 "sentence")
        _check_live_loudness(live["live_loudness"], live.get("max_gain_db"), encoding, "request")
        if not isinstance(synth.model, VitsStreamingModel):
            refuse_live_loudness(live["live_loudness"], "realtime mode")
    pros = {k: req[k] for k in ("pitch_ratio", "tempo", "formant_ratio") if req.get(k) is not None}
    blend = speaker_blend_of(req.get("speaker_blend"))
    _check_prosody(pros.get("pitch_ratio"), pros.get("tempo"), pros.get("formant_ratio"))
    if mode == "realtime" and not output_file and not isinstance(synth.model, VitsStreamingModel):
        refuse_formants(pros.get("formant_ratio"), "realtime mode")
        refuse_prosody(pros.get("pitch_ratio"), pros.get("tempo"), "realtime mode")
    synth.model.set_fallback_synthesis_config(PiperSynthesisConfig(
        req.get("speaker_id"),
        req["noise_scale"] if req.get("noise_scale") is not None else default_cfg.noise_scale,
        req["length_scale"] if req.get("length_scale") is not None else default_cfg.length_scale,
        req["noise_w"] if req.get("noise_w") is not None else default_cfg.noise_w))
    oc = AudioOutputConfig(req.get("rate"), req.get("volume"), req.get("pitch"), req.get("appended_silence_ms"))
    text = req["text"]
    seed = req.get("seed")
    rate = {"output_rate": req["output_rate"]} if req.get("output_rate") else {}
    loud = {} if loudness is None else {"loudness": loudness}
    enc = {} if encoding is None else {"encoding": encoding}
    if blend is not None:
        pros["speaker_blend"] = blend
    if output_file:
        synth.synthesize_to_file(output_file, text, oc, seed=seed, **rate, **loud, **enc, **pros)
        return
    if encoding == FLAC:                              # the bytes -o writes, one stream per request
        out.write(synth.synthesize_flac(text, oc, seed=seed, **rate, **loud, **pros))
        out.flush()
        return
    if mode == "lazy":
        stream = synth.synthesize_lazy(text, oc, seed=seed, **rate, **loud, **enc, **pros)
    elif mode == "parallel":
        stream = synth.synthesize_parallel(text, oc, seed=seed, **rate, **loud, **enc, **pros)
    elif mode == "realtime":
        stream = synth.synthesize_streamed(text, oc, req.get("chunk_size") or 100, req.get("chunk_padding") or 3,
                                          seed=seed, **rate, **enc, **pros, **live)
    else:
        raise ValueError(f"unknown synthesis mode `{mode}`")
    for item in stream:
        if encoding is not None:                      # G.711 bytes, one per sample
            out.write(item)
        else:
            samples = item if mode == "realtime" else item.samples
            out.write(samples.as_wave_bytes(fixed_scale=loudness is not None or bool(live)))
        out.flush()


def main(argv=None) -> int:
    args = build_parser().parse_args(argv)
    model = from_config_path(args.config, device=args.device)
    set_watermark_of(model, args)
    synth = SonataSpeechSynthesizer(model)
    default_cfg = model.get_default_synthesis_config()
    if args.input_file:
        with open(args.input_file, encoding="utf-8") as f:
            text = f.read()
        req = {"text": text, "mode": args.mode, "speaker_id": args.speaker_id, "length_scale": args.length_scale,
               "noise_scale": args.noise_scale, "noise_w": args.noise_w, "rate": args.rate, "volume": args.volume,
               "pitch": args.pitch, "appended_silence_ms": args.silence, "chunk_size": args.chunk_size,
               "chunk_padding": args.chunk_padding, "seed": args.seed, "output_rate": args.output_rate,
               "loudness": args.loudness, "encoding": args.encoding, "pitch_ratio": args.pitch_ratio,
               "tempo": args.tempo, "formant_ratio": args.formant_ratio, "speaker_blend": args.speaker_blend,
               "live_loudness": args.live_loudness, "max_gain_db": args.max_gain_db}
        process_request(synth, default_cfg, req, args.output_file)
    else:
        for i, line in enumerate(sys.stdin):
            if not line.strip():
                continue
            req = json.loads(line)
            if req.get("seed") is None:
                req["seed"] = args.seed
            if req.get("output_rate") is None:
                req["output_rate"] = args.output_rate
            if req.get("loudness") is None:
                req["loudness"] = args.loudness
            if req.get("encoding") is None:
                req["encoding"] = args.encoding
            if req.get("pitch_ratio") is None:
                req["pitch_ratio"] = args.pitch_ratio
            if req.get("tempo") is None:
                req["tempo"] = args.tempo
            if req.get("formant_ratio") is None:
                req["formant_ratio"] = args.formant_ratio
            if req.get("speaker_blend") is None:
                req["speaker_blend"] = args.speaker_blend
            if req.get("live_loudness") is None:
                req["live_loudness"] = args.live_loudness
            if req.get("max_gain_db") is None:
                req["max_gain_db"] = args.max_gain_db
            out_file = None
            if args.output_file:
                stem, ext = os.path.splitext(args.output_file)
                out_file = f"{stem}-{i + 1}{ext or '.wav'}"
            process_request(synth, default_cfg, req, out_file)
    model.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
