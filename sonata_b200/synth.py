"""Host-side mirror of `sonata-synth` (crates/sonata/synth/src/lib.rs): the callers of the hot path.

`SonataSpeechSynthesizer` keeps the reference's three scheduling modes (SURVEY §8 row a8):

* `synthesize_lazy`      — one sentence per `next()`                                  (synth :297-307)
* `synthesize_parallel`  — the reference fans sentences out over rayon and collects     (synth :314-325);
                           here the fan-out IS the batch: all sentences go through ONE
                           `speak_batch` pass (the packed-segment kernels), same results.
* `synthesize_streamed`  — realtime mode: per sentence `stream_synthesis(chunk, pad)`
                           with the reference's chunk-size growth rule                  (synth :337-382)

`AudioOutputConfig` (rate / volume / pitch through Sonic, appended silence) is CPU post-processing after
the path (SURVEY §2 row 7, out of scope): appended silence and volume are honoured (pure sample
arithmetic); a non-neutral rate or pitch raises OperationError instead of silently being ignored.
Sonic's percent controls stay out of scope; pitch and tempo exist as ratio controls instead, the
`pitch_ratio=` and `tempo=` keywords of the lazy, parallel and file modes, which run on the GPU
(`VitsModel.infer_batch_with_values`).  How the percent scale would map onto them is undecided.
The model argument is anything with the `SonataModel` surface (`sonata_b200.VitsModel`, or a fake in
the CPU tests) — like the reference's `Arc<dyn SonataModel + Send + Sync>`.
"""
from __future__ import annotations

import queue
import threading
from dataclasses import dataclass
from typing import Iterator, List, Optional

import numpy as np

from .core import (FLAC, G711_SILENCE, Audio, AudioSamples, OperationError, SonataError, check_encoding, flac_encode,
                   g711_wave_bytes, refuse_flac)

RATE_RANGE = (0.5, 5.5)      # synth/src/lib.rs:13
VOLUME_RANGE = (0.0, 1.0)    # :14
PITCH_RANGE = (0.5, 1.5)     # :15


def percent_to_param(value: int, lo: float, hi: float) -> float:
    """synth/src/utils.rs:6-8 — linear over the range (rate=50 means 3.0x, not 1.0x)."""
    return (value / 100.0) * (hi - lo) + lo


def param_to_percent(value: float, lo: float, hi: float) -> int:
    return int(round((value - lo) / (hi - lo) * 100.0))


@dataclass
class AudioOutputConfig:
    """synth/src/lib.rs:28-34"""
    rate: Optional[int] = None
    volume: Optional[int] = None
    pitch: Optional[int] = None
    appended_silence_ms: Optional[int] = None

    def _check_supported(self):
        if self.rate is not None and abs(percent_to_param(self.rate, *RATE_RANGE) - 1.0) > 1e-6:
            raise OperationError("Sonic Error: time-scale modification (rate) is CPU post-processing outside "
                                 "sonata_b200; use length_scale or rate=10 (1.0x)")
        if self.pitch is not None and abs(percent_to_param(self.pitch, *PITCH_RANGE) - 1.0) > 1e-6:
            raise OperationError("Sonic Error: pitch modification is CPU post-processing outside sonata_b200; "
                                 "use pitch=50 (1.0x)")

    def apply_to_raw_samples(self, samples: AudioSamples) -> AudioSamples:
        self._check_supported()
        v = samples.as_slice()
        if self.volume is not None:
            v = v * np.float32(percent_to_param(self.volume, *VOLUME_RANGE))
        return AudioSamples(v)

    def generate_silence(self, time_ms: int, sample_rate: int) -> AudioSamples:
        return AudioSamples(np.zeros((time_ms * sample_rate) // 1000, dtype=np.float32))   # :107-116

    def gain(self) -> Optional[float]:
        """The linear gain of `volume`, or None without one."""
        return None if self.volume is None else percent_to_param(self.volume, *VOLUME_RANGE)

    def silence_bytes(self, sample_rate: int, encoding: str) -> bytes:
        """The appended silence in G.711: the code of sample 0 (0xFF mu-law, 0xD5 A-law) per sample."""
        n = (self.appended_silence_ms * sample_rate) // 1000 if self.appended_silence_ms else 0
        return bytes([G711_SILENCE[encoding]]) * n

    def apply(self, audio: Audio) -> Audio:
        """synth/src/lib.rs:37-54: silence is appended first, then the whole buffer is processed."""
        s = audio.samples
        if self.appended_silence_ms is not None:
            s = AudioSamples(np.concatenate([s.as_slice(), self.generate_silence(self.appended_silence_ms,
                                                                                  audio.info.sample_rate).as_slice()]))
        return Audio(self.apply_to_raw_samples(s), audio.info.sample_rate, audio.inference_ms)


def next_chunk_size(chunk_size: int, produced: int) -> int:
    """The realtime mode's chunk-size growth rule (synth/src/lib.rs:348-356): before every sentence after the first,
    the chunk size is multiplied by the number of chunks produced so far (chunk_factor = 1)."""
    return chunk_size * 1 * produced if produced != 0 else chunk_size


def sentence_seed(seed: Optional[int], i: int) -> Optional[int]:
    """The noise seed of sentence i of a request seeded with `seed`: (seed + i) mod 2**64, so every sentence has its
    own noise and a request's audio depends on its seed alone.  None (an unseeded request) stays None.  Raises
    OperationError when `seed` is not an int in [0, 2**64)."""
    from .piper import _seed_arrays
    _seed_arrays([seed], 1)
    return None if seed is None else (int(seed) + i) % 2**64


def _check_output_rate(rate) -> None:
    """Raises OperationError unless `rate` is None, 0 or one of piper.OUTPUT_RATES."""
    from .piper import _rate_array
    _rate_array([rate], 1)


def _check_loudness(target) -> None:
    """Raises OperationError unless `target` is None or a loudness target in LUFS, finite and in [-70, 0]."""
    from .piper import _loudness_array
    _loudness_array([target], 1)


def _check_prosody(pitch_ratio, tempo, formant_ratio=None) -> None:
    """Raises OperationError unless each is None or a ratio in piper.PITCH_RANGE / piper.TEMPO_RANGE /
    piper.FORMANT_RANGE."""
    from .piper import _formant_array, _prosody_arrays
    _prosody_arrays([pitch_ratio], [tempo], 1)
    _formant_array([formant_ratio], 1)


def _prosody_extra(n: int, pitch_ratio, tempo, formant_ratio=None) -> dict:
    """The per-utterance keywords of n sentences that share a request's pitch ratio, tempo and formant ratio ({}
    without any)."""
    from .piper import _formant_array, _prosody_arrays
    p, t = _prosody_arrays([pitch_ratio], [tempo], 1)
    out = {} if p is None else {"pitches": [pitch_ratio] * n}
    if t is not None:
        out["tempos"] = [tempo] * n
    if _formant_array([formant_ratio], 1) is not None:
        out["formants"] = [formant_ratio] * n
    return out


def _blend_extra(model, n: int, speaker_blend, where: str) -> dict:
    """The per-utterance keywords of n sentences that share a request's speaker blend ({} without one), checked first:
    an OperationError names `where`."""
    if speaker_blend is None:
        return {}
    from .piper import _blend_arrays
    _blend_arrays(model, [speaker_blend], 1, [where])
    return {"speaker_blends": [speaker_blend] * n}


def _stream_prosody_extra(model, pitch_ratio, tempo, where: str, formant_ratio=None) -> dict:
    """The stream_synthesis keywords of a streaming request's ratios ({} without any).  A model that is not one of
    this library's streaming voices cannot warp a stream on the device and refuses by name (piper.refuse_prosody,
    piper.refuse_formants)."""
    from .piper import VitsStreamingModel, _prosody_arrays, _stream_formant, refuse_formants, refuse_prosody
    if not isinstance(model, VitsStreamingModel):
        refuse_formants(formant_ratio, where)
        refuse_prosody(pitch_ratio, tempo, where)
    p, t = _prosody_arrays([pitch_ratio], [tempo], 1)
    out = {} if p is None else {"pitch": pitch_ratio}
    if t is not None:
        out["tempo"] = tempo
    phi = _stream_formant(formant_ratio, "request")
    if phi is not None:
        out["formant_ratio"] = phi
    return out


def _request_meter(model, live_loudness, max_gain_db, output_rate, encoding, where: str, who: str):
    """The live loudness meter of a streaming request (None without a target): one piper.LoudnessStream at the
    request's output rate, carried across its sentences.  Models that are not this library's streaming voices refuse
    it by name."""
    from .piper import LoudnessStream, VitsStreamingModel, _check_live_loudness, refuse_live_loudness
    if not isinstance(model, VitsStreamingModel):
        refuse_live_loudness(live_loudness, where)
    _check_live_loudness(live_loudness, max_gain_db, encoding, who)
    if live_loudness is None:
        return None
    if isinstance(live_loudness, LoudnessStream):
        raise OperationError(f"{who}: a request makes its own meter: give live_loudness as a target in LUFS")
    return LoudnessStream(model, live_loudness, 20.0 if max_gain_db is None else max_gain_db, output_rate or None, who)


def _device_g711(model) -> bool:
    """Whether `model` encodes G.711 on the device (VitsModel / VitsStreamingModel).  Other SonataModels (fakes in
    tests) get the host definition, AudioSamples.as_g711_bytes, of the audio they return."""
    return hasattr(model, "speak_batch_g711")


def _sentences(model, text: str) -> List[str]:
    """SpeechSynthesisTaskProvider::get_phonemes (:256-258), or newline-separated phoneme sentences when the model has
    no phonemizer."""
    try:
        return model.phonemize_text(text).to_vec()
    except SonataError:
        return [s for s in text.split("\n") if s.strip()]


class SonataSpeechSynthesizer:
    """synth/src/lib.rs:119-203.  `text` is a phoneme string; sentences are separated by newlines when the
    model has no phonemizer (the espeak-ng front-end is outside this repo)."""

    def __init__(self, model):
        self.model = model

    def _phonemes(self, text: str) -> List[str]:
        return _sentences(self.model, text)

    def _process(self, audio: Audio, cfg: Optional[AudioOutputConfig]) -> Audio:
        return cfg.apply(audio) if cfg is not None else audio

    # `seed` (every mode): the request's noise seed, sentence i seeded with sentence_seed(seed, i); None keeps the
    # positional noise.  `output_rate` (every mode): the sample rate of the audio handed out, one of
    # piper.OUTPUT_RATES (None / 0: the voice's), each sentence resampled on the device; appended silence is generated
    # at that rate.  `loudness` (lazy, parallel and file modes): a target integrated loudness in LUFS, [-70, 0], each
    # sentence measured and scaled to it on the device before the output config's volume and silence apply.
    # `encoding` (every mode): "mulaw" / "alaw" hands out G.711 `bytes` instead of Audio / AudioSamples: G.711 of the
    # 16-bit samples of what the mode hands out without it (to_i16_vec per sentence or chunk, or the fixed scale with a
    # loudness target), the output config's volume applied on the device as a gain before the conversion and its
    # silence appended as code-of-zero bytes.  `pitch_ratio` / `tempo` (lazy, parallel and file modes): each sentence's
    # frequencies multiplied by the ratio at the same duration / played that many times faster at the same pitch, on
    # the device before any resampling and loudness (piper.PITCH_RANGE, piper.TEMPO_RANGE).  `formant_ratio` (lazy,
    # parallel and file modes): each sentence's spectral envelope moved by the ratio after the pitch stage; 1.0 with a
    # pitch ratio keeps the voice's own formants (piper.FORMANT_RANGE).  The streamed modes carry it as a stream on
    # this library's streaming voices and refuse it by name on other models.
    # `speaker_blend` (every mode): a mapping {speaker: weight} of a multi-speaker voice that every sentence speaks with
    # in place of the fallback config's speaker (see piper.VitsModel.infer_batch_with_values); checked before any
    # synthesis.

    def _g711_batch(self, phs: List[str], encoding: str, seeds, output_rate, loudness,
                    cfg: Optional[AudioOutputConfig], pitch_ratio=None, tempo=None,
                    formant_ratio=None, speaker_blend=None) -> List[bytes]:
        """The G.711 bytes of sentences `phs`, one synthesis pass, each followed by its appended silence."""
        if cfg is not None:
            cfg._check_supported()
        n = len(phs)
        extra = {} if seeds is None else {"seeds": seeds}
        if output_rate:
            extra["output_rates"] = [output_rate] * n
        if loudness is not None:
            extra["loudness"] = [loudness] * n
        extra.update(_prosody_extra(n, pitch_ratio, tempo, formant_ratio))
        extra.update(_blend_extra(self.model, n, speaker_blend, "request"))
        if not _device_g711(self.model):
            res = self.model.speak_batch(phs, **extra) if extra else self.model.speak_batch(phs)
            return [self._process(a, cfg).samples.as_g711_bytes(encoding, fixed_scale=loudness is not None)
                    for a in res]
        g = cfg.gain() if cfg is not None else None
        if g is not None:
            extra["gains"] = [g] * n
        res = self.model.speak_batch_g711(phs, encoding, **extra)
        if cfg is None:
            return res
        rate = output_rate or self.model.audio_output_info().sample_rate
        return [r + cfg.silence_bytes(rate, encoding) for r in res]

    def synthesize_lazy(self, text: str, output_config: Optional[AudioOutputConfig] = None,
                        seed: Optional[int] = None, output_rate: Optional[int] = None,
                        loudness: Optional[float] = None, encoding: Optional[str] = None,
                        pitch_ratio: Optional[float] = None, tempo: Optional[float] = None,
                        formant_ratio: Optional[float] = None, speaker_blend=None) -> Iterator[Audio]:
        sentence_seed(seed, 0)
        _check_output_rate(output_rate)
        _check_loudness(loudness)
        _check_prosody(pitch_ratio, tempo, formant_ratio)
        refuse_flac(encoding, "synthesize_lazy")
        check_encoding(encoding)
        pros = _prosody_extra(1, pitch_ratio, tempo, formant_ratio)
        pros.update(_blend_extra(self.model, 1, speaker_blend, "request"))
        for i, ph in enumerate(self._phonemes(text)):
            if encoding is not None:
                yield self._g711_batch([ph], encoding, None if seed is None else [sentence_seed(seed, i)], output_rate,
                                       loudness, output_config, pitch_ratio, tempo, formant_ratio, speaker_blend)[0]
                continue
            if output_rate or loudness is not None or pros:
                extra = dict(pros) if seed is None else dict(pros, seeds=[sentence_seed(seed, i)])
                if output_rate:
                    extra["output_rates"] = [output_rate]
                if loudness is not None:
                    extra["loudness"] = [loudness]
                a = self.model.speak_batch([ph], **extra)[0]
            else:
                a = (self.model.speak_one_sentence(ph) if seed is None
                     else self.model.speak_batch([ph], seeds=[sentence_seed(seed, i)])[0])
            yield self._process(a, output_config)

    def synthesize_parallel(self, text: str, output_config: Optional[AudioOutputConfig] = None,
                            seed: Optional[int] = None, output_rate: Optional[int] = None,
                            loudness: Optional[float] = None, encoding: Optional[str] = None,
                            pitch_ratio: Optional[float] = None, tempo: Optional[float] = None,
                            formant_ratio: Optional[float] = None, speaker_blend=None) -> Iterator[Audio]:
        sentence_seed(seed, 0)
        _check_output_rate(output_rate)
        _check_loudness(loudness)
        _check_prosody(pitch_ratio, tempo, formant_ratio)
        refuse_flac(encoding, "synthesize_parallel")
        check_encoding(encoding)
        _blend_extra(self.model, 1, speaker_blend, "request")
        ph = self._phonemes(text)
        if encoding is not None:
            seeds = None if seed is None else [sentence_seed(seed, i) for i in range(len(ph))]
            return iter(self._g711_batch(ph, encoding, seeds, output_rate, loudness, output_config, pitch_ratio, tempo,
                                         formant_ratio, speaker_blend) if ph else [])
        extra = {"output_rates": [output_rate] * len(ph)} if output_rate else {}
        extra.update(_prosody_extra(len(ph), pitch_ratio, tempo, formant_ratio))
        extra.update(_blend_extra(self.model, len(ph), speaker_blend, "request"))
        if loudness is not None:
            extra["loudness"] = [loudness] * len(ph)
        if not ph:
            results = []
        elif seed is None:
            results = self.model.speak_batch(ph, **extra)         # one batched pass == the rayon fan-out + collect
        else:
            results = self.model.speak_batch(ph, seeds=[sentence_seed(seed, i) for i in range(len(ph))], **extra)
        return iter([self._process(a, output_config) for a in results])

    def synthesize_streamed(self, text: str, output_config: Optional[AudioOutputConfig] = None,
                            chunk_size: int = 72, chunk_padding: int = 3,
                            seed: Optional[int] = None, output_rate: Optional[int] = None,
                            encoding: Optional[str] = None, pitch_ratio: Optional[float] = None,
                            tempo: Optional[float] = None, formant_ratio: Optional[float] = None,
                            speaker_blend=None, live_loudness: Optional[float] = None,
                            max_gain_db: Optional[float] = None) -> Iterator[AudioSamples]:
        """RealtimeSpeechStream (:337-382): a background producer pushes chunks into an unbounded channel;
        chunk_size is multiplied by the number of chunks already produced for every following sentence.
        `output_rate`: each sentence is resampled as its own stream (zero history at its start, flushed at its end).
        `encoding`: every chunk is G.711 bytes of its to_i16_vec after the volume, encoded on the device.
        `pitch_ratio` / `tempo`: every sentence warped as its own stream on the device (a fresh piper.ProsodyStream,
        flushed at its end); appended silence is not warped.  `formant_ratio`: every sentence's formant stage carried
        as its own stream on the device, with or without the ratios (see stream_synthesis).  `live_loudness`: a target
        in LUFS that one live loudness meter (piper.LoudnessStream, capped at `max_gain_db`, default 20) holds the
        request to, carried across its sentences; appended silence is not metered, and the volume applies after the
        meter (G.711 is then taken at the fixed scale)."""
        pros = _stream_prosody_extra(self.model, pitch_ratio, tempo, "synthesize_streamed", formant_ratio)
        refuse_flac(encoding, "synthesize_streamed")
        meter = _request_meter(self.model, live_loudness, max_gain_db, output_rate, encoding, "synthesize_streamed",
                               "request")
        sentence_seed(seed, 0)
        _check_output_rate(output_rate)
        check_encoding(encoding)
        if encoding is not None and output_config is not None:
            output_config._check_supported()
        sr = output_rate or self.model.audio_output_info().sample_rate
        rate = {"output_rate": output_rate} if output_rate else {}
        device = encoding is not None and _device_g711(self.model)
        if device:
            rate["encoding"] = encoding
            if output_config is not None and output_config.gain() is not None:
                rate["gain"] = output_config.gain()
        rate.update(pros)
        if _blend_extra(self.model, 1, speaker_blend, "request"):
            rate["speaker_blend"] = speaker_blend
        if meter is not None:
            rate["live_loudness"] = meter
        extra = lambda i: dict(rate) if seed is None else dict(rate, seed=sentence_seed(seed, i))

        def emit(chunk):
            if encoding is None:
                return output_config.apply_to_raw_samples(chunk) if output_config else chunk
            if device:
                return chunk
            return (output_config.apply_to_raw_samples(chunk) if output_config else chunk).as_g711_bytes(encoding)
        q: "queue.Queue" = queue.Queue()
        done = object()

        def producer():
            cs, produced = chunk_size, 0
            try:
                for i, ph in enumerate(self._phonemes(text)):
                    cs = next_chunk_size(cs, produced)
                    n = 0
                    for chunk in self.model.stream_synthesis(ph, cs, chunk_padding, **extra(i)):
                        q.put(emit(chunk))
                        n += 1
                    produced += n
                    if output_config and output_config.appended_silence_ms:
                        q.put(output_config.generate_silence(output_config.appended_silence_ms, sr) if encoding is None
                              else output_config.silence_bytes(sr, encoding))
            except Exception as e:                                  # errors travel through the channel (:368-371)
                q.put(e)
            q.put(done)

        threading.Thread(target=producer, daemon=True).start()
        while True:
            item = q.get()
            if item is done:
                return
            if isinstance(item, Exception):
                raise item
            yield item

    def synthesize_to_file(self, filename, text: str, output_config: Optional[AudioOutputConfig] = None,
                           seed: Optional[int] = None, output_rate: Optional[int] = None,
                           loudness: Optional[float] = None, encoding: Optional[str] = None,
                           pitch_ratio: Optional[float] = None, tempo: Optional[float] = None,
                           formant_ratio: Optional[float] = None, speaker_blend=None) -> None:
        """:168-198 — parallel mode, concatenated, peak-normalised i16 WAV (at output_rate when given).  With
        `loudness` the WAV is written at the fixed scale (trunc(clamp(x * 32767))), so it keeps the sentences' level.
        With `encoding` the WAV is 8-bit G.711 (WAVE_FORMAT_MULAW / _ALAW, with a `fact` chunk) holding the sentences'
        bytes as synthesize_parallel hands them out: each sentence converted at its own peak (or the fixed scale).
        With encoding="flac" the file is one FLAC stream (synthesize_flac) instead of a WAV."""
        if isinstance(encoding, str) and encoding == FLAC:
            data = self.synthesize_flac(text, output_config, seed=seed, output_rate=output_rate, loudness=loudness,
                                        pitch_ratio=pitch_ratio, tempo=tempo, formant_ratio=formant_ratio,
                                        speaker_blend=speaker_blend)
            with open(filename, "wb") as f:
                f.write(data)
            return
        extra = {"output_rate": output_rate} if output_rate else {}
        if loudness is not None:
            extra["loudness"] = loudness
        if pitch_ratio is not None:
            extra["pitch_ratio"] = pitch_ratio
        if tempo is not None:
            extra["tempo"] = tempo
        if formant_ratio is not None:
            extra["formant_ratio"] = formant_ratio
        if speaker_blend is not None:
            extra["speaker_blend"] = speaker_blend
        if check_encoding(encoding) is not None:
            data = b"".join(self.synthesize_parallel(text, output_config, seed=seed, encoding=encoding, **extra))
            if not data:
                raise OperationError("No speech data to write")
            with open(filename, "wb") as f:
                f.write(g711_wave_bytes(data, encoding, output_rate or self.model.audio_output_info().sample_rate))
            return
        self._document(text, output_config, seed, output_rate, loudness, pitch_ratio, tempo, formant_ratio,
                       speaker_blend).save_to_file(filename, fixed_scale=loudness is not None)

    def _document(self, text: str, output_config: Optional[AudioOutputConfig], seed, output_rate, loudness,
                  pitch_ratio=None, tempo=None, formant_ratio=None, speaker_blend=None) -> Audio:
        """The sentences of synthesize_parallel concatenated: what synthesize_to_file writes as a WAV."""
        extra = {"output_rate": output_rate} if output_rate else {}
        if loudness is not None:
            extra["loudness"] = loudness
        if pitch_ratio is not None:
            extra["pitch_ratio"] = pitch_ratio
        if tempo is not None:
            extra["tempo"] = tempo
        if formant_ratio is not None:
            extra["formant_ratio"] = formant_ratio
        if speaker_blend is not None:
            extra["speaker_blend"] = speaker_blend
        parts = [a.samples.as_slice() for a in self.synthesize_parallel(text, output_config, seed=seed, **extra)]
        if not parts or sum(len(p) for p in parts) == 0:
            raise OperationError("No speech data to write")
        rate = output_rate or self.model.audio_output_info().sample_rate
        return Audio(AudioSamples(np.concatenate(parts)), rate)

    def synthesize_flac(self, text: str, output_config: Optional[AudioOutputConfig] = None,
                        seed: Optional[int] = None, output_rate: Optional[int] = None,
                        loudness: Optional[float] = None, pitch_ratio: Optional[float] = None,
                        tempo: Optional[float] = None, formant_ratio: Optional[float] = None,
                        speaker_blend=None) -> bytes:
        """The FLAC file synthesize_to_file(..., encoding="flac") writes: one stream whose decoded samples are exactly
        the 16-bit samples of the WAV the same call writes without an encoding (the concatenation at the document's
        peak, or the fixed scale with `loudness`), encoded on the model's device by flac_encode."""
        doc = self._document(text, output_config, seed, output_rate, loudness, pitch_ratio, tempo, formant_ratio,
                             speaker_blend)
        s = doc.samples
        return flac_encode(s.to_i16_fixed() if loudness is not None else s.to_i16_vec(), doc.info.sample_rate,
                           getattr(self.model, "device", 0))

    # passthroughs of the SonataModel surface (:205-253)
    def speak_one_sentence(self, phonemes: str) -> Audio:
        return self.model.speak_one_sentence(phonemes)

    def speak_batch(self, phoneme_batches) -> List[Audio]:
        return self.model.speak_batch(phoneme_batches)

    def audio_output_info(self):
        return self.model.audio_output_info()


class _Request:
    def __init__(self, key, ids, output_config, config, chunk_size, seed=None, output_rate=None, encoding=None):
        self.key, self.ids, self.output_config, self.config, self.seed = key, ids, output_config, config, seed
        self.output_rate, self.encoding = output_rate, encoding
        self.cs, self.produced, self.n, self.next = chunk_size, 0, 0, 0


class RealtimeBatch:
    """Many realtime requests of one or more sentences served together: `synthesize_streamed` for K clients, with every
    step of every client in one encoder pass (sentences that start) and one decoder pass (the next chunk of each).

    `add(text, output_config, config)` admits a request (config: its PiperSynthesisConfig, None for the fallback);
    `step()` returns [(key, AudioSamples)].  A request's items are exactly what
    `synthesize_streamed(text, output_config, chunk_size, chunk_padding)` yields with `config` as the fallback: the
    chunk-size growth rule across its sentences, volume on every chunk and the appended silence after each sentence.
    Each sentence's ids are mapped and the config's speaker checked at `add`, so a bad request raises there; a request
    whose synthesis fails later gets its SonataError as its last item, (key, error), and the others carry on."""

    def __init__(self, model, chunk_size: int = 72, chunk_padding: int = 3):
        from .piper import StreamBatch
        self.model = model
        self.chunk_size = chunk_size
        self._streams = StreamBatch(model, chunk_size, chunk_padding)
        self._sr = model.audio_output_info().sample_rate
        self._by_stream = {}          # stream key -> request of the sentence it speaks
        self._next_key = 0

    def add(self, text: str, output_config: Optional[AudioOutputConfig] = None, config=None,
            seed: Optional[int] = None, output_rate: Optional[int] = None, encoding: Optional[str] = None,
            pitch_ratio: Optional[float] = None, tempo: Optional[float] = None,
            formant_ratio: Optional[float] = None, speaker_blend=None, live_loudness: Optional[float] = None,
            max_gain_db: Optional[float] = None) -> int:
        """`seed`: the request's noise seed, `output_rate` its sample rate and `encoding` its G.711 encoding, as for
        synthesize_streamed, and `pitch_ratio` / `tempo` its ratios, each sentence warped as its own stream, as there.
        `formant_ratio` its formant ratio, as there.  `speaker_blend`: the request's speaker blend, as for
        synthesize_streamed; it replaces the config's speaker and is checked here, naming the request.
        `live_loudness` / `max_gain_db`: the request's live loudness, one meter across its sentences, as there."""
        from .piper import PiperSynthesisConfig
        pros = _stream_prosody_extra(self.model, pitch_ratio, tempo, "RealtimeBatch", formant_ratio)
        refuse_flac(encoding, "RealtimeBatch")
        sentence_seed(seed, 0)
        _check_output_rate(output_rate)
        check_encoding(encoding)
        if output_config is not None:
            output_config._check_supported()
        if config is not None and not isinstance(config, PiperSynthesisConfig):
            raise OperationError("Invalid configuration for Vits Model")
        if config is not None and config.speaker is not None and config.speaker not in (self.model.get_speakers() or {}):
            raise OperationError(f"No speaker was found with the given id `{config.speaker}`")
        _blend_extra(self.model, 1, speaker_blend, f"request {self._next_key}")
        ids = [self.model.phonemes_to_input_ids(ph) for ph in _sentences(self.model, text)]
        if any(len(i) == 0 for i in ids):
            raise OperationError("Failed to run model inference. Error: empty input sequence")
        req = _Request(self._next_key, ids, output_config, config, self.chunk_size, seed, output_rate or None, encoding)
        req.prosody, req.blend = pros, speaker_blend
        req.meter = _request_meter(self.model, live_loudness, max_gain_db, output_rate, encoding, "RealtimeBatch",
                                   f"request {req.key}")
        self._next_key += 1
        self._start_sentence(req)
        return req.key

    def _start_sentence(self, req: _Request) -> None:
        if req.next == len(req.ids):
            return
        req.cs = next_chunk_size(req.cs, req.produced)
        req.n = 0
        # the volume of an encoded request is a gain before its encoding; otherwise it applies to the chunks here
        gain = req.output_config.gain() if req.encoding is not None and req.output_config is not None else None
        key = self._streams._add(req.ids[req.next], req.config, req.cs, sentence_seed(req.seed, req.next),
                                 req.output_rate, req.encoding, gain, speaker_blend=req.blend,
                                 live_loudness=req.meter, **req.prosody)
        self._by_stream[key] = req
        req.next += 1

    def __len__(self) -> int:
        """Requests added and not yet finished."""
        return len(self._by_stream)

    def step(self) -> List[tuple]:
        out = []
        for skey, chunk in self._streams.step():
            req = self._by_stream[skey]
            if isinstance(chunk, SonataError):          # the request ends with its error, as synthesize_streamed's
                del self._by_stream[skey]               # channel delivers it (:368-371); the others carry on
                out.append((req.key, chunk))
                continue
            oc = req.output_config
            out.append((req.key, chunk if req.encoding is not None or not oc else oc.apply_to_raw_samples(chunk)))
            req.n += 1
            if skey in self._streams:
                continue
            del self._by_stream[skey]                  # the sentence is done
            req.produced += req.n
            if oc and oc.appended_silence_ms:
                sr = req.output_rate or self._sr
                out.append((req.key, oc.generate_silence(oc.appended_silence_ms, sr) if req.encoding is None
                            else oc.silence_bytes(sr, req.encoding)))
            self._start_sentence(req)
        return out
