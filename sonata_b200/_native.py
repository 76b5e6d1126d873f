"""ctypes binding of libsonata_b200.so (the C ABI in include/sonata_b200.h).

This is the Python analogue of the `extern "C"` block a Rust `impl SonataModel` would carry
(INTEGRATION.md shows that stub).  There is deliberately NO fallback: if the CUDA library is
missing or no GPU is visible, loading a voice fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SB200_LIB") or os.path.join(_HERE, "lib", "libsonata_b200.so")   # SB200_LIB: A/B builds


class sb200_error(C.Structure):
    _fields_ = [("code", C.c_int32), ("message", C.c_void_p)]


class sb200_audio(C.Structure):
    _fields_ = [("data", C.POINTER(C.c_float)), ("len", C.c_size_t), ("inference_ms", C.c_float),
                ("sample_rate", C.c_uint32)]


class sb200_synth_config(C.Structure):
    _fields_ = [("speaker", C.c_int64), ("has_speaker", C.c_int32), ("noise_scale", C.c_float),
                ("length_scale", C.c_float), ("noise_w", C.c_float)]


class sb200_audio_info(C.Structure):
    _fields_ = [("sample_rate", C.c_uint32), ("num_channels", C.c_uint32), ("sample_width", C.c_uint32)]


class sb200_region_stat(C.Structure):
    _fields_ = [("name", C.c_char * 32), ("ms", C.c_double), ("flops", C.c_double), ("bytes", C.c_double),
                ("launches", C.c_int32)]


class sb200_chunk_capture(C.Structure):
    _fields_ = [("name", C.c_char * 32), ("chunk", C.c_size_t), ("rows", C.c_size_t), ("cols", C.c_size_t),
                ("data", C.POINTER(C.c_float))]


_P = C.c_void_p
_ERR = C.POINTER(sb200_error)

# name -> (restype, argtypes); this table is also what tests/test_abi.py checks against the header
SIGNATURES = {
    "sb200_version": (C.c_char_p, []),
    "sb200_string_free": (None, [C.c_void_p]),
    "sb200_audio_free": (None, [C.POINTER(sb200_audio)]),
    "sb200_device_count": (C.c_int32, []),
    "sb200_voice_load": (C.c_int32, [C.c_char_p, C.c_int32, C.POINTER(_P), _ERR]),
    "sb200_voice_free": (None, [_P]),
    "sb200_audio_output_info": (C.c_int32, [_P, C.POINTER(sb200_audio_info), _ERR]),
    "sb200_get_default_synthesis_config": (C.c_int32, [_P, C.POINTER(sb200_synth_config), _ERR]),
    "sb200_get_fallback_synthesis_config": (C.c_int32, [_P, C.POINTER(sb200_synth_config), _ERR]),
    "sb200_set_fallback_synthesis_config": (C.c_int32, [_P, C.POINTER(sb200_synth_config), _ERR]),
    "sb200_get_language": (C.c_int32, [_P, C.POINTER(C.c_void_p), _ERR]),
    "sb200_get_quality": (C.c_int32, [_P, C.POINTER(C.c_void_p), _ERR]),
    "sb200_supports_streaming_output": (C.c_int32, [_P]),
    "sb200_num_speakers": (C.c_int32, [_P]),
    "sb200_speaker_name_to_id": (C.c_int64, [_P, C.c_char_p]),
    "sb200_phonemes_to_input_ids": (C.c_int32, [_P, C.c_char_p, C.POINTER(C.POINTER(C.c_int64)),
                                                C.POINTER(C.c_size_t), _ERR]),
    "sb200_ids_free": (None, [C.POINTER(C.c_int64)]),
    "sb200_phonemes_to_input_ids_map": (C.c_int32, [_P, C.c_char_p, C.POINTER(C.POINTER(C.c_int64)),
                                                    C.POINTER(C.POINTER(C.c_int64)), C.POINTER(C.c_size_t), _ERR]),
    "sb200_speak_one_sentence": (C.c_int32, [_P, C.c_char_p, C.POINTER(sb200_audio), _ERR]),
    "sb200_speak_batch": (C.c_int32, [_P, C.POINTER(C.c_char_p), C.c_size_t, C.POINTER(sb200_audio), _ERR]),
    "sb200_speak_ids": (C.c_int32, [_P, C.POINTER(C.c_int64), C.c_size_t, C.POINTER(sb200_audio), _ERR]),
    "sb200_speak_batch_ids": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.c_size_t,
                                          C.POINTER(sb200_audio), _ERR]),
    "sb200_speak_batch_ids_configs": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.c_size_t,
                                                  C.POINTER(sb200_synth_config), C.POINTER(sb200_audio), _ERR]),
    "sb200_speak_batch_ids_durations": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.c_size_t,
                                                    C.POINTER(sb200_synth_config), C.POINTER(C.c_float),
                                                    C.POINTER(C.c_int32), C.POINTER(sb200_audio), C.POINTER(C.c_int32),
                                                    _ERR]),
    "sb200_speak_batch_ids_seeded": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.c_size_t,
                                                 C.POINTER(sb200_synth_config), C.POINTER(C.c_float),
                                                 C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.POINTER(C.c_int32),
                                                 C.POINTER(sb200_audio), C.POINTER(C.c_int32), _ERR]),
    "sb200_speak_batch_ids_rates": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.c_size_t,
                                                C.POINTER(sb200_synth_config), C.POINTER(C.c_float),
                                                C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.POINTER(C.c_int32),
                                                C.POINTER(C.c_uint32), C.POINTER(sb200_audio), C.POINTER(C.c_int32),
                                                _ERR]),
    "sb200_speak_batch_ids_loudness": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.c_size_t,
                                                   C.POINTER(sb200_synth_config), C.POINTER(C.c_float),
                                                   C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.POINTER(C.c_int32),
                                                   C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(sb200_audio),
                                                   C.POINTER(C.c_int32), C.POINTER(C.c_double), C.POINTER(C.c_float),
                                                   _ERR]),
    "sb200_speak_batch_ids_prosody": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.c_size_t,
                                                  C.POINTER(sb200_synth_config), C.POINTER(C.c_float),
                                                  C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.POINTER(C.c_int32),
                                                  C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                                  C.POINTER(C.c_float), C.POINTER(sb200_audio), C.POINTER(C.c_int32),
                                                  C.POINTER(C.c_double), C.POINTER(C.c_float), _ERR]),
    "sb200_speak_batch_ids_contour": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.c_size_t,
                                                  C.POINTER(sb200_synth_config), C.POINTER(C.c_float),
                                                  C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.POINTER(C.c_int32),
                                                  C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                                  C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(sb200_audio),
                                                  C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_double),
                                                  C.POINTER(C.c_float), _ERR]),
    "sb200_speak_batch_ids_formants": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.c_size_t,
                                                   C.POINTER(sb200_synth_config), C.POINTER(C.c_float),
                                                   C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.POINTER(C.c_int32),
                                                   C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                                   C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                                   C.POINTER(sb200_audio), C.POINTER(C.c_int32), C.POINTER(C.c_int64),
                                                   C.POINTER(C.c_double), C.POINTER(C.c_float), _ERR]),
    "sb200_job_set_formants": (C.c_int32, [_P, C.POINTER(C.c_float), _ERR]),
    "sb200_speak_batch_ids_blends": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.c_size_t,
                                                 C.POINTER(sb200_synth_config), C.POINTER(C.c_float),
                                                 C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.POINTER(C.c_int32),
                                                 C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                                 C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                                 C.POINTER(C.c_int64), C.POINTER(C.c_float), C.POINTER(C.c_size_t),
                                                 C.POINTER(sb200_audio), C.POINTER(C.c_int32), C.POINTER(C.c_int64),
                                                 C.POINTER(C.c_double), C.POINTER(C.c_float), _ERR]),
    "sb200_job_set_speaker_blends": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_float),
                                                 C.POINTER(C.c_size_t), _ERR]),
    "sb200_debug_speaker_blend": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_float), C.c_size_t,
                                              C.POINTER(C.c_float), C.c_size_t, C.POINTER(C.c_float), C.c_size_t,
                                              _ERR]),
    "sb200_debug_formant": (C.c_int32, [C.c_int32, C.POINTER(C.c_float), C.c_size_t, C.c_int32, C.c_float, C.c_float,
                                        C.POINTER(C.c_int64), C.POINTER(C.c_float), C.c_size_t, C.c_float,
                                        C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_size_t, C.POINTER(C.c_int64),
                                        _ERR]),
    "sb200_job_create": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.c_size_t,
                                     C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.POINTER(C.c_float)),
                                     C.POINTER(C.c_size_t), C.POINTER(_P), _ERR]),
    "sb200_job_set_debug": (C.c_int32, [_P, C.c_int32]),
    "sb200_job_set_configs": (C.c_int32, [_P, C.POINTER(sb200_synth_config), _ERR]),
    "sb200_job_set_durations": (C.c_int32, [_P, C.POINTER(C.c_float), C.POINTER(C.c_int32), _ERR]),
    "sb200_job_set_seeds": (C.c_int32, [_P, C.POINTER(C.c_uint64), C.POINTER(C.c_int32), _ERR]),
    "sb200_job_set_output_rates": (C.c_int32, [_P, C.POINTER(C.c_uint32), _ERR]),
    "sb200_job_set_loudness": (C.c_int32, [_P, C.POINTER(C.c_float), _ERR]),
    "sb200_job_loudness": (C.c_int32, [_P, C.POINTER(C.c_double), C.POINTER(C.c_float), _ERR]),
    "sb200_job_set_prosody": (C.c_int32, [_P, C.POINTER(C.c_float), C.POINTER(C.c_float), _ERR]),
    "sb200_job_prosody": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int32), _ERR]),
    "sb200_job_set_pitch_contour": (C.c_int32, [_P, C.POINTER(C.c_float), _ERR]),
    "sb200_job_prosody_bounds": (C.c_int32, [_P, C.POINTER(C.c_int64), C.c_size_t, _ERR]),
    "sb200_job_id_frames":(C.c_int32, [_P, C.POINTER(C.c_int32), C.c_size_t, _ERR]),
    "sb200_job_run": (C.c_int32, [_P, C.c_void_p, C.c_size_t, C.POINTER(C.c_float), _ERR]),
    "sb200_job_fetch": (C.c_int32, [_P, C.POINTER(sb200_audio), _ERR]),
    "sb200_job_fetch_i16": (C.c_int32, [_P, C.POINTER(C.POINTER(C.c_int16)), C.POINTER(C.c_size_t), _ERR]),
    "sb200_i16_free": (None, [C.POINTER(C.c_int16)]),
    "sb200_job_fetch_g711": (C.c_int32, [_P, C.c_int32, C.POINTER(C.c_float), C.POINTER(C.POINTER(C.c_uint8)),
                                         C.POINTER(C.c_size_t), _ERR]),
    "sb200_bytes_free": (None, [C.POINTER(C.c_uint8)]),
    "sb200_job_fetch_flac": (C.c_int32, [_P, C.POINTER(C.c_float), C.POINTER(C.POINTER(C.c_uint8)),
                                         C.POINTER(C.c_size_t), _ERR]),
    "sb200_flac_encode": (C.c_int32, [C.c_int32, C.POINTER(C.c_int16), C.c_size_t, C.c_uint32,
                                      C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_size_t), _ERR]),
    "sb200_job_batch": (C.c_size_t, [_P]),
    "sb200_job_lengths": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "sb200_job_copy_out": (C.c_int32, [_P, C.c_void_p, C.c_size_t, C.c_int32, C.POINTER(C.c_size_t), _ERR]),
    "sb200_host_register": (C.c_int32, [C.c_void_p, C.c_size_t, _ERR]),
    "sb200_host_unregister": (C.c_int32, [C.c_void_p]),
    "sb200_job_free": (None, [_P]),
    "sb200_encode_ids": (C.c_int32, [_P, C.POINTER(C.c_int64), C.c_size_t, C.POINTER(_P), _ERR]),
    "sb200_latent_frames": (C.c_int64, [_P]),
    "sb200_decode_chunk": (C.c_int32, [_P, _P, C.c_int64, C.c_int64, C.POINTER(sb200_audio), _ERR]),
    "sb200_latent_free": (None, [_P]),
    "sb200_encode_batch_ids_configs": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.c_size_t,
                                                   C.POINTER(sb200_synth_config), C.POINTER(_P), _ERR]),
    "sb200_encode_batch_ids_durations": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.c_size_t,
                                                     C.POINTER(sb200_synth_config), C.POINTER(C.c_float),
                                                     C.POINTER(C.c_int32), C.POINTER(_P), _ERR]),
    "sb200_encode_batch_ids_seeded": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.c_size_t,
                                                  C.POINTER(sb200_synth_config), C.POINTER(C.c_float),
                                                  C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.POINTER(C.c_int32),
                                                  C.POINTER(_P), _ERR]),
    "sb200_encode_batch_ids_blends": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_size_t), C.c_size_t,
                                                  C.POINTER(sb200_synth_config), C.POINTER(C.c_float),
                                                  C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.POINTER(C.c_int32),
                                                  C.POINTER(C.c_int64), C.POINTER(C.c_float), C.POINTER(C.c_size_t),
                                                  C.POINTER(_P), _ERR]),
    "sb200_latent_id_frames":(C.c_int64, [_P, C.POINTER(C.c_int32), C.c_size_t]),
    "sb200_decode_chunks": (C.c_int32, [_P, C.POINTER(_P), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_size_t,
                                        C.POINTER(sb200_audio), _ERR]),
    "sb200_decode_chunks_i16": (C.c_int32, [_P, C.POINTER(_P), C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                            C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_size_t, C.c_int32,
                                            C.POINTER(C.c_float), C.POINTER(C.POINTER(C.c_int16)),
                                            C.POINTER(C.c_size_t), _ERR]),
    "sb200_decode_chunks_g711": (C.c_int32, [_P, C.POINTER(_P), C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                             C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_size_t, C.c_int32,
                                             C.POINTER(C.c_float), C.c_int32, C.POINTER(C.POINTER(C.c_uint8)),
                                             C.POINTER(C.c_size_t), _ERR]),
    "sb200_job_debug_fetch": (C.c_int32, [_P, C.c_char_p, C.c_size_t, C.POINTER(C.POINTER(C.c_float)),
                                          C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), _ERR]),
    "sb200_buffer_free": (None, [C.POINTER(C.c_float)]),
    "sb200_job_debug_durations": (C.c_int32, [_P, C.c_size_t, C.POINTER(C.POINTER(C.c_int32)),
                                              C.POINTER(C.c_size_t), _ERR]),
    "sb200_debug_decode_chunks": (C.c_int32, [_P, C.POINTER(_P), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_size_t,
                                              C.POINTER(C.POINTER(sb200_chunk_capture)), C.POINTER(C.c_size_t), _ERR]),
    "sb200_job_profile": (C.c_int32, [_P, C.POINTER(sb200_region_stat), C.c_int32]),
    "sb200_debug_plan": (C.c_int32, [C.c_int32, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, C.POINTER(C.c_int32)]),
    "sb200_debug_plan_staging": (C.c_int32, [C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                              C.c_int32, C.c_int32, C.POINTER(C.c_int32)]),
    "sb200_debug_conv_grid_cap": (C.c_int32, [C.c_int32]),
    "sb200_debug_conv": (C.c_int32, [C.c_int32, C.c_int32, C.POINTER(C.c_float), C.c_int32, C.c_int32,
                                     C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_int32, C.c_int32, C.c_int32,
                                     C.c_float, C.c_int32, C.POINTER(C.c_float), C.c_float, C.c_int32,
                                     C.POINTER(C.c_float), C.c_int32, _ERR]),
    "sb200_debug_conv_ex": (C.c_int32, [C.c_int32, C.c_int32, C.POINTER(C.c_float), C.c_int32, C.c_int32,
                                        C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_int32, C.c_int32, C.c_int32,
                                        C.c_float, C.c_int32, C.POINTER(C.c_float), C.c_float, C.POINTER(C.c_int32),
                                        C.c_int32, C.c_int32, C.POINTER(C.c_float), C.c_int32, C.c_int32,
                                        C.POINTER(C.c_float), C.c_int32, _ERR]),
    "sb200_debug_resblock2_stage": (C.c_int32, [C.c_int32, C.POINTER(C.c_float), C.c_int32, C.c_int32,
                                                C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_float),
                                                C.POINTER(C.c_float), C.POINTER(C.c_int32), C.c_int32, C.c_int32,
                                                C.POINTER(C.c_float), _ERR]),
    "sb200_debug_resblock2_plan": (C.c_int32, [C.c_int64, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                               C.POINTER(C.c_int32)]),
    "sb200_debug_spline": (C.c_int32, [C.c_int32, C.POINTER(C.c_float), C.c_int32, C.POINTER(C.c_float), C.c_int32,
                                       C.c_int32, C.c_int32, _ERR]),
    "sb200_debug_durations": (C.c_int32, [C.c_int32, C.POINTER(C.c_float), C.c_int32, C.POINTER(C.c_int32),
                                          C.POINTER(C.c_int32), C.c_int32, C.c_float, C.c_float, C.c_float,
                                          C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_int32), _ERR]),
    "sb200_debug_resample_filter": (C.c_int32, [C.c_int32, C.c_int32, C.POINTER(C.c_float), C.c_size_t,
                                                C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "sb200_resampler_create": (C.c_int32, [_P, C.c_uint32, C.POINTER(_P), _ERR]),
    "sb200_resampler_free": (None, [_P]),
    "sb200_decode_chunks_resampled": (C.c_int32, [_P, C.POINTER(_P), C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                                  C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_size_t, C.c_int32,
                                                  C.POINTER(C.c_float), C.POINTER(_P), C.POINTER(C.c_int32), C.c_int32,
                                                  C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), _ERR]),
    "sb200_prosody_stream_create": (C.c_int32, [_P, C.c_float, C.c_float, C.POINTER(_P), _ERR]),
    "sb200_prosody_stream_free": (None, [_P]),
    "sb200_prosody_stream_profile": (C.c_int32, [_P, C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    "sb200_decode_chunks_warped": (C.c_int32, [_P, C.POINTER(_P), C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                               C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_size_t, C.c_int32,
                                               C.POINTER(C.c_float), C.POINTER(_P), C.POINTER(_P), C.POINTER(C.c_int32),
                                               C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), _ERR]),
    "sb200_debug_prosody_stream_plan": (C.c_int32, [C.c_int32, C.c_float, C.c_float, C.POINTER(C.c_int64), C.c_size_t,
                                                    C.POINTER(C.c_int64)]),
    "sb200_debug_prosody_stream": (C.c_int32, [C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_int64), C.c_size_t,
                                               C.c_int32, C.c_float, C.c_float, C.POINTER(C.c_float), C.c_size_t,
                                               C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.c_size_t, _ERR]),
    "sb200_prosody_stream_create_contour": (C.c_int32, [_P, _P, C.POINTER(C.c_float), C.c_size_t, C.c_float,
                                                        C.POINTER(_P), _ERR]),
    "sb200_prosody_stream_bounds": (C.c_int32, [_P, C.POINTER(C.c_int64), C.c_size_t, _ERR]),
    "sb200_prosody_stream_create_formant": (C.c_int32, [_P, _P, C.c_float, C.POINTER(C.c_float), C.c_size_t,
                                                        C.c_float, C.c_float, C.POINTER(_P), _ERR]),
    "sb200_prosody_stream_profile_formant": (C.c_int32, [_P, C.POINTER(C.c_float)]),
    "sb200_loudness_stream_create": (C.c_int32, [_P, C.c_uint32, C.c_float, C.c_float, C.POINTER(_P), _ERR]),
    "sb200_loudness_stream_free": (None, [_P]),
    "sb200_loudness_stream_state": (C.c_int32, [_P, C.POINTER(C.c_double), C.POINTER(C.c_float),
                                                C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_float),
                                                _ERR]),
    "sb200_decode_chunks_metered": (C.c_int32, [_P, C.POINTER(_P), C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                                C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_size_t, C.c_int32,
                                                C.POINTER(C.c_float), C.POINTER(_P), C.POINTER(_P), C.POINTER(_P),
                                                C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_void_p),
                                                C.POINTER(C.c_size_t), _ERR]),
    "sb200_debug_formant_stream_plan": (C.c_int32, [C.c_int32, C.c_float, C.c_float, C.POINTER(C.c_int64),
                                                    C.POINTER(C.c_float), C.c_size_t, C.c_float, C.POINTER(C.c_int64),
                                                    C.c_size_t, C.POINTER(C.c_int64), _ERR]),
    "sb200_debug_formant_stream": (C.c_int32, [C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_int64), C.c_size_t,
                                               C.c_int32, C.c_float, C.c_float, C.POINTER(C.c_int64),
                                               C.POINTER(C.c_float), C.c_size_t, C.c_float, C.POINTER(C.c_float),
                                               C.c_size_t, C.POINTER(C.c_int64), _ERR]),
    "sb200_debug_prosody_contour_stream_plan": (C.c_int32, [C.c_int32, C.c_int64, C.POINTER(C.c_int64),
                                                            C.POINTER(C.c_float), C.c_size_t, C.c_float,
                                                            C.POINTER(C.c_int64), C.c_size_t, C.POINTER(C.c_int64)]),
    "sb200_debug_prosody_contour_stream": (C.c_int32, [C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_int64),
                                                       C.c_size_t, C.c_int32, C.POINTER(C.c_int64),
                                                       C.POINTER(C.c_float), C.c_size_t, C.c_float,
                                                       C.POINTER(C.c_float), C.c_size_t, C.POINTER(C.c_int64),
                                                       C.POINTER(C.c_int32), C.c_size_t, _ERR]),
    "sb200_debug_resample_emit": (C.c_int32, [C.c_int32, C.c_int32, C.POINTER(C.c_int64), C.c_size_t,
                                              C.POINTER(C.c_int64)]),
    "sb200_debug_resample": (C.c_int32, [C.c_int32, C.POINTER(C.c_float), C.c_size_t, C.c_int32, C.c_int32,
                                         C.POINTER(C.c_float), _ERR]),
    "sb200_debug_loudness_filter": (C.c_int32, [C.c_int32, C.POINTER(C.c_double)]),
    "sb200_debug_loudness": (C.c_int32, [C.c_int32, C.POINTER(C.c_float), C.c_size_t, C.c_int32, C.POINTER(C.c_double),
                                         _ERR]),
    "sb200_debug_loudness_stream": (C.c_int32, [C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_size_t), C.c_size_t,
                                                C.c_int32, C.c_float, C.c_float, C.POINTER(C.c_float),
                                                C.POINTER(C.c_double), C.POINTER(C.c_float), C.POINTER(C.c_int64),
                                                _ERR]),
    "sb200_debug_prosody_plan": (C.c_int32, [C.c_int32, C.c_int64, C.c_float, C.c_float, C.POINTER(C.c_int64),
                                             C.POINTER(C.c_int64), C.c_size_t]),
    "sb200_debug_prosody": (C.c_int32, [C.c_int32, C.POINTER(C.c_float), C.c_size_t, C.c_int32, C.c_float, C.c_float,
                                        C.POINTER(C.c_float), C.c_size_t, C.POINTER(C.c_int32), C.c_size_t,
                                        C.POINTER(C.c_float), C.c_size_t, _ERR]),
    "sb200_debug_prosody_contour_plan": (C.c_int32, [C.c_int32, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_float),
                                                     C.c_size_t, C.c_float, C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                                     C.c_size_t, C.POINTER(C.c_int64)]),
    "sb200_debug_prosody_contour": (C.c_int32, [C.c_int32, C.POINTER(C.c_float), C.c_size_t, C.c_int32,
                                                C.POINTER(C.c_int64), C.POINTER(C.c_float), C.c_size_t, C.c_float,
                                                C.POINTER(C.c_float), C.c_size_t, C.POINTER(C.c_int32), C.c_size_t,
                                                C.POINTER(C.c_float), C.c_size_t, _ERR]),
    "sb200_debug_g711": (C.c_int32, [C.c_int32, C.c_int32, C.POINTER(C.c_int16), C.c_size_t, C.POINTER(C.c_uint8),
                                     _ERR]),
    "sb200_launch_count": (C.c_uint64, []),
    "sb200_set_backend": (C.c_int32, [_P, C.c_int32]),
}

_lib = None


def lib() -> C.CDLL:
    """Load the shared library (once).  Raises ImportError with a build hint when absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(libsonata_b200 has no CPU fallback)")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib
