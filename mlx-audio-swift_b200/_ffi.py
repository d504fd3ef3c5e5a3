"""ctypes binding of libb200audio.so (include/b200audio.h).  This is the same C ABI a Swift wrapper
binds (INTEGRATION.md); Python is only the host language available in this image.

There is no CPU fallback: if the library is missing, `lib()` raises; if no CUDA device is visible,
every create/compute call raises `AudioGenerationError` with code B2A_ERR_CUDA."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

LIB_PATH = Path(__file__).resolve().parent / "lib" / "libb200audio.so"

(OK, ERR_MODEL_NOT_INITIALIZED, ERR_GENERATION_FAILED, ERR_INVALID_INPUT, ERR_AUDIO_DECODING_FAILED,
 ERR_AUDIO_ENCODING_FAILED, ERR_CANCELLED, ERR_CUDA) = range(8)
DTYPE_F32, DTYPE_BF16, DTYPE_I32 = 0, 1, 2


class AudioGenerationError(RuntimeError):
    """Sources/MLXAudioCore/Generation/GenerationTypes.swift:66-87 (+ cancelled, cuda)."""
    CASES = {1: "modelNotInitialized", 2: "generationFailed", 3: "invalidInput", 4: "audioDecodingFailed",
             5: "audioEncodingFailed", 6: "cancelled", 7: "cudaError"}

    def __init__(self, code: int, message: str):
        super().__init__(f"{self.CASES.get(code, code)}: {message}")
        self.code, self.case, self.message = code, self.CASES.get(code, str(code)), message


class Tensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("dtype", C.c_int32), ("ndim", C.c_int32), ("shape", C.c_int64 * 4),
                ("data", C.c_void_p)]


class SnacConfig(C.Structure):
    _fields_ = [("sampling_rate", C.c_int32), ("encoder_dim", C.c_int32), ("n_encoder_rates", C.c_int32),
                ("encoder_rates", C.c_int32 * 8), ("latent_dim", C.c_int32), ("decoder_dim", C.c_int32),
                ("n_decoder_rates", C.c_int32), ("decoder_rates", C.c_int32 * 8), ("attn_window_size", C.c_int32),
                ("codebook_size", C.c_int32), ("codebook_dim", C.c_int32), ("n_vq_strides", C.c_int32),
                ("vq_strides", C.c_int32 * 8), ("noise", C.c_int32), ("depthwise", C.c_int32)]


class LlamaConfig(C.Structure):
    _fields_ = [("hidden_size", C.c_int32), ("num_hidden_layers", C.c_int32), ("intermediate_size", C.c_int32),
                ("num_attention_heads", C.c_int32), ("num_key_value_heads", C.c_int32), ("head_dim", C.c_int32),
                ("vocab_size", C.c_int32), ("rms_norm_eps", C.c_float), ("rope_theta", C.c_float),
                ("rope_factor", C.c_float), ("rope_low_freq_factor", C.c_float), ("rope_high_freq_factor", C.c_float),
                ("rope_old_context_len", C.c_float), ("tie_word_embeddings", C.c_int32), ("max_batch", C.c_int32),
                ("max_context", C.c_int32)]


class Qwen3LMConfig(C.Structure):
    _fields_ = ([(n, C.c_int32) for n in ("hidden_size", "num_hidden_layers", "intermediate_size", "num_attention_heads",
                                           "num_key_value_heads", "head_dim", "vocab_size")]
                + [("rms_norm_eps", C.c_float), ("rope_theta", C.c_float), ("rope_linear_factor", C.c_float)]
                + [(n, C.c_int32) for n in ("tie_word_embeddings", "max_position_embeddings", "sample_rate", "eos_token_id", "max_batch",
                                             "max_context")])


class SopranoConfig(C.Structure):
    _fields_ = ([(n, C.c_int32) for n in ("hidden_size", "num_hidden_layers", "intermediate_size", "num_attention_heads",
                                           "num_key_value_heads", "head_dim", "vocab_size")]
                + [("rms_norm_eps", C.c_float), ("rope_theta", C.c_float)]
                + [(n, C.c_int32) for n in ("tie_word_embeddings", "max_position_embeddings", "bos_token_id", "eos_token_id", "pad_token_id",
                                             "stop_token_id", "sample_rate", "decoder_num_layers", "decoder_dim", "decoder_intermediate_dim",
                                             "hop_length", "n_fft", "upscale", "input_kernel", "dw_kernel", "token_size", "receptive_field",
                                             "max_batch", "max_context")])


class GenParams(C.Structure):
    _fields_ = [("max_tokens", C.c_int32), ("temperature", C.c_float), ("top_p", C.c_float),
                ("repetition_penalty", C.c_float), ("repetition_context_size", C.c_int32), ("seed", C.c_uint64)]


class GenInfo(C.Structure):
    _fields_ = [("prompt_token_count", C.c_int32), ("generation_token_count", C.c_int32), ("prefill_time", C.c_double),
                ("generate_time", C.c_double), ("tokens_per_second", C.c_double), ("codec_time", C.c_double),
                ("peak_memory_gb", C.c_double)]


class VocosConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("input_channels", "dim", "intermediate_dim", "num_layers", "n_fft", "hop_length",
                                          "input_kernel_size", "dw_kernel_size", "adanorm_num_embeddings")]


class EncodecConfig(C.Structure):
    _fields_ = ([(n, C.c_int32) for n in ("audio_channels", "num_filters", "kernel_size", "num_residual_layers",
                                           "dilation_growth_rate", "codebook_size", "codebook_dim", "hidden_size",
                                           "num_lstm_layers", "residual_kernel_size", "use_causal_conv", "pad_mode_reflect",
                                           "norm_type", "last_kernel_size", "compress", "n_upsampling_ratios")]
                + [("upsampling_ratios", C.c_int32 * 8), ("sampling_rate", C.c_int32), ("use_conv_shortcut", C.c_int32),
                   ("trim_right_ratio", C.c_float), ("chunk_length_s", C.c_float), ("overlap", C.c_float),
                   ("normalize", C.c_int32)])


class SpeechTokenizerConfig(C.Structure):
    _fields_ = ([(n, C.c_int32) for n in ("codebook_size", "codebook_dim", "latent_dim", "decoder_dim", "hidden_size",
                                           "intermediate_size", "head_dim", "num_attention_heads", "num_key_value_heads",
                                           "num_hidden_layers", "num_quantizers", "num_semantic_quantizers")]
                + [("rms_norm_eps", C.c_float), ("rope_theta", C.c_float), ("attention_bias", C.c_int32),
                   ("num_upsample_rates", C.c_int32), ("upsample_rates", C.c_int32 * 8),
                   ("num_upsampling_ratios", C.c_int32), ("upsampling_ratios", C.c_int32 * 8),
                   ("max_batch", C.c_int32), ("max_cache_frames", C.c_int32)])


class SpeechTokenizerEncoderConfig(C.Structure):
    _fields_ = ([("sampling_rate", C.c_int32), ("frame_rate", C.c_float)]
                + [(n, C.c_int32) for n in ("audio_channels", "num_filters", "num_residual_layers", "num_upsampling_ratios")]
                + [("upsampling_ratios", C.c_int32 * 8)]
                + [(n, C.c_int32) for n in ("kernel_size", "residual_kernel_size", "last_kernel_size", "compress", "use_causal_conv",
                                           "use_conv_shortcut", "hidden_size", "intermediate_size", "num_hidden_layers",
                                           "num_attention_heads", "num_key_value_heads", "head_dim")]
                + [("rope_theta", C.c_float)]
                + [(n, C.c_int32) for n in ("codebook_size", "codebook_dim", "num_quantizers", "valid_num_quantizers")])


class MimiConfig(C.Structure):
    _fields_ = ([("sample_rate", C.c_int32), ("frame_rate", C.c_float)]
                + [(n, C.c_int32) for n in ("channels", "dimension", "n_filters", "n_residual_layers", "num_ratios")]
                + [("ratios", C.c_int32 * 8)]
                + [(n, C.c_int32) for n in ("kernel_size", "residual_kernel_size", "last_kernel_size", "dilation_base", "compress", "causal",
                                           "true_skip", "num_heads", "num_layers", "dim_feedforward", "context", "max_period", "gating",
                                           "norm_rms", "kv_repeat", "num_codebooks", "codebook_size", "codebook_dim", "max_batch",
                                           "max_cache_frames")])


class Qwen3SpeakerEncoderConfig(C.Structure):
    _fields_ = ([(n, C.c_int32) for n in ("mel_dim", "enc_dim", "num_enc_layers")]
                + [(n, C.c_int32 * 8) for n in ("enc_channels", "enc_kernel_sizes", "enc_dilations")]
                + [(n, C.c_int32) for n in ("enc_attention_channels", "enc_res2net_scale", "enc_se_channels", "sample_rate")])


class Qwen3TalkerConfig(C.Structure):
    _fields_ = ([(n, C.c_int32) for n in ("vocab_size", "hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads",
                                           "num_key_value_heads", "head_dim")]
                + [("rms_norm_eps", C.c_float), ("rope_theta", C.c_float)]
                + [(n, C.c_int32) for n in ("num_code_groups", "text_hidden_size", "text_vocab_size", "codec_eos_token_id", "cp_vocab_size",
                                             "cp_hidden_size", "cp_intermediate_size", "cp_num_hidden_layers", "cp_num_attention_heads",
                                             "cp_num_key_value_heads", "cp_head_dim")]
                + [("cp_rms_norm_eps", C.c_float), ("cp_rope_theta", C.c_float), ("max_batch", C.c_int32), ("max_context", C.c_int32)])


class Qwen3GenParams(C.Structure):
    _fields_ = [("max_tokens", C.c_int32), ("temperature", C.c_float), ("top_p", C.c_float), ("top_k", C.c_int32), ("min_p", C.c_float),
                ("repetition_penalty", C.c_float), ("seed", C.c_uint64)]


class WhisperConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("vocab_size", "num_mel_bins", "d_model", "encoder_layers", "encoder_attention_heads",
                                          "encoder_ffn_dim", "max_source_positions", "decoder_layers", "decoder_attention_heads",
                                          "decoder_ffn_dim", "max_target_positions", "max_batch")]


class SttParams(C.Structure):
    _fields_ = [("max_tokens", C.c_int32), ("temperature", C.c_float), ("prompt_ids", C.c_void_p), ("n_prompt", C.c_int32),
                ("begin_suppress", C.c_void_p), ("n_begin_suppress", C.c_int32), ("suppress", C.c_void_p),
                ("n_suppress", C.c_int32), ("timestamp_begin", C.c_int32), ("eot", C.c_int32), ("seed", C.c_uint64)]


class SttInfo(C.Structure):
    _fields_ = [("prompt_tokens", C.c_int32), ("generation_tokens", C.c_int32), ("decode_steps", C.c_int32),
                ("encode_time", C.c_double), ("decode_time", C.c_double), ("total_time", C.c_double)]


TOKEN_CB = C.CFUNCTYPE(None, C.c_void_p, C.c_int32, C.c_int32, C.c_int32)
AUDIO_CB = C.CFUNCTYPE(None, C.c_void_p, C.c_int32, C.POINTER(C.c_float), C.c_int64, C.c_int32)
STT_DECODE_CB = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.POINTER(C.c_float), C.c_int64, C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_int32),
                            C.c_int32, C.POINTER(C.c_int32))


class SttStreamConfig(C.Structure):
    _fields_ = [("decode_interval_s", C.c_double), ("window_s", C.c_double), ("window_overlap_s", C.c_double), ("delay_ms", C.c_int32),
                ("min_agreement_passes", C.c_int32), ("max_tokens_per_pass", C.c_int32), ("sample_rate", C.c_int32)]


class SttStreamUpdate(C.Structure):
    _fields_ = [("kind", C.c_int32), ("promoted", C.c_int32), ("completed_windows", C.c_int32), ("n_confirmed", C.c_int32),
                ("n_provisional", C.c_int32), ("total_audio_s", C.c_double), ("pass_encode_time", C.c_double), ("pass_decode_time", C.c_double)]


# name -> (restype, argtypes); every symbol include/b200audio.h and include/b200audio_internal.h declare
_P = C.c_void_p
SIGNATURES = {
    "b2a_last_error": (C.c_char_p, []),
    "b2a_version": (C.c_char_p, []),
    "b2a_device_count": (C.c_int32, []),
    "b2a_launch_count": (C.c_int64, []),
    "b2a_hanning_window": (C.c_int32, [C.c_int32, C.c_int32, _P]),
    "b2a_hamming_window": (C.c_int32, [C.c_int32, C.c_int32, _P]),
    "b2a_power_to_db": (C.c_int32, [_P, C.c_int64, C.c_float, C.c_float, _P]),
    "b2a_mel_filters": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_int32, C.c_int32, _P]),
    "b2a_mel_create": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_P)]),
    "b2a_mel_max_frames": (C.c_int64, [_P, C.c_int64]),
    "b2a_mel_process": (C.c_int32, [_P, _P, C.c_int64, _P, C.c_int64, C.POINTER(C.c_int64)]),
    "b2a_mel_flush": (C.c_int32, [_P, _P, C.c_int64, C.POINTER(C.c_int64)]),
    "b2a_mel_reset": (C.c_int32, [_P]),
    "b2a_mel_total_frames": (C.c_int64, [_P]),
    "b2a_mel_destroy": (None, [_P]),
    "b2a_logmel_create": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_P)]),
    "b2a_logmel_frames": (C.c_int64, [_P, C.c_int64]),
    "b2a_logmel_compute": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, _P]),
    "b2a_logmel_compute_dev": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, _P, _P]),
    "b2a_logmel_destroy": (None, [_P]),
    "b2a_snac_create": (C.c_int32, [C.c_int32, C.POINTER(SnacConfig), C.POINTER(Tensor), C.c_int32, C.POINTER(_P)]),
    "b2a_snac_hop_length": (C.c_int64, [_P]),
    "b2a_snac_decoded_length": (C.c_int64, [_P, C.c_int64]),
    "b2a_snac_decode": (C.c_int32, [_P, C.POINTER(_P), C.c_int32, C.c_int64, C.POINTER(_P), C.c_int32, C.c_uint64, _P]),
    "b2a_snac_decode_dev": (C.c_int32, [_P, C.POINTER(_P), C.c_int32, C.c_int64, C.POINTER(_P), C.c_int32, C.c_uint64, _P, _P]),
    "b2a_snac_quantize": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, C.POINTER(_P), _P]),
    "b2a_snac_encoded_length": (C.c_int64, [_P, C.c_int64]),
    "b2a_snac_encode": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, C.POINTER(_P)]),
    "b2a_snac_encode_dev": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, C.POINTER(_P), _P]),
    "b2a_snac_encode_latent_test": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, _P]),
    "b2a_snac_local_attn_test": (C.c_int32, [_P, _P] + [C.c_int32] * 4 + [_P]),
    "b2a_snac_destroy": (None, [_P]),
    "b2a_tts_create": (C.c_int32, [C.c_int32, C.POINTER(LlamaConfig), C.POINTER(Tensor), C.c_int32, _P, C.POINTER(_P)]),
    "b2a_tts_debug_trace": (C.c_int32, [_P, C.c_int32, C.c_int32, _P]),
    "b2a_debug_step_smem": (C.c_int32, [C.c_int32, C.POINTER(C.c_int32)]),
    "b2a_debug_step_smem_rows": (C.c_int32, [C.c_int32, C.c_int32, C.POINTER(C.c_int32)]),
    "b2a_tts_create_random": (C.c_int32, [C.c_int32, C.POINTER(LlamaConfig), C.c_float, C.c_uint64, _P, C.POINTER(_P)]),
    "b2a_tts_stream": (C.c_void_p, [_P]),
    "b2a_tts_set_bench_flags": (C.c_int32, [_P, C.c_int32, C.c_int32]),
    "b2a_stt_set_bench_flags": (C.c_int32, [_P, C.c_int32]),
    "b2a_tts_time_steps": (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_float)]),
    "b2a_snac_stream": (C.c_void_p, [_P]),
    "b2a_tts_prepare_input_ids": (C.c_int32, [C.POINTER(_P), _P, C.c_int32, _P, C.POINTER(C.c_int32)]),
    "b2a_tts_prepare_input_ids_ref": (C.c_int32, [C.POINTER(_P), _P, C.c_int32, _P, C.c_int32, _P, C.c_int32, _P, C.POINTER(C.c_int32)]),
    "b2a_tts_forward_logits": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32, _P]),
    "b2a_tts_generate": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.POINTER(GenParams), _P, _P, _P, C.c_int64, _P,
                                     C.POINTER(GenInfo), TOKEN_CB, _P]),
    "b2a_tts_generate_stream": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.POINTER(GenParams), C.c_int32, C.c_int32, _P, _P,
                                            C.POINTER(GenInfo), TOKEN_CB, AUDIO_CB, _P]),
    "b2a_tts_generate_dev": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.POINTER(GenParams), _P, C.c_int64, _P,
                                         C.POINTER(GenInfo)]),
    "b2a_tts_cancel": (C.c_int32, [_P]),
    "b2a_tts_parse_output": (C.c_int32, [_P, C.c_int32, C.c_int32, _P, _P]),
    "b2a_tts_deinterleave": (C.c_int32, [_P, C.c_int32, _P, _P, _P, C.POINTER(C.c_int32)]),
    "b2a_tts_interleave": (C.c_int32, [_P, _P, _P, C.c_int32, _P]),
    "b2a_tts_destroy": (None, [_P]),
    "b2a_qwen3_lm_create": (C.c_int32, [C.c_int32, C.POINTER(Qwen3LMConfig), C.POINTER(Tensor), C.c_int32, _P, C.POINTER(_P)]),
    "b2a_qwen3_lm_create_random": (C.c_int32, [C.c_int32, C.POINTER(Qwen3LMConfig), C.c_float, C.c_uint64, _P, C.POINTER(_P)]),
    "b2a_qwen3_lm_config_from_json": (C.c_int32, [C.c_char_p, C.c_int32, C.c_int32, C.POINTER(Qwen3LMConfig), C.POINTER(C.c_int32),
                                                  C.POINTER(C.c_int32)]),
    "b2a_qwen3_lm_create_from_directory": (C.c_int32, [C.c_char_p, C.c_int32, C.c_int32, C.c_int32, _P, C.POINTER(_P)]),
    "b2a_qwen3_lm_prepare_input_ids": (C.c_int32, [C.POINTER(_P), _P, C.c_int32, _P, C.POINTER(C.c_int32)]),
    "b2a_qwen3_lm_prepare_input_ids_ref": (C.c_int32, [C.POINTER(_P), _P, C.c_int32, _P, C.c_int32, _P, C.c_int32, _P,
                                                       C.POINTER(C.c_int32)]),
    "b2a_qwen3_lm_parse_output": (C.c_int32, [_P, C.c_int32, C.c_int32, _P, _P]),
    "b2a_soprano_create": (C.c_int32, [C.c_int32, C.POINTER(SopranoConfig), C.POINTER(Tensor), C.c_int32, C.POINTER(_P)]),
    "b2a_soprano_create_random": (C.c_int32, [C.c_int32, C.POINTER(SopranoConfig), C.c_float, C.c_uint64, C.POINTER(Tensor), C.c_int32,
                                              C.POINTER(_P)]),
    "b2a_soprano_config_from_json": (C.c_int32, [C.c_char_p, C.c_char_p, C.c_int32, C.c_int32, C.POINTER(SopranoConfig),
                                                 C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "b2a_soprano_create_from_directory": (C.c_int32, [C.c_char_p, C.c_char_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_P)]),
    "b2a_soprano_decode_hidden": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, _P, C.c_int64, _P]),
    "b2a_soprano_wave_length": (C.c_int64, [_P, C.c_int32]),
    "b2a_soprano_hidden_states": (C.c_int32, [_P, C.c_int32, _P, _P]),
    "b2a_vocos_create": (C.c_int32, [C.c_int32, C.POINTER(VocosConfig), C.POINTER(Tensor), C.c_int32, C.POINTER(_P)]),
    "b2a_vocos_output_length": (C.c_int64, [_P, C.c_int32]),
    "b2a_vocos_stream": (C.c_void_p, [_P]),
    "b2a_vocos_decode": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, _P]),
    "b2a_vocos_decode_dev": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, _P, _P]),
    "b2a_vocos_decode_cond": (C.c_int32, [_P, _P, _P, C.c_int32, C.c_int32, _P]),
    "b2a_vocos_destroy": (None, [_P]),
    "b2a_vocos_decode_upsampled_dev": (C.c_int32, [_P, _P, C.c_int64, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    "b2a_vocos_upsampled_length": (C.c_int64, [_P, C.c_int32, C.c_int32]),
    "b2a_speech_tokenizer_create": (C.c_int32, [C.c_int32, C.POINTER(SpeechTokenizerConfig), C.POINTER(Tensor), C.c_int32, C.POINTER(_P)]),
    "b2a_speech_tokenizer_total_upsample": (C.c_int32, [_P]),
    "b2a_speech_tokenizer_stream": (C.c_void_p, [_P]),
    "b2a_speech_tokenizer_reset": (C.c_int32, [_P]),
    "b2a_speech_tokenizer_streaming_step": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32, _P]),
    "b2a_speech_tokenizer_streaming_step_dev": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    "b2a_speech_tokenizer_streaming_decode": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P]),
    "b2a_speech_tokenizer_chunked_decode": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P]),
    "b2a_speech_tokenizer_destroy": (None, [_P]),
    "b2a_weights_sanitize_speech_tokenizer": (C.c_int32, [_P]),
    "b2a_speech_tokenizer_config_from_json": (C.c_int32, [C.c_char_p, C.c_int32, C.c_int32, C.POINTER(SpeechTokenizerConfig), C.POINTER(C.c_int32)]),
    "b2a_speech_tokenizer_create_from_directory": (C.c_int32, [C.c_char_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_P), C.POINTER(C.c_int32)]),
    "b2a_qwen3_sample_test": (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_int32, C.c_float, C.c_float, C.c_int32, C.c_int32,
                                         C.c_int32, _P, C.c_int32, C.c_uint64, C.c_int32, _P, _P]),
    "b2a_implicit_conv_test": (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int32, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                          _P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P, C.c_int32, C.c_int32, _P, _P]),
    "b2a_tc_gemm_test": (C.c_int32, [_P, _P, _P] + [C.c_int32] * 8 + [_P]),
    "b2a_tc_gemm_epilogue_test": (C.c_int32, [_P, _P, _P] + [C.c_int32] * 8 + [_P, C.c_int32, C.c_int32, C.c_int32, _P, C.c_int32,
                                                                             C.c_float, C.c_int32, _P]),
    "b2a_tc_gemm_splitk_test": (C.c_int32, [_P, _P, _P, _P, _P, _P] + [C.c_int32] * 5 + [_P]),
    "b2a_tc_gemm_splitk_store_test": (C.c_int32, [_P, _P, _P, _P, C.c_int32, C.c_float] + [C.c_int32] * 6 + [_P]),
    "b2a_debug_qkv_split": (C.c_int32, [C.c_int32, C.c_int32, C.POINTER(C.c_int32)]),
    "b2a_mha_tc_test": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32, _P]),
    "b2a_prompt_attn_test": (C.c_int32, [_P, _P, _P, _P, C.c_float, _P, _P, _P] + [C.c_int32] * 6 + [_P]),
    "b2a_decode_attn_test": (C.c_int32, [_P, _P, _P, _P, _P, C.c_float, _P, _P, _P] + [C.c_int32] * 4 + [_P]),
    "b2a_wh_decode_attn_test": (C.c_int32, [C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P]),
    "b2a_conv_gemm_test": (C.c_int32, [_P, C.c_int32, C.c_int32, _P, C.c_int32, C.c_int32, _P, _P, _P, C.c_int32, _P, C.c_int32, _P,
                                       C.c_int32] + [C.c_int32] * 6 + [_P, C.c_uint64, C.c_int32, _P]),
    "b2a_snac_unit_test": (C.c_int32, [C.c_int32] * 3 + [_P, _P, C.c_int32, C.c_int32] + [_P] * 6 + [_P, C.c_uint64, _P, _P, C.c_int32, _P]),
    "b2a_snac_convt_test": (C.c_int32, [_P] * 5 + [C.c_int32] * 5 + [_P]),
    "b2a_speech_tokenizer_debug_stage": (C.c_int32, [_P, C.c_int32, _P, C.c_int64, _P]),
    "b2a_speech_tokenizer_debug_layout": (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, C.c_int64, _P, _P, _P]),
    "b2a_encodec_create": (C.c_int32, [C.c_int32, C.POINTER(EncodecConfig), C.POINTER(Tensor), C.c_int32, C.POINTER(_P)]),
    "b2a_encodec_output_length": (C.c_int64, [_P, C.c_int32, C.c_int32]),
    "b2a_encodec_num_codebooks": (C.c_int32, [_P]),
    "b2a_encodec_stream": (C.c_void_p, [_P]),
    "b2a_encodec_decode": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    "b2a_encodec_decode_dev": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P]),
    "b2a_encodec_encoded_shape": (C.c_int32, [_P, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "b2a_encodec_encode": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, C.c_int32, _P, _P]),
    "b2a_encodec_encode_dev": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, C.c_int32, _P, _P, _P]),
    "b2a_encodec_encode_latent_test": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, _P]),
    "b2a_speech_tokenizer_encoder_create": (C.c_int32, [C.c_int32, C.POINTER(SpeechTokenizerEncoderConfig), C.POINTER(Tensor), C.c_int32, C.POINTER(_P)]),
    "b2a_speech_tokenizer_encoder_encoded_length": (C.c_int64, [_P, C.c_int64]),
    "b2a_speech_tokenizer_encoder_num_code_groups": (C.c_int32, [_P]),
    "b2a_speech_tokenizer_encoder_encode": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, _P]),
    "b2a_speech_tokenizer_encoder_encode_dev": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, _P, _P]),
    "b2a_speech_tokenizer_encoder_stream": (C.c_void_p, [_P]),
    "b2a_speech_tokenizer_encoder_destroy": (None, [_P]),
    "b2a_speech_tokenizer_encoder_latent_test": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, _P, _P]),
    "b2a_weights_sanitize_speech_tokenizer_encoder": (C.c_int32, [_P]),
    "b2a_speech_tokenizer_encoder_config_from_json": (C.c_int32, [C.c_char_p, C.POINTER(SpeechTokenizerEncoderConfig)]),
    "b2a_speech_tokenizer_encoder_create_from_directory": (C.c_int32, [C.c_char_p, C.c_int32, C.POINTER(_P)]),
    "b2a_qwen3_speaker_encoder_create": (C.c_int32, [C.c_int32, C.POINTER(Qwen3SpeakerEncoderConfig), C.POINTER(Tensor), C.c_int32, C.POINTER(_P)]),
    "b2a_qwen3_speaker_encoder_frames": (C.c_int64, [_P, C.c_int64]),
    "b2a_qwen3_speaker_encoder_embed": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, _P]),
    "b2a_qwen3_speaker_encoder_embed_dev": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, _P, _P]),
    "b2a_qwen3_speaker_encoder_embed_mel": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, _P]),
    "b2a_qwen3_speaker_encoder_stream": (C.c_void_p, [_P]),
    "b2a_qwen3_speaker_encoder_destroy": (None, [_P]),
    "b2a_weights_sanitize_qwen3_speaker_encoder": (C.c_int32, [_P]),
    "b2a_qwen3_speaker_encoder_config_from_json": (C.c_int32, [C.c_char_p, C.POINTER(Qwen3SpeakerEncoderConfig)]),
    "b2a_qwen3_speaker_encoder_create_from_directory": (C.c_int32, [C.c_char_p, C.c_int32, C.POINTER(_P)]),
    "b2a_mimi_config_default": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(MimiConfig)]),
    "b2a_mimi_create": (C.c_int32, [C.c_int32, C.POINTER(MimiConfig), C.POINTER(Tensor), C.c_int32, C.POINTER(_P)]),
    "b2a_weights_sanitize_mimi": (C.c_int32, [_P]),
    "b2a_mimi_create_from_file": (C.c_int32, [C.c_char_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_P)]),
    "b2a_mimi_num_codebooks": (C.c_int32, [_P]),
    "b2a_mimi_samples_per_frame": (C.c_int32, [_P]),
    "b2a_mimi_encoded_length": (C.c_int64, [_P, C.c_int64]),
    "b2a_mimi_encode": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, _P]),
    "b2a_mimi_encode_dev": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, _P, _P]),
    "b2a_mimi_decode": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32, _P]),
    "b2a_mimi_decode_dev": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    "b2a_mimi_decode_step": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32, _P]),
    "b2a_mimi_decode_step_dev": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    "b2a_mimi_decode_frames": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32, _P]),
    "b2a_mimi_reset": (C.c_int32, [_P]),
    "b2a_mimi_stream": (C.c_void_p, [_P]),
    "b2a_mimi_destroy": (None, [_P]),
    "b2a_encodec_destroy": (None, [_P]),
    "b2a_weights_load": (C.c_int32, [C.c_char_p, C.POINTER(_P)]),
    "b2a_weights_count": (C.c_int32, [_P]),
    "b2a_weights_get": (C.c_int32, [_P, C.c_int32, C.POINTER(Tensor)]),
    "b2a_weights_sanitize_whisper": (C.c_int32, [_P, C.POINTER(C.c_int32)]),
    "b2a_weights_sanitize_llama": (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int32]),
    "b2a_weights_sanitize_llama_config": (C.c_int32, [_P, C.c_char_p]),
    "b2a_weights_sanitize_soprano_config": (C.c_int32, [_P, C.c_char_p]),
    "b2a_weights_dequantize": (C.c_int32, [_P, C.c_int32, C.c_int32]),
    "b2a_weights_free": (None, [_P]),
    "b2a_tts_config_from_json": (C.c_int32, [C.c_char_p, C.c_int32, C.c_int32, C.POINTER(LlamaConfig), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "b2a_tts_create_from_directory": (C.c_int32, [C.c_char_p, C.c_int32, C.c_int32, C.c_int32, _P, C.POINTER(_P)]),
    "b2a_stt_create": (C.c_int32, [C.c_int32, C.POINTER(WhisperConfig), C.POINTER(Tensor), C.c_int32, C.POINTER(_P)]),
    "b2a_stt_create_random": (C.c_int32, [C.c_int32, C.POINTER(WhisperConfig), C.c_float, C.c_uint64, C.POINTER(_P)]),
    "b2a_stt_stream": (C.c_void_p, [_P]),
    "b2a_stt_encode": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, _P]),
    "b2a_stt_decoder_logits": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, _P]),
    "b2a_stt_transcribe": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, C.POINTER(SttParams), _P, _P, C.POINTER(SttInfo)]),
    "b2a_stt_transcribe_dev": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, C.POINTER(SttParams), _P, _P, C.POINTER(SttInfo)]),
    "b2a_stt_transcribe_long": (C.c_int32, [_P, _P, C.c_int64, C.POINTER(SttParams), C.c_int32, _P, _P, _P, C.POINTER(C.c_int32), C.POINTER(SttInfo)]),
    "b2a_qwen3_talker_create": (C.c_int32, [C.c_int32, C.POINTER(Qwen3TalkerConfig), C.POINTER(Tensor), C.c_int32, C.POINTER(_P)]),
    "b2a_qwen3_talker_create_random": (C.c_int32, [C.c_int32, C.POINTER(Qwen3TalkerConfig), C.c_float, C.c_uint64, C.POINTER(_P)]),
    "b2a_qwen3_talker_set_bench_flags": (C.c_int32, [_P, C.c_int32]),
    "b2a_qwen3_talker_stream": (C.c_void_p, [_P]),
    "b2a_qwen3_talker_embed_text": (C.c_int32, [_P, _P, C.c_int32, _P]),
    "b2a_qwen3_talker_embed_codec": (C.c_int32, [_P, _P, C.c_int32, _P]),
    "b2a_qwen3_talker_embed_code_frames": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, _P]),
    "b2a_qwen3_talker_forward": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, _P, _P]),
    "b2a_qwen3_talker_generate": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, _P, _P, C.c_int32, _P, C.POINTER(Qwen3GenParams), _P, _P,
                                              C.POINTER(GenInfo), _P, _P]),
    "b2a_qwen3_talker_config_from_json": (C.c_int32, [C.c_char_p, C.c_int32, C.c_int32, C.POINTER(Qwen3TalkerConfig)]),
    "b2a_weights_sanitize_qwen3_talker": (C.c_int32, [_P, C.c_char_p]),
    "b2a_qwen3_talker_create_from_directory": (C.c_int32, [C.c_char_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_P)]),
    "b2a_qwen3_talker_cancel": (C.c_int32, [_P]),
    "b2a_qwen3_talker_destroy": (None, [_P]),
    "b2a_stt_session_create": (C.c_int32, [_P, C.POINTER(SttParams), C.POINTER(SttStreamConfig), C.POINTER(_P)]),
    "b2a_stt_session_create_with_decoder": (C.c_int32, [STT_DECODE_CB, _P, C.POINTER(SttStreamConfig), C.POINTER(_P)]),
    "b2a_stt_session_feed": (C.c_int32, [_P, _P, C.c_int64, C.c_double, C.POINTER(SttStreamUpdate)]),
    "b2a_stt_session_stop": (C.c_int32, [_P, C.c_double, C.POINTER(SttStreamUpdate)]),
    "b2a_stt_session_tokens": (C.c_int32, [_P, C.c_int32, C.c_int32, _P, C.c_int32, C.POINTER(C.c_int32)]),
    "b2a_stt_session_destroy": (None, [_P]),
    "b2a_stt_cancel": (C.c_int32, [_P]),
    "b2a_stt_destroy": (None, [_P]),
}

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`"
                              " -- there is no CPU fallback")
        _lib = C.CDLL(str(LIB_PATH))
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(_lib, name)
            fn.restype, fn.argtypes = res, args
    return _lib


def check(status: int) -> None:
    if status != OK:
        raise AudioGenerationError(status, lib().b2a_last_error().decode("utf-8", "replace"))


def ptr(a) -> C.c_void_p:
    """Pointer to a C-contiguous numpy array or torch tensor (host or device)."""
    if a is None:
        return C.c_void_p(None)
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"]
        return C.c_void_p(a.ctypes.data)
    return C.c_void_p(a.data_ptr())  # torch tensor


def make_tensor_table(weights: dict):
    """dict name -> numpy fp32/int32 array or torch bf16/fp32 tensor  ->  (Tensor array, keepalive list)."""
    import torch
    arr = (Tensor * len(weights))()
    keep = []
    for i, (name, w) in enumerate(weights.items()):
        if isinstance(w, torch.Tensor):
            w = w.detach().contiguous().cpu()
            if w.dtype == torch.bfloat16:
                dt = DTYPE_BF16
            elif w.dtype == torch.float32:
                dt = DTYPE_F32
            else:
                w = w.to(torch.float32); dt = DTYPE_F32
            data, shape = w.data_ptr(), tuple(w.shape)
        else:
            w = np.ascontiguousarray(w)
            if w.dtype == np.int32:
                dt = DTYPE_I32
            else:
                if w.dtype != np.float32:
                    w = w.astype(np.float32)
                dt = DTYPE_F32
            data, shape = w.ctypes.data, w.shape
        assert len(shape) <= 4, name
        nm = name.encode()
        keep += [w, nm]
        arr[i].name, arr[i].dtype, arr[i].ndim, arr[i].data = nm, dt, len(shape), data
        for j, s in enumerate(shape):
            arr[i].shape[j] = s
    return arr, keep
