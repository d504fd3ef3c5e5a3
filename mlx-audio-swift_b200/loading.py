"""Weight / format plumbing over the C ABI (SURVEY.md 8f row N4): safetensors directories, the reference's `sanitize` key maps and
the MLX affine de-quantisation all run in C++ inside libb200audio (csrc/weights.cu); this module is the thin host mirror of
`MLX.loadArrays` / `WhisperModel.sanitize` / `LlamaTTSModel.sanitize` (file:line in include/b200audio.h)."""
from __future__ import annotations

import ctypes as C
from pathlib import Path
from typing import Dict, Union

import numpy as np

from . import _ffi

FORMAT_HUGGING_FACE, FORMAT_MLX_WHISPER = 0, 1


class Weights:
    """An open checkpoint (one .safetensors file or every *.safetensors of a directory; later files win)."""

    def __init__(self, path: Union[str, Path]):
        self._h = C.c_void_p()
        _ffi.check(_ffi.lib().b2a_weights_load(str(path).encode(), C.byref(self._h)))

    def __len__(self) -> int:
        return int(_ffi.lib().b2a_weights_count(self._h))

    def sanitize_whisper(self) -> int:
        """WhisperModel.sanitize (WhisperModel.swift:328-333); returns the detected format."""
        fmt = C.c_int32(0)
        _ffi.check(_ffi.lib().b2a_weights_sanitize_whisper(self._h, C.byref(fmt)))
        return int(fmt.value)

    def sanitize_llama(self, tie_word_embeddings: bool = True, group_size: int = 0, bits: int = 0) -> None:
        """LlamaTTSModel.sanitize (LlamaTTS.swift:583-593) + MLX affine de-quantisation to bf16 when bits > 0."""
        _ffi.check(_ffi.lib().b2a_weights_sanitize_llama(self._h, int(tie_word_embeddings), group_size, bits))

    def sanitize_llama_config(self, config_path: Union[str, Path]) -> None:
        """sanitize + de-quantisation driven by config.json, per-layer "quantization" overrides included (LlamaTTS.swift:955-966)."""
        _ffi.check(_ffi.lib().b2a_weights_sanitize_llama_config(self._h, str(config_path).encode()))

    def dequantize(self, group_size: int, bits: int) -> None:
        """MLX affine de-quantisation (to bf16) of every layer with "<path>.scales" (quantised Whisper checkpoints, WhisperModel.swift:499-511)."""
        _ffi.check(_ffi.lib().b2a_weights_dequantize(self._h, group_size, bits))

    def sanitize_speech_tokenizer(self) -> None:
        """Decoder half of Qwen3TTSSpeechTokenizer.sanitize (Qwen3TTSSpeechTokenizer.swift:1094-1440); keys end up relative to the decoder."""
        _ffi.check(_ffi.lib().b2a_weights_sanitize_speech_tokenizer(self._h))

    def sanitize_speech_tokenizer_encoder(self) -> None:
        """Encoder half of Qwen3TTSSpeechTokenizer.sanitize (:1093-1440); keys are the encoder's (encoder.*, encoder_transformer.*,
        downsample.*, quantizer.*) in MLX layouts, every other key dropped."""
        _ffi.check(_ffi.lib().b2a_weights_sanitize_speech_tokenizer_encoder(self._h))

    def sanitize_mimi(self) -> None:
        """Mimi.sanitize (Mimi/Mimi.swift:337-413), key for key; no key is dropped."""
        _ffi.check(_ffi.lib().b2a_weights_sanitize_mimi(self._h))

    def sanitize_qwen3_speaker_encoder(self) -> None:
        """Qwen3TTSSpeakerEncoder.sanitize (Qwen3TTSSpeakerEncoder.swift:324-354): the keys after the "speaker_encoder" component,
        3-D ".weight" tensors that fail checkArrayShapeQwen3 transposed [out, in, k] -> [out, k, in], every other key dropped."""
        _ffi.check(_ffi.lib().b2a_weights_sanitize_qwen3_speaker_encoder(self._h))

    def tensors(self) -> Dict[str, object]:
        """name -> numpy array (float32 / int32) or torch.bfloat16 tensor.  COPIES (the handle owns the mapped bytes)."""
        import torch
        out: Dict[str, object] = {}
        t = _ffi.Tensor()
        for i in range(len(self)):
            _ffi.check(_ffi.lib().b2a_weights_get(self._h, i, C.byref(t)))
            shape = tuple(int(t.shape[k]) for k in range(t.ndim))
            n = int(np.prod(shape)) if shape else 1
            if t.dtype == _ffi.DTYPE_BF16:
                raw = np.ctypeslib.as_array(C.cast(t.data, C.POINTER(C.c_int16)), shape=(n,)).copy()
                out[t.name.decode()] = torch.from_numpy(raw).view(torch.bfloat16).reshape(shape)
            else:
                ct, dt = (C.c_float, np.float32) if t.dtype == _ffi.DTYPE_F32 else (C.c_int32, np.int32)
                out[t.name.decode()] = np.ctypeslib.as_array(C.cast(t.data, C.POINTER(ct)), shape=(n,)).astype(dt).reshape(shape)
        return out

    def close(self) -> None:
        if getattr(self, "_h", None) and self._h.value:
            _ffi.lib().b2a_weights_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def llama_config_from_json(config_path: Union[str, Path], max_batch: int = 8, max_context: int = 2048):
    """config.json -> (LlamaConfig ctypes struct, quantisation group_size, bits)   (LlamaTTSConfig.swift:100-166)."""
    cfg, gs, bits = _ffi.LlamaConfig(), C.c_int32(0), C.c_int32(0)
    _ffi.check(_ffi.lib().b2a_tts_config_from_json(str(config_path).encode(), max_batch, max_context, C.byref(cfg), C.byref(gs), C.byref(bits)))
    return cfg, int(gs.value), int(bits.value)


def speech_tokenizer_config_from_json(config_path: Union[str, Path, None], max_batch: int = 1, max_cache_frames: int = 4096):
    """speech_tokenizer/config.json -> (SpeechTokenizerConfig ctypes struct, decode_upsample_rate); a missing file gives the
    defaults (Qwen3TTSConfig.swift:358-385,518-527; Qwen3TTS.swift:1246-1255)."""
    cfg, rate = _ffi.SpeechTokenizerConfig(), C.c_int32(0)
    path = b"" if config_path is None else str(config_path).encode()
    _ffi.check(_ffi.lib().b2a_speech_tokenizer_config_from_json(path, max_batch, max_cache_frames, C.byref(cfg), C.byref(rate)))
    return cfg, int(rate.value)
