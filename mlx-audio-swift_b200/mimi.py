"""Host-side mirror of `Mimi` and `MimiStreamingDecoder` (Sources/MLXAudioCodecs/Mimi/Mimi.swift) behind AudioCodecModel, over
the C ABI (b2a_mimi_*, include/b200audio.h)."""
from __future__ import annotations

import ctypes as C
from pathlib import Path
from typing import Dict, Optional, Union

import numpy as np

from . import _ffi

DEFAULT_MAX_CACHE_FRAMES = 2250          # code frames one stream may decode before a reset: 3 minutes at 12.5 Hz


class Mimi:
    """Mimi(cfg: mimi_202407(numCodebooks:)) with its weights (MLX layouts, Mimi.sanitize's names).  Config fields of
    b2a_mimi_config may be overridden by keyword (the tests' small geometry)."""

    def __init__(self, weights: Optional[Dict[str, np.ndarray]] = None, num_codebooks: int = 32, *, device: int = 0, max_batch: int = 8,
                 max_cache_frames: int = DEFAULT_MAX_CACHE_FRAMES, _handle: Optional[C.c_void_p] = None, **config):
        self._h = C.c_void_p()
        if _handle is not None:
            self._h = _handle
        else:
            cfg = _ffi.MimiConfig()
            _ffi.check(_ffi.lib().b2a_mimi_config_default(num_codebooks, max_batch, max_cache_frames, C.byref(cfg)))
            for k, v in config.items():
                if k == "ratios":
                    cfg.num_ratios = len(v)
                    for j, r in enumerate(v):
                        cfg.ratios[j] = r
                else:
                    if not hasattr(cfg, k):
                        raise TypeError(f"unknown Mimi config field {k!r}")
                    setattr(cfg, k, v)
            table, keep = _ffi.make_tensor_table(weights or {})
            _ffi.check(_ffi.lib().b2a_mimi_create(device, C.byref(cfg), table, len(weights or {}), C.byref(self._h)))
            del keep
        self.num_codebooks = int(_ffi.lib().b2a_mimi_num_codebooks(self._h))
        self.samples_per_frame = int(_ffi.lib().b2a_mimi_samples_per_frame(self._h))

    @classmethod
    def from_file(cls, path: Union[str, Path], num_codebooks: int = 32, *, device: int = 0, max_batch: int = 8,
                  max_cache_frames: int = DEFAULT_MAX_CACHE_FRAMES) -> "Mimi":
        """Mimi.fromPretrained on a local checkpoint file: mimi_202407(num_codebooks), sanitize, load."""
        h = C.c_void_p()
        _ffi.check(_ffi.lib().b2a_mimi_create_from_file(str(path).encode(), num_codebooks, device, max_batch, max_cache_frames, C.byref(h)))
        return cls(_handle=h)

    # AudioCodecModel
    sample_rate = 24000.0
    frame_rate = 12.5

    @property
    def codec_sample_rate(self) -> float:
        return self.sample_rate

    @property
    def stream(self) -> int:
        return int(_ffi.lib().b2a_mimi_stream(self._h) or 0)

    def encoded_length(self, n_samples: int) -> int:
        return int(_ffi.lib().b2a_mimi_encoded_length(self._h, n_samples))

    def encode(self, audio) -> np.ndarray:
        """[B, 1, n] (or [n]) float32 at 24 kHz -> codes [B, num_codebooks, T] int32."""
        x = np.ascontiguousarray(audio, dtype=np.float32)
        x = x.reshape(1, -1) if x.ndim == 1 else x.reshape(x.shape[0], -1)
        B, n = x.shape
        out = np.empty((B, self.num_codebooks, max(self.encoded_length(n), 0)), np.int32)
        _ffi.check(_ffi.lib().b2a_mimi_encode(self._h, _ffi.ptr(x), B, n, _ffi.ptr(out)))
        return out

    def encode_audio(self, audio) -> np.ndarray:
        return self.encode(audio)

    @staticmethod
    def _codes(codes) -> np.ndarray:
        c = np.ascontiguousarray(codes, dtype=np.int32)
        return c[None] if c.ndim == 2 else c

    def _call(self, fn, codes) -> np.ndarray:
        c = self._codes(codes)
        B, K, T = c.shape
        out = np.empty((B, 1, T * self.samples_per_frame), np.float32)
        _ffi.check(fn(self._h, _ffi.ptr(c), B, K, T, _ffi.ptr(out)))
        return out

    def decode(self, codes) -> np.ndarray:
        """codes [B, K, T], 1 <= K <= num_codebooks -> [B, 1, T * 1920].  A reset followed by one streaming step."""
        return self._call(_ffi.lib().b2a_mimi_decode, codes)

    def decode_audio(self, codes) -> np.ndarray:
        return self.decode(codes)

    def reconstruct(self, audio) -> np.ndarray:
        return self.decode(self.encode(audio))

    def decode_step(self, codes) -> np.ndarray:
        """Mimi.decodeStep: the next T code frames of the current stream -> their samples."""
        return self._call(_ffi.lib().b2a_mimi_decode_step, codes)

    def decode_step_dev(self, d_codes, d_wave, stream: int = 0) -> None:
        B, K, T = d_codes.shape
        _ffi.check(_ffi.lib().b2a_mimi_decode_step_dev(self._h, _ffi.ptr(d_codes), B, K, T, _ffi.ptr(d_wave), C.c_void_p(stream)))

    def decode_dev(self, d_codes, d_wave, stream: int = 0) -> None:
        B, K, T = d_codes.shape
        _ffi.check(_ffi.lib().b2a_mimi_decode_dev(self._h, _ffi.ptr(d_codes), B, K, T, _ffi.ptr(d_wave), C.c_void_p(stream)))

    def encode_dev(self, d_audio, d_codes, stream: int = 0) -> None:
        B, n = d_audio.shape[0], d_audio.shape[-1]
        _ffi.check(_ffi.lib().b2a_mimi_encode_dev(self._h, _ffi.ptr(d_audio), B, n, _ffi.ptr(d_codes), C.c_void_p(stream)))

    def reset(self) -> None:
        _ffi.check(_ffi.lib().b2a_mimi_reset(self._h))

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                _ffi.lib().b2a_mimi_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass


class MimiStreamingDecoder:
    """MimiStreamingDecoder(mimi): reset() and decode_frames(tokens), [K, T] or [B, K, T] -> [B, 1, T * 1920]."""

    def __init__(self, mimi: Mimi):
        self.mimi = mimi
        self.reset()

    def reset(self) -> None:
        self.mimi.reset()

    def decode_frames(self, tokens) -> np.ndarray:
        return self.mimi._call(_ffi.lib().b2a_mimi_decode_frames, tokens)
