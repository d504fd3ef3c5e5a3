"""Host-side mirror of `Encodec` (Sources/MLXAudioCodecs/Encodec/Encodec.swift:170-461) behind AudioCodecModel (encode and
decode) (Sources/MLXAudioCodecs/AudioCodecModel.swift:4-27), over the C ABI."""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import _ffi


@dataclass
class EncodecConfig:
    """EncodecConfig.swift:116-141 (snake_case keys of config.json, same defaults)."""
    audio_channels: int = 1
    num_filters: int = 32
    kernel_size: int = 7
    num_residual_layers: int = 1
    dilation_growth_rate: int = 2
    codebook_size: int = 1024
    codebook_dim: int = 128
    hidden_size: int = 128
    num_lstm_layers: int = 2
    residual_kernel_size: int = 3
    use_causal_conv: bool = True
    normalize: bool = False
    pad_mode: str = "reflect"
    norm_type: str = "weight_norm"
    last_kernel_size: int = 7
    trim_right_ratio: float = 1.0
    compress: int = 2
    upsampling_ratios: List[int] = field(default_factory=lambda: [8, 5, 4, 2])
    target_bandwidths: List[float] = field(default_factory=lambda: [1.5, 3.0, 6.0, 12.0, 24.0])
    sampling_rate: int = 24000
    chunk_length_s: Optional[float] = None
    overlap: Optional[float] = None
    use_conv_shortcut: bool = True

    @classmethod
    def from_dict(cls, d: dict) -> "EncodecConfig":
        return cls(**{k: v for k, v in d.items() if k in cls.__dataclass_fields__})


@dataclass
class EncodecEncodedAudio:
    """Encodec.swift:436-445: decode needs both codes [n_chunks, B, n_q, T] and per-chunk scales."""
    codes: np.ndarray
    scales: Optional[Sequence] = None


class Encodec:
    def __init__(self, config: EncodecConfig, *, weights: Dict[str, np.ndarray], device: int = 0):
        self.config = config
        c = _ffi.EncodecConfig()
        for name in ("audio_channels", "num_filters", "kernel_size", "num_residual_layers", "dilation_growth_rate", "codebook_size",
                     "codebook_dim", "hidden_size", "num_lstm_layers", "residual_kernel_size", "last_kernel_size", "compress",
                     "sampling_rate"):
            setattr(c, name, int(getattr(config, name)))
        c.use_causal_conv, c.use_conv_shortcut = int(config.use_causal_conv), int(config.use_conv_shortcut)
        c.pad_mode_reflect = int(config.pad_mode == "reflect")
        c.norm_type = {"weight_norm": 0, "time_group_norm": 1}.get(config.norm_type, 2)    # 2: the library's invalidInput
        c.n_upsampling_ratios = len(config.upsampling_ratios)
        for i, r in enumerate(config.upsampling_ratios[:8]):
            c.upsampling_ratios[i] = int(r)
        c.trim_right_ratio = float(config.trim_right_ratio)
        c.chunk_length_s = float(config.chunk_length_s) if config.chunk_length_s is not None else 0.0
        c.overlap = float(config.overlap) if config.overlap is not None else -1.0
        c.normalize = int(config.normalize)
        table, keep = _ffi.make_tensor_table(weights)
        self._h = C.c_void_p()
        _ffi.check(_ffi.lib().b2a_encodec_create(device, C.byref(c), table, len(weights), C.byref(self._h)))
        del keep

    @classmethod
    def from_model_directory(cls, model_dir, device: int = 0) -> "Encodec":
        """fromModelDirectory (Encodec.swift:423-440): config.json + model.safetensors, keys as shipped (the library's reader).
        The mlx-community layout is the library's own: ``*.conv.weight [out, k, in]`` and, for time_group_norm checkpoints such
        as encodec-48khz, ``*.norm.weight`` / ``*.norm.bias [C_out]`` after every conv."""
        import json
        from pathlib import Path
        from .loading import Weights
        model_dir = Path(model_dir)
        config = EncodecConfig.from_dict(json.loads((model_dir / "config.json").read_text()))
        w = Weights(model_dir / "model.safetensors")
        tensors = w.tensors()
        w.close()
        return cls(config, weights=tensors, device=device)

    # ---- properties of the reference class (Encodec.swift:186-208)
    @property
    def channels(self) -> int:
        return self.config.audio_channels

    @property
    def sampling_rate(self) -> int:
        return self.config.sampling_rate

    @property
    def codec_sample_rate(self) -> float:
        return float(self.config.sampling_rate)

    @property
    def chunk_length(self) -> Optional[int]:
        c = self.config
        return None if c.chunk_length_s is None else int(c.chunk_length_s * c.sampling_rate)

    @property
    def chunk_stride(self) -> Optional[int]:
        c = self.config
        if c.chunk_length_s is None or c.overlap is None:
            return None
        return max(1, int((1.0 - c.overlap) * self.chunk_length))

    @property
    def num_codebooks(self) -> int:
        return int(_ffi.lib().b2a_encodec_num_codebooks(self._h))

    @property
    def stream(self) -> int:
        return int(_ffi.lib().b2a_encodec_stream(self._h) or 0)

    @staticmethod
    def random_init_weights(config: EncodecConfig, seed: int = 1234, n_codebooks: int = 8, encoder: bool = False) -> Dict[str, np.ndarray]:
        """Random-init weights with the checkpoint's keys / MLX layouts (benchmarks): U(+-1/sqrt(fan_in)), N(0,1) codebooks.
        encoder=True appends the encoder's weights (drawn after everything else, so the decoder / codebooks do not change).
        time_group_norm adds every conv's ``norm.weight`` / ``norm.bias`` from a generator of their own (the other tensors are
        those of the same config under weight_norm), gamma = +-U(0.5, 1.5) and beta = +-U(0.1, 0.5): away from 1 and 0, so a
        dropped or swapped affine shows."""
        rng = np.random.default_rng(seed)
        nrng = np.random.default_rng([seed, 1])
        w: Dict[str, np.ndarray] = {}
        gn = config.norm_type == "time_group_norm"

        def u(shape, fan):
            s = (1.0 / fan) ** 0.5
            return rng.uniform(-s, s, size=shape).astype(np.float32)

        def conv(pre, cout, k, cin):
            w[pre + "conv.weight"] = u((cout, k, cin), k * cin)
            w[pre + "conv.bias"] = u((cout,), k * cin)
            if gn:
                sign = np.where(nrng.random(cout) < 0.5, -1.0, 1.0)
                w[pre + "norm.weight"] = (sign * nrng.uniform(0.5, 1.5, cout)).astype(np.float32)
                w[pre + "norm.bias"] = (np.where(nrng.random(cout) < 0.5, -1.0, 1.0) * nrng.uniform(0.1, 0.5, cout)).astype(np.float32)

        for q in range(n_codebooks):
            w[f"quantizer.layers.{q}.codebook.embed"] = rng.standard_normal((config.codebook_size, config.codebook_dim)).astype(np.float32)
        scaling = 2 ** len(config.upsampling_ratios)
        i = 0
        d0 = scaling * config.num_filters
        conv(f"decoder.layers.{i}.", d0, config.kernel_size, config.hidden_size); i += 1
        for l in range(config.num_lstm_layers):
            for n, shape in (("Wx", (4 * d0, d0)), ("Wh", (4 * d0, d0)), ("bias", (4 * d0,))):
                w[f"decoder.layers.{i}.lstm.{l}.{n}"] = u(shape, d0)
        i += 1
        for ratio in config.upsampling_ratios:
            cur = scaling * config.num_filters
            i += 1
            conv(f"decoder.layers.{i}.", cur // 2, 2 * ratio, cur); i += 1
            for _ in range(config.num_residual_layers):
                dim, hid = cur // 2, cur // 2 // config.compress
                conv(f"decoder.layers.{i}.block.1.", hid, config.residual_kernel_size, dim)
                conv(f"decoder.layers.{i}.block.3.", dim, 1, hid)
                if config.use_conv_shortcut:
                    conv(f"decoder.layers.{i}.shortcut.", dim, 1, dim)
                i += 1
            scaling //= 2
        i += 1
        conv(f"decoder.layers.{i}.", config.audio_channels, config.last_kernel_size, config.num_filters)
        if encoder:                     # EncodecEncoder's module array (Encodec.swift:20-70), ELU slots counted
            i, cur = 0, config.num_filters
            conv(f"encoder.layers.{i}.", cur, config.kernel_size, config.audio_channels); i += 1
            for ratio in reversed(config.upsampling_ratios):
                for _ in range(config.num_residual_layers):
                    hid = cur // config.compress
                    conv(f"encoder.layers.{i}.block.1.", hid, config.residual_kernel_size, cur)
                    conv(f"encoder.layers.{i}.block.3.", cur, 1, hid)
                    if config.use_conv_shortcut:
                        conv(f"encoder.layers.{i}.shortcut.", cur, 1, cur)
                    i += 1
                i += 1
                conv(f"encoder.layers.{i}.", 2 * cur, 2 * ratio, cur); i += 1
                cur *= 2
            for l in range(config.num_lstm_layers):
                for n, shape in (("Wx", (4 * cur, cur)), ("Wh", (4 * cur, cur)), ("bias", (4 * cur,))):
                    w[f"encoder.layers.{i}.lstm.{l}.{n}"] = u(shape, cur)
            i += 2
            conv(f"encoder.layers.{i}.", config.hidden_size, config.last_kernel_size, cur)
        return w

    def output_length(self, n_chunks: int, frames: int) -> int:
        return int(_ffi.lib().b2a_encodec_output_length(self._h, n_chunks, frames))

    def decode(self, audio_codes, audio_scales: Optional[Sequence] = None, padding_mask=None) -> np.ndarray:
        """decode(_:_:paddingMask:) (Encodec.swift:366-402): [n_chunks, B, n_q, T] codes -> [B, samples, channels]."""
        codes = np.ascontiguousarray(audio_codes, dtype=np.int32)
        if codes.ndim != 4:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "audio_codes must be [n_chunks, B, n_q, T]")
        nc, B, nq, T = codes.shape
        scales = None
        if audio_scales is not None and any(s is not None for s in audio_scales):
            scales = np.ones((nc, B), dtype=np.float32)
            for i, s in enumerate(audio_scales):
                if s is not None:
                    scales[i, :] = np.asarray(s, dtype=np.float32).reshape(-1)
        n = self.output_length(nc, T) if nc and T else 0
        out = np.empty((B, n, self.config.audio_channels), dtype=np.float32)
        _ffi.check(_ffi.lib().b2a_encodec_decode(self._h, _ffi.ptr(codes), nc, B, nq, T, _ffi.ptr(scales), _ffi.ptr(out)))
        if padding_mask is not None and np.asarray(padding_mask).shape[1] < out.shape[1]:
            out = out[:, :np.asarray(padding_mask).shape[1], :]
        return out

    def decode_audio(self, encoded: EncodecEncodedAudio) -> np.ndarray:
        """AudioDecoderModel.decodeAudio (Encodec.swift:458-460)."""
        return self.decode(encoded.codes, encoded.scales, None)

    def decode_dev(self, d_codes, d_wave, d_scales=None, stream: int = 0) -> None:
        nc, B, nq, T = d_codes.shape
        _ffi.check(_ffi.lib().b2a_encodec_decode_dev(self._h, _ffi.ptr(d_codes), nc, B, nq, T, _ffi.ptr(d_scales), _ffi.ptr(d_wave),
                                                     C.c_void_p(stream)))

    # ---- encode side (Encodec.swift:212-291, 457-460)
    def num_quantizers_for_bandwidth(self, bandwidth: Optional[float]) -> int:
        """getNumQuantizersForBandwidth (EncodecQuantization.swift:90-97), in the reference's Float arithmetic."""
        c = self.config
        frame_rate = math.ceil(c.sampling_rate / int(np.prod(c.upsampling_ratios)))
        n = int(1000 * max(c.target_bandwidths) / (frame_rate * 10))
        bw_per_q = np.float32(math.log2(c.codebook_size)) * np.float32(frame_rate)
        if bandwidth is not None and bandwidth > 0.0:
            n = max(1, int(math.floor(np.float32(bandwidth) * np.float32(1000) / bw_per_q)))
        return n

    def encoded_shape(self, samples: int):
        """(n_chunks, frames) of the codes of a `samples`-long input (encode's chunk loop, Encodec.swift:267-287)."""
        nc, fr = C.c_int32(0), C.c_int32(0)
        _ffi.check(_ffi.lib().b2a_encodec_encoded_shape(self._h, int(samples), C.byref(nc), C.byref(fr)))
        return nc.value, fr.value

    def _bandwidth_codebooks(self, bandwidth: Optional[float]) -> int:
        bw = self.config.target_bandwidths[0] if bandwidth is None else bandwidth
        if bw not in self.config.target_bandwidths:       # the reference's fatalError (Encodec.swift:253-255)
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT,
                                            f"This model doesn't support bandwidth {bw}. Select one of {self.config.target_bandwidths}")
        return self.num_quantizers_for_bandwidth(bw)

    def _check_audio_shape(self, shape) -> None:
        if len(shape) != 3 or shape[2] != self.config.audio_channels:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT,
                                            f"expected audio [B, samples, {self.config.audio_channels}], got {tuple(shape)}")

    def encode(self, input_values, padding_mask=None, bandwidth: Optional[float] = None):
        """encode(_:paddingMask:bandwidth:) (Encodec.swift:245-291): [B, samples, channels] -> (codes [n_chunks, B, n_q, frames]
        int32, scales: per chunk a [B] float32 array with normalize, else None)."""
        x = np.ascontiguousarray(input_values, dtype=np.float32)
        self._check_audio_shape(x.shape)
        nq = self._bandwidth_codebooks(bandwidth)
        if padding_mask is not None and self.config.normalize:    # only ever `values * mask` ahead of the normalisation (:224-226)
            x = np.ascontiguousarray(x * np.asarray(padding_mask, dtype=np.float32).reshape(x.shape[0], x.shape[1], 1))
        B, n, _ = x.shape
        nc, T = self.encoded_shape(n)
        codes = np.empty((nc, B, nq, T), dtype=np.int32)
        scales = np.empty((nc, B), dtype=np.float32) if self.config.normalize else None
        _ffi.check(_ffi.lib().b2a_encodec_encode(self._h, _ffi.ptr(x), B, n, nq, _ffi.ptr(codes), _ffi.ptr(scales)))
        return codes, ([scales[i] for i in range(nc)] if scales is not None else [None] * nc)

    def encode_audio(self, waveform) -> EncodecEncodedAudio:
        """AudioCodecModel.encodeAudio (Encodec.swift:457-460): default bandwidth, no padding mask."""
        codes, scales = self.encode(waveform)
        return EncodecEncodedAudio(codes, scales)

    def reconstruct(self, waveform) -> np.ndarray:
        """AudioCodecModel.reconstruct: decodeAudio(encodeAudio(x))."""
        return self.decode_audio(self.encode_audio(waveform))

    def encode_dev(self, d_audio, d_codes, d_scales=None, stream: int = 0, bandwidth: Optional[float] = None) -> None:
        """Device-resident encode: torch CUDA float32 d_audio [B, samples, channels] -> int32 d_codes [n_chunks, B, n_q, frames]
        (+ float32 d_scales [n_chunks, B] with normalize), enqueued on `stream`.  n_q follows `bandwidth` as in encode."""
        import torch
        if not isinstance(d_audio, torch.Tensor):
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "d_audio must be a CUDA tensor")
        self._check_audio_shape(tuple(d_audio.shape))
        B, n, ch = d_audio.shape
        self._check_dev(d_audio, "float32", (B, n, ch), "d_audio")
        nq = self._bandwidth_codebooks(bandwidth)
        nc, T = self.encoded_shape(n)
        self._check_dev(d_codes, "int32", (nc, B, nq, T), "d_codes")
        if d_scales is not None:
            self._check_dev(d_scales, "float32", (nc, B), "d_scales")
        _ffi.check(_ffi.lib().b2a_encodec_encode_dev(self._h, _ffi.ptr(d_audio), B, n, nq, _ffi.ptr(d_codes), _ffi.ptr(d_scales),
                                                     C.c_void_p(stream)))

    @staticmethod
    def _check_dev(t, dtype: str, shape, what: str) -> None:
        # the library reads / writes exactly these extents through raw device pointers: anything else is an input error, not a fault
        import torch
        ok = (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == getattr(torch, dtype) and t.is_contiguous()
              and tuple(t.shape) == tuple(shape))
        if not ok:
            got = tuple(t.shape) if hasattr(t, "shape") else type(t).__name__
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, f"{what}: expected a contiguous CUDA {dtype} tensor {tuple(shape)}, got {got}")

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                _ffi.lib().b2a_encodec_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass
