"""Host-side mirror of `SNAC` (Sources/MLXAudioCodecs/SNAC/SNACDecoder.swift:12-204) behind the
AudioCodecModel protocol (encode and decode) (Sources/MLXAudioCodecs/AudioCodecModel.swift:4-27), over the C ABI."""
from __future__ import annotations

import ctypes as C
import json
from pathlib import Path
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import _ffi


class SNAC:
    def __init__(self, sampling_rate: int = 24000, encoder_dim: int = 48, encoder_rates: Sequence[int] = (2, 4, 8, 8),
                 latent_dim: Optional[int] = None, decoder_dim: int = 1024, decoder_rates: Sequence[int] = (8, 8, 4, 2),
                 attn_window_size: Optional[int] = None, codebook_size: int = 4096, codebook_dim: int = 8,
                 vq_strides: Sequence[int] = (4, 2, 1), noise: bool = True, depthwise: bool = True, *,
                 weights: Dict[str, np.ndarray], device: int = 0):
        cfg = _ffi.SnacConfig()
        cfg.sampling_rate, cfg.encoder_dim = sampling_rate, encoder_dim
        cfg.n_encoder_rates = len(encoder_rates)
        for i, r in enumerate(encoder_rates):
            cfg.encoder_rates[i] = r
        cfg.latent_dim = latent_dim or 0
        cfg.decoder_dim, cfg.n_decoder_rates = decoder_dim, len(decoder_rates)
        for i, r in enumerate(decoder_rates):
            cfg.decoder_rates[i] = r
        cfg.attn_window_size = attn_window_size or 0
        cfg.codebook_size, cfg.codebook_dim, cfg.n_vq_strides = codebook_size, codebook_dim, len(vq_strides)
        for i, r in enumerate(vq_strides):
            cfg.vq_strides[i] = r
        cfg.noise, cfg.depthwise = int(noise), int(depthwise)
        self.sampling_rate, self.vq_strides, self.decoder_rates = sampling_rate, tuple(vq_strides), tuple(decoder_rates)
        self.latent_dim = latent_dim or encoder_dim * 2 ** len(encoder_rates)
        self.n_codebooks = len(vq_strides)
        table, keep = _ffi.make_tensor_table(weights)
        self._h = C.c_void_p()
        _ffi.check(_ffi.lib().b2a_snac_create(device, C.byref(cfg), table, len(weights), C.byref(self._h)))
        del keep
        self.hop_length = int(_ffi.lib().b2a_snac_hop_length(self._h))
        self.attn_window_size = attn_window_size or 0

    def decoded_length(self, t_latent: int) -> int:
        """Samples decoded from t_latent frames: t_latent * hop_length, less one frame per odd-stride decoder stage (the reference
        drops DecoderBlock's outputPadding), e.g. 384 t_latent - 2 for the 32 / 44 kHz models."""
        return int(_ffi.lib().b2a_snac_decoded_length(self._h, t_latent))

    @staticmethod
    def random_init_weights(seed: int = 1234, latent: int = 768, decoder_dim: int = 1024,
                            decoder_rates: Sequence[int] = (8, 8, 4, 2), vq_strides: Sequence[int] = (4, 2, 1),
                            codebook_size: int = 4096, codebook_dim: int = 8, encoder: bool = False, encoder_dim: int = 48,
                            encoder_rates: Sequence[int] = (2, 4, 8, 8), attn_window_size: Optional[int] = None) -> Dict[str, np.ndarray]:
        """Random-init snac_24khz-shaped weights (benchmarks): conv v ~ U(+-1/sqrt(fan_in)) as
        Layers.swift:81-86, g = ||v||, zero biases, Snake alpha = 1.  encoder=True appends the encoder's
        weights (drawn after everything else, so the decoder / quantizer weights do not change).
        attn_window_size adds the 32 / 44 kHz models' LocalMHA blocks (decoder.model.layers.2 and, with the encoder,
        encoder.block.layers.{n+1}), drawn from a generator of their own (seed + 1), so every other tensor is unchanged."""
        rng = np.random.default_rng(seed)
        w: Dict[str, np.ndarray] = {}

        def wn(prefix, shape, fan, bias_n):
            s = (1.0 / fan) ** 0.5
            v = rng.uniform(-s, s, size=shape).astype(np.float32)
            w[prefix + ".weight_v"] = v
            w[prefix + ".weight_g"] = np.sqrt((v.astype(np.float64) ** 2).sum(axis=(1, 2), keepdims=True)).astype(np.float32)
            if bias_n:
                w[prefix + ".bias"] = np.zeros(bias_n, dtype=np.float32)

        for i in range(len(vq_strides)):
            q = f"quantizer.quantizers.{i}"
            wn(q + ".in_proj", (codebook_dim, 1, latent), latent, codebook_dim)
            wn(q + ".out_proj", (latent, 1, codebook_dim), codebook_dim, latent)
            w[q + ".codebook.weight"] = rng.standard_normal((codebook_size, codebook_dim)).astype(np.float32)
        arng = np.random.default_rng(seed + 1)

        def attn(prefix, dim):       # LocalMHA (Attention.swift:14-95): LayerNorm, to_qkv / to_out without bias, rotary inv_freq
            s = (1.0 / dim) ** 0.5
            w[prefix + ".norm.weight"] = np.ones(dim, dtype=np.float32)
            w[prefix + ".norm.bias"] = np.zeros(dim, dtype=np.float32)
            w[prefix + ".to_qkv.weight"] = arng.uniform(-s, s, size=(3 * dim, dim)).astype(np.float32)
            w[prefix + ".to_out.weight"] = arng.uniform(-s, s, size=(dim, dim)).astype(np.float32)
            w[prefix + ".rel_pos.inv_freq"] = (1.0 / 10000.0 ** (np.arange(0, 64, 2) / 64.0)).astype(np.float32)

        p = "decoder.model.layers"
        wn(f"{p}.0", (latent, 7, 1), 7 * latent, latent)
        wn(f"{p}.1", (decoder_dim, 1, latent), latent, decoder_dim)
        li = 2
        if attn_window_size:
            attn(f"{p}.2", decoder_dim)
            li = 3
        for i, s in enumerate(decoder_rates):
            cin, cout = decoder_dim // 2 ** i, decoder_dim // 2 ** (i + 1)
            b = f"{p}.{li}.block.layers"
            w[f"{b}.0.alpha"] = np.ones((1, cin, 1), dtype=np.float32)
            wn(f"{b}.1", (cin, 2 * s, cout), cin * 2 * s, cout)
            wn(f"{b}.2.linear", (cout, 1, cout), cout, 0)
            for j in (3, 4, 5):
                r = f"{b}.{j}.block.layers"
                w[f"{r}.0.alpha"] = np.ones((1, cout, 1), dtype=np.float32)
                wn(f"{r}.1", (cout, 7, 1), cout * 7, cout)
                w[f"{r}.2.alpha"] = np.ones((1, cout, 1), dtype=np.float32)
                wn(f"{r}.3", (cout, 1, cout), cout, cout)
            li += 1
        cf = decoder_dim // 2 ** len(decoder_rates)
        w[f"{p}.{li}.alpha"] = np.ones((1, cf, 1), dtype=np.float32)
        wn(f"{p}.{li + 1}", (1, 7, cf), cf * 7, 1)
        if encoder:
            p, d = "encoder.block.layers", encoder_dim
            wn(f"{p}.0", (d, 7, 1), 7, d)
            for i, s in enumerate(encoder_rates):
                b = f"{p}.{i + 1}.block.layers"
                for j in range(3):
                    r = f"{b}.{j}.block.layers"
                    w[f"{r}.0.alpha"] = np.ones((1, d, 1), dtype=np.float32)
                    wn(f"{r}.1", (d, 7, 1), 7, d)
                    w[f"{r}.2.alpha"] = np.ones((1, d, 1), dtype=np.float32)
                    wn(f"{r}.3", (d, 1, d), d, d)
                w[f"{b}.3.alpha"] = np.ones((1, d, 1), dtype=np.float32)
                wn(f"{b}.4", (2 * d, 2 * s, d), 2 * s * d, 2 * d)
                d *= 2
            if attn_window_size:
                attn(f"{p}.{len(encoder_rates) + 1}", d)
            wn(f"{p}.{len(encoder_rates) + 1 + bool(attn_window_size)}", (d, 7, 1), 7, d)
        return w

    # -- loading (SNACDecoder.swift:135-189) ------------------------------------------------------
    @classmethod
    def from_config_dict(cls, cfg: dict, weights, device: int = 0) -> "SNAC":
        return cls(cfg["sampling_rate"], cfg["encoder_dim"], cfg["encoder_rates"], cfg.get("latent_dim"),
                   cfg["decoder_dim"], cfg["decoder_rates"], cfg.get("attn_window_size"), cfg["codebook_size"],
                   cfg["codebook_dim"], cfg["vq_strides"], cfg["noise"], cfg["depthwise"], weights=weights, device=device)

    @classmethod
    def from_model_directory(cls, model_dir, device: int = 0) -> "SNAC":
        model_dir = Path(model_dir)
        wpath = model_dir / "model.safetensors"
        if not wpath.exists():
            raise FileNotFoundError(f"Could not find model at {wpath}")   # SNACError.modelNotFound
        from safetensors.numpy import load_file
        cfg = json.loads((model_dir / "config.json").read_text())
        return cls.from_config_dict(cfg, load_file(str(wpath)), device)

    @property
    def stream(self) -> int:
        return int(_ffi.lib().b2a_snac_stream(self._h) or 0)

    # -- AudioCodecModel ------------------------------------------------------------------------
    @property
    def codec_sample_rate(self) -> float:
        return float(self.sampling_rate)

    def decode(self, codes: List[np.ndarray], noise: Optional[List[Optional[np.ndarray]]] = None,
               zero_noise: bool = False, seed: int = 0, out: Optional[np.ndarray] = None) -> np.ndarray:
        """SNAC.decode (:127-131): codes[i] [B, T_i] int -> waveform [B, 1, decoded_length(T)] float32.
        `noise[i]` supplies NoiseBlock i's Gaussian draw explicitly (SURVEY.md F6), [B, 1, length of stage i's output]."""
        cs = [np.ascontiguousarray(c, dtype=np.int32) for c in codes]
        if len(cs) != self.n_codebooks:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, f"expected {self.n_codebooks} code layers")
        B = cs[0].shape[0]
        T = cs[0].shape[1] * self.vq_strides[0]
        for c, s in zip(cs, self.vq_strides):
            if c.shape != (B, T // s):
                raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "code layer shapes do not match vq_strides")
        cp = (C.c_void_p * len(cs))(*[c.ctypes.data for c in cs])
        nz, np_ = None, None
        if noise is not None:
            nz = [None if n is None else np.ascontiguousarray(n, dtype=np.float32) for n in noise]
            np_ = (C.c_void_p * len(self.decoder_rates))(*[None if n is None else n.ctypes.data for n in nz])
        n_out = self.decoded_length(T)
        wave = out if out is not None else np.empty((B, 1, n_out), dtype=np.float32)   # `out`: a caller-owned (e.g. pinned) buffer
        assert wave.shape == (B, 1, n_out) and wave.dtype == np.float32 and wave.flags["C_CONTIGUOUS"]
        _ffi.check(_ffi.lib().b2a_snac_decode(self._h, cp, B, T, np_, int(zero_noise), seed, _ffi.ptr(wave)))
        return wave

    def decode_audio(self, codes):            # AudioDecoderModel.decodeAudio (:199)
        return self.decode(codes)

    @staticmethod
    def _check_dev(t, dtype: str, shape, what: str) -> None:
        # the library reads / writes exactly these extents through raw device pointers: anything else is an input error, not a fault
        import torch
        ok = (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == getattr(torch, dtype) and t.is_contiguous()
              and tuple(t.shape) == tuple(shape))
        if not ok:
            got = tuple(t.shape) if hasattr(t, "shape") else type(t).__name__
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, f"{what}: expected a contiguous CUDA {dtype} tensor {tuple(shape)}, got {got}")

    def _check_code_list(self, d_codes, B: int, T: int) -> None:
        if len(d_codes) != self.n_codebooks:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, f"expected {self.n_codebooks} code layers")
        for i, (c, s) in enumerate(zip(d_codes, self.vq_strides)):
            self._check_dev(c, "int32", (B, T // s), f"code layer {i}")

    def decode_dev(self, d_codes, d_wave, zero_noise: bool = False, seed: int = 0, stream: int = 0) -> None:
        """Device-resident decode: torch CUDA int32 tensors [B, T_i] -> d_wave [B, 1, decoded_length(T)]."""
        if len(d_codes) != self.n_codebooks or d_codes[0].dim() != 2:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, f"expected {self.n_codebooks} code layers [B, T_i]")
        B = d_codes[0].shape[0]
        T = d_codes[0].shape[1] * self.vq_strides[0]
        self._check_code_list(d_codes, B, T)
        n_wave = self.decoded_length(T)
        n_out = B * n_wave                       # any contiguous layout of [B, 1, decoded_length(T)], as before
        self._check_dev(d_wave, "float32", tuple(d_wave.shape) if getattr(d_wave, "numel", lambda: -1)() == n_out else (B, 1, n_wave), "d_wave")
        cp = (C.c_void_p * len(d_codes))(*[c.data_ptr() for c in d_codes])
        _ffi.check(_ffi.lib().b2a_snac_decode_dev(self._h, cp, B, T, None, int(zero_noise), seed, _ffi.ptr(d_wave),
                                                  C.c_void_p(stream)))

    def quantize(self, z: np.ndarray):
        """ResidualVectorQuantize.callAsFunction (VQ.swift:150-163): z [B, D, T] -> (z_q, [codes_i])."""
        z = np.ascontiguousarray(z, dtype=np.float32)
        B, D, T = z.shape
        codes = [np.empty((B, T // s), dtype=np.int32) for s in self.vq_strides]
        cp = (C.c_void_p * len(codes))(*[c.ctypes.data for c in codes])
        zq = np.empty_like(z)
        _ffi.check(_ffi.lib().b2a_snac_quantize(self._h, _ffi.ptr(z), B, T, cp, _ffi.ptr(zq)))
        return zq, codes

    def encoded_length(self, n_samples: int) -> int:
        """Latent steps of an n-sample clip after preprocess's padding (SNACDecoder.swift:86-105); 0 without encoder weights."""
        return int(_ffi.lib().b2a_snac_encoded_length(self._h, n_samples))

    def encode(self, wave) -> List[np.ndarray]:
        """SNAC.encode (:120-125): waveform [B, 1, n] (or [B, n]) float -> [codes_i [B, t_latent / stride_i] int32]."""
        w = np.ascontiguousarray(wave, dtype=np.float32)
        if w.ndim == 3:
            if w.shape[1] != 1:
                raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "SNAC encodes mono audio [B, 1, n]")
            w = w[:, 0]
        if w.ndim != 2:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "expected a waveform [B, 1, n]")
        B, n = w.shape
        w = np.ascontiguousarray(w)
        T = self.encoded_length(n)
        codes = [np.empty((B, T // s), dtype=np.int32) for s in self.vq_strides]
        cp = (C.c_void_p * len(codes))(*[c.ctypes.data for c in codes])
        _ffi.check(_ffi.lib().b2a_snac_encode(self._h, _ffi.ptr(w), B, n, cp))
        return codes

    def encode_audio(self, wave) -> List[np.ndarray]:        # AudioCodecModel.encodeAudio (:197-199)
        return self.encode(wave)

    def encode_dev(self, d_wave, d_codes, stream: int = 0) -> None:
        """Device-resident encode: torch CUDA float32 d_wave [B, 1, n] (or [B, n]) -> int32 tensors d_codes[i]
        [B, encoded_length(n) / stride_i], enqueued on `stream`."""
        if d_wave.dim() not in (2, 3):
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "expected a waveform [B, 1, n]")
        B, n = d_wave.shape[0], d_wave.shape[-1]
        self._check_dev(d_wave, "float32", (B, 1, n) if d_wave.dim() == 3 else (B, n), "d_wave")
        T = self.encoded_length(n)
        if len(d_codes) != self.n_codebooks:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, f"expected {self.n_codebooks} code layers")
        if T > 0:          # T == 0: no encoder weights or no samples -- the library reports which
            self._check_code_list(d_codes, B, T)
        cp = (C.c_void_p * len(d_codes))(*[c.data_ptr() for c in d_codes])
        _ffi.check(_ffi.lib().b2a_snac_encode_dev(self._h, _ffi.ptr(d_wave), B, n, cp, C.c_void_p(stream)))

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                _ffi.lib().b2a_snac_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:   # interpreter shutdown: ctypes globals may already be gone
            pass
