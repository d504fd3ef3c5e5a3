"""Host-side mirror of the Qwen3-TTS speech tokenizer (Sources/MLXAudioTTS/Models/Qwen3TTS/Qwen3TTSSpeechTokenizer.swift:790-1092)
over the C ABI (SURVEY.md section 8f row N1): the decoder (parity tests: tests/test_gpu_qwen3_tts_codec.py) and the encoder that
turns reference audio into codes for voice cloning (tests/test_gpu_qwen3_tts_encode.py)."""
from __future__ import annotations

import ctypes as C
import re
from pathlib import Path
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import _ffi


@dataclass
class Qwen3TTSTokenizerDecoderConfig:
    """Qwen3TTSConfig.swift:358-385 (same keys, same defaults)."""
    attention_bias: bool = False
    latent_dim: int = 1024
    codebook_dim: int = 512
    codebook_size: int = 2048
    decoder_dim: int = 1536
    hidden_size: int = 512
    intermediate_size: int = 1024
    head_dim: int = 64
    num_attention_heads: int = 16
    num_hidden_layers: int = 8
    num_key_value_heads: int = 16
    num_quantizers: int = 16
    num_semantic_quantizers: int = 1
    rms_norm_eps: float = 1e-5
    rope_theta: float = 10000.0
    upsample_rates: List[int] = field(default_factory=lambda: [8, 5, 4, 3])
    upsampling_ratios: List[int] = field(default_factory=lambda: [2, 2])

    @classmethod
    def from_dict(cls, d: dict) -> "Qwen3TTSTokenizerDecoderConfig":
        known = {f for f in cls.__dataclass_fields__}
        return cls(**{k: v for k, v in d.items() if k in known})


@dataclass
class Qwen3TTSTokenizerEncoderConfig:
    """Qwen3TTSTokenizerEncoderConfig (Qwen3TTSConfig.swift:391-494: same keys, same defaults) plus the tokenizer config's
    encoder_valid_num_quantizers (:518-527)."""
    frame_rate: float = 12.5
    audio_channels: int = 1
    codebook_dim: int = 256
    codebook_size: int = 2048
    compress: int = 2
    hidden_size: int = 512
    intermediate_size: int = 2048
    kernel_size: int = 7
    last_kernel_size: int = 3
    layer_scale_initial_scale: float = 0.01
    num_attention_heads: int = 8
    num_filters: int = 64
    num_hidden_layers: int = 8
    num_key_value_heads: int = 8
    num_quantizers: int = 32
    num_residual_layers: int = 1
    residual_kernel_size: int = 3
    rope_theta: float = 10000.0
    sampling_rate: int = 24000
    sliding_window: int = 250
    upsampling_ratios: List[int] = field(default_factory=lambda: [8, 6, 5, 4])
    use_causal_conv: bool = True
    use_conv_shortcut: bool = False
    valid_num_quantizers: int = 16

    @classmethod
    def from_dict(cls, d: dict, valid_num_quantizers: int = 16) -> "Qwen3TTSTokenizerEncoderConfig":
        known = {f for f in cls.__dataclass_fields__}
        return cls(**{k: v for k, v in d.items() if k in known and k != "valid_num_quantizers"}, valid_num_quantizers=valid_num_quantizers)

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads

    @property
    def downsample_stride(self) -> int:                 # :810-812
        return max(1, int(self.sampling_rate / int(np.prod(self.upsampling_ratios)) / self.frame_rate))

    @property
    def num_code_groups(self) -> int:
        return min(self.valid_num_quantizers, self.num_quantizers)

    @classmethod
    def from_ffi(cls, c: "_ffi.SpeechTokenizerEncoderConfig") -> "Qwen3TTSTokenizerEncoderConfig":
        d = {name: getattr(c, name) for name, _ in c._fields_ if name in cls.__dataclass_fields__ and name != "upsampling_ratios"}
        d["upsampling_ratios"] = list(c.upsampling_ratios)[: c.num_upsampling_ratios]
        d["use_causal_conv"], d["use_conv_shortcut"] = bool(c.use_causal_conv), bool(c.use_conv_shortcut)
        return cls(**d)

    def to_ffi(self) -> "_ffi.SpeechTokenizerEncoderConfig":
        if len(self.upsampling_ratios) > 8:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "at most 8 upsampling ratios")
        c = _ffi.SpeechTokenizerEncoderConfig()
        for name in ("sampling_rate", "audio_channels", "num_filters", "num_residual_layers", "kernel_size", "residual_kernel_size",
                     "last_kernel_size", "compress", "hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads",
                     "num_key_value_heads", "head_dim", "codebook_size", "codebook_dim", "num_quantizers", "valid_num_quantizers"):
            setattr(c, name, int(getattr(self, name)))
        c.frame_rate, c.rope_theta = float(self.frame_rate), float(self.rope_theta)
        c.use_causal_conv, c.use_conv_shortcut = int(bool(self.use_causal_conv)), int(bool(self.use_conv_shortcut))
        c.num_upsampling_ratios = len(self.upsampling_ratios)
        for i, r in enumerate(self.upsampling_ratios):
            c.upsampling_ratios[i] = int(r)
        return c


def random_init_encoder_weights(cfg: Qwen3TTSTokenizerEncoderConfig, seed: int = 4321, layer_scale: float = 0.01) -> Dict[str, np.ndarray]:
    """Random-init encoder weights with the sanitized key set (Qwen3TTSSpeechTokenizer.sanitize's encoder paths without
    "encoder_model.") in MLX layouts: conv / linear weights N(0, 1 / fan_in), biases N(0, 0.05^2), LayerNorm gains 1 + N(0, 0.1^2)
    and biases N(0, 0.05^2), layer scales `layer_scale`, codebooks N(0, 1) sums over usages in [0.5, 2]."""
    rng = np.random.default_rng(seed)
    W: Dict[str, np.ndarray] = {}

    def rn(shape, s):
        return (rng.standard_normal(shape) * s).astype(np.float32)

    def conv(prefix, cout, k, cin, bias=True):
        W[prefix + ".weight"] = rn((cout, k, cin), 1.0 / np.sqrt(k * cin))
        if bias:
            W[prefix + ".bias"] = rn((cout,), 0.05)

    F, H = cfg.num_filters, cfg.hidden_size
    conv("encoder.init_conv1d.conv.conv", F, cfg.kernel_size, cfg.audio_channels)
    ch = F
    for i, r in enumerate(reversed(cfg.upsampling_ratios)):
        conv(f"encoder.layers.{i}.residuals.0.block.0.conv.conv", ch // cfg.compress, cfg.residual_kernel_size, ch)
        conv(f"encoder.layers.{i}.residuals.0.block.1.conv.conv", ch, 1, ch // cfg.compress)
        conv(f"encoder.layers.{i}.downsample.conv.conv", 2 * ch, 2 * r, ch)
        ch *= 2
    conv("encoder.final_conv1d.conv.conv", H, cfg.last_kernel_size, ch)
    for l in range(cfg.num_hidden_layers):
        p = f"encoder_transformer.transformer.layers.{l}."
        W[p + "self_attn.in_proj.weight"] = rn((3 * H, H), 1.0 / np.sqrt(H))
        W[p + "self_attn.out_proj.weight"] = rn((H, H), 1.0 / np.sqrt(H))
        W[p + "gating.linear1.weight"] = rn((cfg.intermediate_size, H), 1.0 / np.sqrt(H))
        W[p + "gating.linear2.weight"] = rn((H, cfg.intermediate_size), 1.0 / np.sqrt(cfg.intermediate_size))
        for n in ("norm1", "norm2"):
            W[p + n + ".weight"] = (1.0 + rn((H,), 0.1)).astype(np.float32)
            W[p + n + ".bias"] = rn((H,), 0.05)
        W[p + "layer_scale_1.scale"] = np.full(H, layer_scale, np.float32)
        W[p + "layer_scale_2.scale"] = np.full(H, layer_scale, np.float32)
    conv("downsample.conv.conv.conv", H, 2 * cfg.downsample_stride, H, bias=False)
    D = cfg.codebook_dim
    for name, n in (("rvq_first", 1), ("rvq_rest", cfg.num_quantizers - 1)):
        conv(f"quantizer.{name}.input_proj", D, 1, H, bias=False)
        conv(f"quantizer.{name}.output_proj", H, 1, D, bias=False)
        for i in range(n):
            p = f"quantizer.{name}.vq.layers.{i}.codebook"
            use = rng.uniform(0.5, 2.0, cfg.codebook_size).astype(np.float32)
            W[p + ".cluster_usage"] = use
            W[p + ".embedding_sum"] = (rn((cfg.codebook_size, D), 1.0) * use[:, None]).astype(np.float32)
    return W


def random_init_weights(cfg: "Qwen3TTSTokenizerDecoderConfig", seed: int = 1234, layer_scale: float = 0.01, out_gain: float = 0.02,
                        encoder: bool = False, encoder_config: Optional[Qwen3TTSTokenizerEncoderConfig] = None) -> Dict[str, np.ndarray]:
    """Random-init weights with the reference's key set and MLX layouts (benchmarks; there are no checkpoints here): conv / linear
    weights N(0, 1 / fan_in), biases N(0, 0.05^2), norm gains 1, SnakeBeta alpha = beta = 0.  encoder=True appends the encoder's
    weights (random_init_encoder_weights; keys prefixed "encoder_model.") after the decoder's, which stay the same draws."""
    if encoder:
        W = random_init_weights(cfg, seed, layer_scale, out_gain)
        for k, v in random_init_encoder_weights(encoder_config or Qwen3TTSTokenizerEncoderConfig(), seed + 1).items():
            W["encoder_model." + k] = v
        return W
    rng = np.random.default_rng(seed)
    W: Dict[str, np.ndarray] = {}

    def rn(shape, s):
        return (rng.standard_normal(shape) * s).astype(np.float32)

    def conv(prefix, cout, k, cin, bias=True):
        W[prefix + ".weight"] = rn((cout, k, cin), 1.0 / np.sqrt(k * cin))
        if bias:
            W[prefix + ".bias"] = rn((cout,), 0.05)

    def lin(prefix, cout, cin, bias=True):
        W[prefix + ".weight"] = rn((cout, cin), 1.0 / np.sqrt(cin))
        if bias:
            W[prefix + ".bias"] = rn((cout,), 0.05)

    def snake(prefix, c):
        W[prefix + ".alpha"] = np.zeros(c, np.float32)
        W[prefix + ".beta"] = np.zeros(c, np.float32)

    half = cfg.codebook_dim // 2
    for name, n in (("rvq_first", cfg.num_semantic_quantizers), ("rvq_rest", cfg.num_quantizers - cfg.num_semantic_quantizers)):
        for i in range(n):
            p = f"quantizer.{name}.vq.layers.{i}.codebook"
            W[p + ".cluster_usage"] = np.ones(cfg.codebook_size, np.float32)
            W[p + ".embedding_sum"] = rn((cfg.codebook_size, half), 1.0)
        conv(f"quantizer.{name}.output_proj", cfg.codebook_dim, 1, half, bias=False)
    conv("pre_conv.conv", cfg.latent_dim, 3, cfg.codebook_dim)
    H, hd = cfg.hidden_size, cfg.head_dim
    lin("pre_transformer.input_proj", H, cfg.latent_dim)
    lin("pre_transformer.output_proj", cfg.latent_dim, H)
    W["pre_transformer.norm.weight"] = np.ones(H, np.float32)
    for i in range(cfg.num_hidden_layers):
        p = f"pre_transformer.layers.{i}"
        lin(p + ".self_attn.q_proj", cfg.num_attention_heads * hd, H, bias=cfg.attention_bias)
        lin(p + ".self_attn.k_proj", cfg.num_key_value_heads * hd, H, bias=cfg.attention_bias)
        lin(p + ".self_attn.v_proj", cfg.num_key_value_heads * hd, H, bias=cfg.attention_bias)
        lin(p + ".self_attn.o_proj", H, cfg.num_attention_heads * hd, bias=cfg.attention_bias)
        lin(p + ".mlp.gate_proj", cfg.intermediate_size, H, bias=False)
        lin(p + ".mlp.up_proj", cfg.intermediate_size, H, bias=False)
        lin(p + ".mlp.down_proj", H, cfg.intermediate_size, bias=False)
        W[p + ".input_layernorm.weight"] = np.ones(H, np.float32)
        W[p + ".post_attention_layernorm.weight"] = np.ones(H, np.float32)
        W[p + ".self_attn_layer_scale.scale"] = np.full(H, layer_scale, np.float32)
        W[p + ".mlp_layer_scale.scale"] = np.full(H, layer_scale, np.float32)
    L = cfg.latent_dim
    for i, f in enumerate(cfg.upsampling_ratios):
        conv(f"upsample.{i}.layers.0.conv", L, f, L)
        p = f"upsample.{i}.layers.1"
        conv(p + ".dwconv.conv", L, 7, 1)
        W[p + ".norm.weight"] = np.ones(L, np.float32)
        W[p + ".norm.bias"] = np.zeros(L, np.float32)
        lin(p + ".pwconv1", 4 * L, L)
        lin(p + ".pwconv2", L, 4 * L)
        W[p + ".gamma"] = np.full(L, 0.3, np.float32)
    conv("decoder.0.conv", cfg.decoder_dim, 7, L)
    for b, r in enumerate(cfg.upsample_rates):
        cin, cout = cfg.decoder_dim >> b, cfg.decoder_dim >> (b + 1)
        p = f"decoder.{1 + b}.block"
        snake(p + ".0", cin)
        conv(p + ".1.conv", cout, 2 * r, cin)
        for j in (2, 3, 4):
            snake(f"{p}.{j}.act1", cout)
            conv(f"{p}.{j}.conv1.conv", cout, 7, cout)
            snake(f"{p}.{j}.act2", cout)
            conv(f"{p}.{j}.conv2.conv", cout, 1, cout)
    n = len(cfg.upsample_rates)
    snake(f"decoder.{n + 1}", cfg.decoder_dim >> n)
    conv(f"decoder.{n + 2}.conv", 1, 7, cfg.decoder_dim >> n)
    W[f"decoder.{n + 2}.conv.weight"] *= out_gain
    return W


def check_array_shape(shape: Tuple[int, ...]) -> bool:
    """checkArrayShapeQwen3 (:1445-1455)."""
    if len(shape) != 3:
        return False
    _, d2, d3 = shape
    if d2 == 1:
        return d3 > 64
    if d3 == 1:
        return d2 <= 64
    return d2 < d3


def sanitize(weights: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    """Qwen3TTSSpeechTokenizer.sanitize (:1094-1440), decoder keys only (encoder.* keys are the library's encoder sanitize's,
    loading.Weights.sanitize_speech_tokenizer_encoder; speaker-encoder keys are dropped).  PyTorch-layout checkpoint -> keys below
    ``decoder.`` in MLX layouts."""
    out: Dict[str, np.ndarray] = {}
    books: Dict[str, Dict[str, np.ndarray]] = {}
    for raw, v in weights.items():
        k = raw
        stripped = True
        while stripped:
            stripped = False
            for p in ("speech_tokenizer.", "encoder_model.", "decoder_model."):
                if k.startswith(p):
                    k, stripped = k[len(p):], True
                    break
        parts = k.split(".")
        if k in ("", "encoder_model", "decoder_model", "speech_tokenizer") or ("speaker_encoder" in parts and parts.index("speaker_encoder") + 1 < len(parts)):
            continue
        v = np.asarray(v)
        if "_codebook.cluster_usage" in k or "_codebook.embedding_sum" in k:
            base = k[: k.rfind("._codebook.")]
            books.setdefault(base, {})["cluster_usage" if "cluster_usage" in k else "embedding_sum"] = v
            continue
        if "_codebook.initialized" in k or ".codebook.initialized" in k or k.startswith("encoder."):
            continue
        is_tconv = ("upsample" in k and ".0.conv.weight" in k) or ("decoder.decoder" in k and "block.1.conv.weight" in k)
        if is_tconv and v.ndim == 3:
            if not check_array_shape(v.shape):
                v = v.transpose(1, 2, 0)
        elif ("conv.weight" in k or "_proj.weight" in k) and v.ndim == 3:
            if not check_array_shape(v.shape):
                v = v.transpose(0, 2, 1)
        if "upsample." in k:
            k = re.sub(r"upsample\.(\d+)\.(\d+)", r"upsample.\1.layers.\2", k)
        out[k] = np.ascontiguousarray(v)
    for base, d in books.items():
        if "cluster_usage" in d and "embedding_sum" in d:
            out[base + ".codebook.cluster_usage"] = d["cluster_usage"]
            out[base + ".codebook.embedding_sum"] = d["embedding_sum"]
    return out


class Qwen3TTSSpeechTokenizerDecoder:
    """Qwen3TTSSpeechTokenizerDecoder(config:) (:888-924).  ``weights``: sanitized keys relative to the decoder module
    (``quantizer.*``, ``pre_conv.*``, ``pre_transformer.*``, ``upsample.*``, ``decoder.*``); a leading ``decoder.`` is dropped."""

    def __init__(self, config: Qwen3TTSTokenizerDecoderConfig, *, weights: Dict[str, np.ndarray], device: int = 0, max_batch: int = 1,
                 max_cache_frames: int = 4096):
        self.config = config
        c = _ffi.SpeechTokenizerConfig()
        for name in ("codebook_size", "codebook_dim", "latent_dim", "decoder_dim", "hidden_size", "intermediate_size", "head_dim",
                     "num_attention_heads", "num_key_value_heads", "num_hidden_layers", "num_quantizers", "num_semantic_quantizers"):
            setattr(c, name, int(getattr(config, name)))
        c.rms_norm_eps, c.rope_theta, c.attention_bias = float(config.rms_norm_eps), float(config.rope_theta), int(bool(config.attention_bias))
        if len(config.upsample_rates) > 8 or len(config.upsampling_ratios) > 8:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "at most 8 upsample rates / upsampling ratios")
        c.num_upsample_rates, c.num_upsampling_ratios = len(config.upsample_rates), len(config.upsampling_ratios)
        for i, r in enumerate(config.upsample_rates):
            c.upsample_rates[i] = int(r)
        for i, r in enumerate(config.upsampling_ratios):
            c.upsampling_ratios[i] = int(r)
        c.max_batch, c.max_cache_frames = int(max_batch), int(max_cache_frames)
        w = {}
        for k, v in weights.items():
            if k.endswith(".initialized"):
                continue
            if k.startswith("decoder.") and not re.match(r"decoder\.\d+\.", k):
                k = k[len("decoder."):]
            w[k] = v
        table, keep = _ffi.make_tensor_table(w)
        self._h = C.c_void_p()
        _ffi.check(_ffi.lib().b2a_speech_tokenizer_create(device, C.byref(c), table, len(w), C.byref(self._h)))
        del keep
        self.total_upsample = int(_ffi.lib().b2a_speech_tokenizer_total_upsample(self._h))

    @classmethod
    def from_model_directory(cls, path, device: int = 0, max_batch: int = 1, max_cache_frames: int = 4096) -> "Qwen3TTSSpeechTokenizerDecoder":
        """loadSpeechTokenizer (Qwen3TTS.swift:1244-1275): <path>/config.json (optional) + every *.safetensors -> sanitize -> weights on
        the device, all inside the library."""
        self = cls.__new__(cls)
        self.config = None
        self._h = C.c_void_p()
        rate = C.c_int32(0)
        _ffi.check(_ffi.lib().b2a_speech_tokenizer_create_from_directory(str(path).encode(), device, max_batch, max_cache_frames, C.byref(self._h), C.byref(rate)))
        self.total_upsample = int(_ffi.lib().b2a_speech_tokenizer_total_upsample(self._h))
        self.decode_upsample_rate = int(rate.value)
        return self

    @property
    def stream(self) -> int:
        return int(_ffi.lib().b2a_speech_tokenizer_stream(self._h) or 0)

    @staticmethod
    def _codes(codes) -> np.ndarray:
        a = np.ascontiguousarray(codes, dtype=np.int32)
        if a.ndim != 3:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "codes must be [batch, num_quantizers, time]")
        return a

    def reset_streaming_state(self) -> None:
        """resetStreamingState (:949-970)."""
        _ffi.check(_ffi.lib().b2a_speech_tokenizer_reset(self._h))

    def streaming_step(self, codes) -> np.ndarray:
        """streamingStep (:973-1008): new code frames [B, n_q, T] -> their audio [B, 1, T * total_upsample]."""
        a = self._codes(codes)
        B, nq, T = a.shape
        out = np.empty((B, T * self.total_upsample), dtype=np.float32)
        _ffi.check(_ffi.lib().b2a_speech_tokenizer_streaming_step(self._h, _ffi.ptr(a), B, nq, T, _ffi.ptr(out)))
        return out[:, None, :]

    def __call__(self, codes) -> np.ndarray:
        """callAsFunction (:926-947): the whole sequence from a clean state."""
        self.reset_streaming_state()
        y = self.streaming_step(codes)
        self.reset_streaming_state()
        return y

    def chunked_decode(self, codes, chunk_size: int = 300, left_context_size: int = 25) -> np.ndarray:
        """chunkedDecode (:1010-1024)."""
        a = self._codes(codes)
        B, nq, T = a.shape
        out = np.empty((B, T * self.total_upsample), dtype=np.float32)
        _ffi.check(_ffi.lib().b2a_speech_tokenizer_chunked_decode(self._h, _ffi.ptr(a), B, nq, T, int(chunk_size), int(left_context_size), _ffi.ptr(out)))
        return out[:, None, :]

    def streaming_decode(self, codes, chunk_tokens: int = 100) -> np.ndarray:
        a = self._codes(codes)
        B, nq, T = a.shape
        out = np.empty((B, T * self.total_upsample), dtype=np.float32)
        _ffi.check(_ffi.lib().b2a_speech_tokenizer_streaming_decode(self._h, _ffi.ptr(a), B, nq, T, int(chunk_tokens), _ffi.ptr(out)))
        return out

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                _ffi.lib().b2a_speech_tokenizer_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass


class Qwen3TTSSpeechTokenizerEncoder:
    """Qwen3TTSSpeechTokenizerEncoder (:790-884) on the device: audio [B, 1, n] at 24 kHz -> codes [B, num_code_groups, T] int32,
    T = encoded_length(n).  ``weights``: the sanitized encoder keys (random_init_encoder_weights' key set); a leading
    "encoder_model." is dropped.  No encoder weights -> AudioGenerationError modelNotInitialized."""

    def __init__(self, config: Optional[Qwen3TTSTokenizerEncoderConfig] = None, *, weights: Dict[str, np.ndarray], device: int = 0):
        self.config = config or Qwen3TTSTokenizerEncoderConfig()
        c = self.config.to_ffi()
        w = {(k[len("encoder_model."):] if k.startswith("encoder_model.") else k): v for k, v in weights.items() if not k.endswith(".initialized")}
        self._h = C.c_void_p()
        if not w:
            raise _ffi.AudioGenerationError(_ffi.ERR_MODEL_NOT_INITIALIZED, "speech tokenizer encoder: no weights")
        table, keep = _ffi.make_tensor_table(w)
        _ffi.check(_ffi.lib().b2a_speech_tokenizer_encoder_create(device, C.byref(c), table, len(w), C.byref(self._h)))
        del keep
        self.num_code_groups = int(_ffi.lib().b2a_speech_tokenizer_encoder_num_code_groups(self._h))

    @classmethod
    def from_model_directory(cls, path, device: int = 0) -> "Qwen3TTSSpeechTokenizerEncoder":
        """The encoder half of loadSpeechTokenizer (Qwen3TTS.swift:1244-1275): <path>/config.json's encoder_config + every
        *.safetensors -> sanitize -> weights on the device, all inside the library."""
        self = cls.__new__(cls)
        self._h = C.c_void_p()
        c = _ffi.SpeechTokenizerEncoderConfig()
        _ffi.check(_ffi.lib().b2a_speech_tokenizer_encoder_config_from_json(str(Path(path) / "config.json").encode(), C.byref(c)))
        self.config = Qwen3TTSTokenizerEncoderConfig.from_ffi(c)
        _ffi.check(_ffi.lib().b2a_speech_tokenizer_encoder_create_from_directory(str(path).encode(), device, C.byref(self._h)))
        self.num_code_groups = int(_ffi.lib().b2a_speech_tokenizer_encoder_num_code_groups(self._h))
        return self

    @property
    def stream(self) -> int:
        return int(_ffi.lib().b2a_speech_tokenizer_encoder_stream(self._h) or 0)

    def encoded_length(self, n_samples: int) -> int:
        return int(_ffi.lib().b2a_speech_tokenizer_encoder_encoded_length(self._h, int(n_samples)))

    @staticmethod
    def _audio(audio) -> np.ndarray:
        a = np.ascontiguousarray(audio, dtype=np.float32)
        if a.ndim != 3 or a.shape[1] != 1:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "audio must be [batch, 1, samples]")
        return a

    def encode(self, audio) -> np.ndarray:
        """encode (:872-883): audio [B, 1, n] -> codes [B, num_code_groups, T]."""
        a = self._audio(audio)
        B, _, n = a.shape
        out = np.empty((B, self.num_code_groups, max(self.encoded_length(n), 0)), dtype=np.int32)
        _ffi.check(_ffi.lib().b2a_speech_tokenizer_encoder_encode(self._h, _ffi.ptr(a), B, n, _ffi.ptr(out)))
        return out

    def encode_dev(self, audio, codes, stream: int = 0) -> None:
        """Device tensors (torch, contiguous): audio float32 [B, 1, n] -> codes int32 [B, num_code_groups, T], enqueued on `stream`
        (0: the handle's) without a host synchronisation."""
        import torch
        if not (isinstance(audio, torch.Tensor) and isinstance(codes, torch.Tensor) and audio.is_cuda and codes.is_cuda):
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "encode_dev takes CUDA tensors")
        if audio.dtype != torch.float32 or codes.dtype != torch.int32 or not audio.is_contiguous() or not codes.is_contiguous() or audio.dim() != 3 \
                or audio.shape[1] != 1 or tuple(codes.shape) != (audio.shape[0], self.num_code_groups, self.encoded_length(audio.shape[2])):
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "encode_dev: audio must be float32 [B, 1, n] and codes int32 [B, groups, T]")
        _ffi.check(_ffi.lib().b2a_speech_tokenizer_encoder_encode_dev(self._h, _ffi.ptr(audio), int(audio.shape[0]), int(audio.shape[2]),
                                                                       _ffi.ptr(codes), C.c_void_p(stream or None)))

    def encode_latent(self, audio) -> Tuple[np.ndarray, np.ndarray]:
        """Parity hook: (z [B, T, hidden_size], codes [B, num_code_groups, T]) of one run."""
        a = self._audio(audio)
        B, _, n = a.shape
        T = self.encoded_length(n)
        z = np.empty((B, T, self.config.hidden_size), dtype=np.float32)
        codes = np.empty((B, self.num_code_groups, T), dtype=np.int32)
        _ffi.check(_ffi.lib().b2a_speech_tokenizer_encoder_latent_test(self._h, _ffi.ptr(a), B, n, _ffi.ptr(z), _ffi.ptr(codes)))
        return z, codes

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                _ffi.lib().b2a_speech_tokenizer_encoder_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass


class Qwen3TTSSpeechTokenizer:
    """Qwen3TTSSpeechTokenizer (:1027-1092).  ``audio_codes`` are ``[batch, time, num_quantizers]``.  ``encoder`` (optional, borrowed)
    is a Qwen3TTSSpeechTokenizerEncoder; without it the tokenizer only decodes, as the reference does without encoder_config."""

    def __init__(self, decoder_config: Optional[Qwen3TTSTokenizerDecoderConfig] = None, *, weights: Dict[str, np.ndarray], decode_upsample_rate: int = 1920,
                 device: int = 0, max_batch: int = 1, max_cache_frames: int = 4096, encoder: Optional[Qwen3TTSSpeechTokenizerEncoder] = None):
        self.decode_upsample_rate = int(decode_upsample_rate)
        self.decoder = Qwen3TTSSpeechTokenizerDecoder(decoder_config or Qwen3TTSTokenizerDecoderConfig(), weights=weights, device=device,
                                                      max_batch=max_batch, max_cache_frames=max_cache_frames)
        self.encoder = encoder

    @property
    def has_encoder(self) -> bool:
        return self.encoder is not None

    def encode(self, audio) -> np.ndarray:
        """encode (:1049-1057) with referenceAudioForEncoder's shapes (Qwen3TTS.swift:239-247): [n] -> [1, 1, n], [B, n] -> [B, 1, n],
        [B, 1, n] as is.  Returns codes [B, num_code_groups, T]."""
        if self.encoder is None:
            raise _ffi.AudioGenerationError(_ffi.ERR_MODEL_NOT_INITIALIZED, "Speech tokenizer encoder not available")
        a = np.asarray(audio, dtype=np.float32)
        if a.ndim == 1:
            a = a[None, None, :]
        elif a.ndim == 2:
            a = a[:, None, :]
        return self.encoder.encode(a)

    def decode(self, audio_codes) -> Tuple[np.ndarray, np.ndarray]:
        """decode (:1059-1068) -> (wav [B, samples], valid lengths [B])."""
        ac = np.asarray(audio_codes)
        wav = self.decoder.chunked_decode(np.ascontiguousarray(ac.transpose(0, 2, 1)))[:, 0]
        lengths = (ac[:, :, 0] > 0).sum(axis=1).astype(np.int32) * np.int32(self.decode_upsample_rate)
        return wav, lengths

    def streaming_decode(self, audio_codes, chunk_tokens: int = 100) -> List[np.ndarray]:
        """streamingDecode (:1070-1092): the per-chunk waveforms."""
        ac = np.asarray(audio_codes)
        wav = self.decoder.streaming_decode(np.ascontiguousarray(ac.transpose(0, 2, 1)), chunk_tokens)
        up, T = self.decoder.total_upsample, ac.shape[1]
        return [wav[:, s * up: min(s + chunk_tokens, T) * up] for s in range(0, T, chunk_tokens)]

    def decode_chunk(self, audio_codes, chunk_tokens: int = 300) -> np.ndarray:
        """Qwen3TTSModel.decodeChunk (Qwen3TTS.swift:214-231): row 0 of the streamed audio cut to the valid length."""
        ac = np.asarray(audio_codes)
        audio = np.concatenate(self.streaming_decode(ac, chunk_tokens), axis=-1)[0]
        valid = int((ac[:, :, 0] > 0).sum()) * self.decode_upsample_rate
        return audio[:valid] if 0 < valid < audio.shape[0] else audio
