"""float64 torch restatement of the Mimi codec: encode, decode, the streaming decodeStep with all its state, decodeFrames and the
checkpoint sanitize.  Test infrastructure only: the encoder half is tests/qwen3_encoder_reference.py's (the Qwen3-TTS
speech-tokenizer encoder is Mimi's encoder), reached through the adapter properties of MimiConfig.

Follows (paths relative to the reference checkout, directory Sources/MLXAudioCodecs/Mimi/):
  Mimi.swift:47-97          mimi_202407(numCodebooks)
  Mimi.swift:168-232        encode, decode, decodeStep, MimiStreamingDecoder (reset, decodeFrames)
  Mimi.swift:337-413        sanitize
  Quantization.swift        EuclideanCodebook (embedding_sum / max(cluster_usage, 1e-5)), split RVQ decode
  Conv.swift                StreamableConv1d(.step), StreamableConvTranspose1d(.step), ConvTrUpsample1d
  Transformer.swift         Attention (per-call context window), TransformerLayer, ProjectedTransformer
  Seanet.swift              StreamingAdd, SeanetResnetBlock, DecoderLayer, SeanetDecoder

Restatement traps:
  1. RoPE is MLX RoPE(traditional: true): interleaved pairs (2i, 2i + 1), base maxPeriod.  transformers.MimiModel rotates halves,
     so its q / k rows must be permuted per head before the two agree (as for the Qwen3 encoder, DESIGN.md §3.8b).
  2. The attention window is per CALL, not per query (Transformer.swift:156-176).  With cache offset p0 and T new positions the
     call keeps the last T + min(context, p0) keys, and MLXFast's causal mask is aligned bottom-right, so query t sees cache
     positions [max(0, p0 - context), p0 + t].  The mask rule is mlx-swift-lm's createAttentionMask(h:cache:) and MLX's
     "causal" mode (not vendored in the reference checkout): .causal for T > 1, no mask for T = 1.  A one-shot decode (p0 = 0) is
     full causal over the clip; a stream past `context` latent positions differs from it and from transformers' per-query window.
  3. StreamableConvTranspose1d.step subtracts the bias from the carried tail before the overlap-add (Conv.swift:316), so
     overlap frames get the bias once (the Qwen3-TTS decoder's DecoderBlockUpsample adds it twice).
  4. StreamingAdd holds back the longer operand's excess frames for the next call (Seanet.swift:61-89).  With stride-1 causal
     convs both operands have the same length, so nothing is ever held -- restated anyway.
  5. decode with K < nq codebooks decodes layers[0 ..< K]: rvq_first on level 0, rvq_rest's first K - 1 layers on the rest
     (Quantization.swift:113-120, 203-210).  K = 1 uses rvq_first alone (the reference would index an empty rest).
  6. MimiStreamingDecoder.reset clears the decoder convs, the upsample tail and the KV cache; Mimi.decode() resets the decoder
     and the cache but uses the NON-streaming upsample and SEANet, so it neither reads nor updates any streaming tail.
"""
from __future__ import annotations

import re
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

DT = torch.float64


@dataclass
class MimiConfig:
    sample_rate: int = 24000
    frame_rate: float = 12.5
    dimension: int = 512
    n_filters: int = 64
    ratios: Tuple[int, ...] = (8, 6, 5, 4)
    kernel_size: int = 7
    residual_kernel_size: int = 3
    last_kernel_size: int = 3
    compress: int = 2
    num_heads: int = 8
    num_layers: int = 8
    dim_feedforward: int = 2048
    context: int = 250
    max_period: int = 10000
    num_codebooks: int = 32
    codebook_size: int = 2048
    codebook_dim: int = 256

    @property
    def hop(self) -> int:
        return int(np.prod(self.ratios))

    @property
    def downsample_stride(self) -> int:              # Mimi.init (:122-123)
        return int(self.sample_rate / self.hop / self.frame_rate)

    @property
    def samples_per_frame(self) -> int:
        return self.hop * self.downsample_stride

    @property
    def head_dim(self) -> int:
        return self.dimension // self.num_heads

    # the names tests/qwen3_encoder_reference.py reads
    @property
    def upsampling_ratios(self):
        return list(self.ratios)

    @property
    def num_attention_heads(self) -> int:
        return self.num_heads

    @property
    def num_hidden_layers(self) -> int:
        return self.num_layers

    @property
    def rope_theta(self) -> float:
        return float(self.max_period)

    @property
    def num_code_groups(self) -> int:
        return self.num_codebooks


def mimi_202407(num_codebooks: int = 32) -> MimiConfig:
    """Mimi.swift:47-97."""
    return MimiConfig(num_codebooks=num_codebooks)


def small_config(num_codebooks: int = 8) -> MimiConfig:
    """The test geometry: every layer of the shipped one, narrower (decoder widths 256 .. 16, residual hidden 8)."""
    return MimiConfig(dimension=64, n_filters=16, num_heads=2, num_layers=2, dim_feedforward=128, num_codebooks=num_codebooks,
                      codebook_size=64, codebook_dim=16)


# ---------------------------------------------------------------- weights (MLX layouts, sanitized names)
def init_weights(cfg: MimiConfig, seed: int = 0) -> Dict[str, np.ndarray]:
    """Random weights for every tensor the codec reads, scaled so that activations stay O(1) through the stack."""
    rng = np.random.default_rng(seed)
    W: Dict[str, np.ndarray] = {}
    D, nf, L = cfg.dimension, cfg.n_filters, len(cfg.ratios)

    def conv(name, cout, k, cin, bias=True, gain=1.0):
        W[name + ".weight"] = (rng.standard_normal((cout, k, cin)) * gain / np.sqrt(k * cin)).astype(np.float32)
        if bias:
            W[name + ".bias"] = (0.05 * rng.standard_normal(cout)).astype(np.float32)

    def tlayers(prefix):
        for l in range(cfg.num_layers):
            p = f"{prefix}.transformer.layers.{l}."
            W[p + "self_attn.in_proj.weight"] = (rng.standard_normal((3 * D, D)) / np.sqrt(D)).astype(np.float32)
            W[p + "self_attn.out_proj.weight"] = (rng.standard_normal((D, D)) / np.sqrt(D)).astype(np.float32)
            W[p + "gating.linear1.weight"] = (rng.standard_normal((cfg.dim_feedforward, D)) / np.sqrt(D)).astype(np.float32)
            W[p + "gating.linear2.weight"] = (rng.standard_normal((D, cfg.dim_feedforward)) / np.sqrt(cfg.dim_feedforward)).astype(np.float32)
            for n in ("norm1", "norm2"):
                W[p + n + ".weight"] = (1 + 0.1 * rng.standard_normal(D)).astype(np.float32)
                W[p + n + ".bias"] = (0.05 * rng.standard_normal(D)).astype(np.float32)
            for n in ("layer_scale_1", "layer_scale_2"):
                W[p + n + ".scale"] = (0.3 + 0.2 * rng.random(D)).astype(np.float32)

    # encoder
    conv("encoder.init_conv1d.conv.conv", nf, cfg.kernel_size, 1)
    ch = nf
    for i, r in enumerate(reversed(cfg.ratios)):
        p = f"encoder.layers.{i}."
        conv(p + "residuals.0.block.0.conv.conv", ch // cfg.compress, cfg.residual_kernel_size, ch)
        conv(p + "residuals.0.block.1.conv.conv", ch, 1, ch // cfg.compress)
        conv(p + "downsample.conv.conv", 2 * ch, 2 * r, ch)
        ch *= 2
    conv("encoder.final_conv1d.conv.conv", D, cfg.last_kernel_size, ch)
    tlayers("encoder_transformer")
    conv("downsample.conv.conv.conv", D, 2 * cfg.downsample_stride, D, bias=False)
    # quantizer
    qd, bins = cfg.codebook_dim, cfg.codebook_size
    for name, n in (("rvq_first", 1), ("rvq_rest", cfg.num_codebooks - 1)):
        W[f"quantizer.{name}.input_proj.weight"] = (rng.standard_normal((qd, 1, D)) / np.sqrt(D)).astype(np.float32)
        W[f"quantizer.{name}.output_proj.weight"] = (rng.standard_normal((D, 1, qd)) / np.sqrt(qd)).astype(np.float32)
        for i in range(n):
            p = f"quantizer.{name}.vq.layers.{i}.codebook."
            W[p + "embedding_sum"] = (0.5 * rng.standard_normal((bins, qd))).astype(np.float32)
            W[p + "cluster_usage"] = (0.5 + 1.5 * rng.random(bins)).astype(np.float32)
    # decoder
    W["upsample.convtr.convtr.convtr.weight"] = (0.5 + 0.3 * rng.standard_normal((D, 2 * cfg.downsample_stride, 1))).astype(np.float32)
    tlayers("decoder_transformer")
    conv("decoder.init_conv1d.conv.conv", nf << L, cfg.kernel_size, D)
    for i, r in enumerate(cfg.ratios):
        cin = nf << (L - i)
        p = f"decoder.layers.{i}."
        W[p + "upsample.convtr.convtr.weight"] = (rng.standard_normal((cin // 2, 2 * r, cin)) / np.sqrt(2 * cin)).astype(np.float32)
        W[p + "upsample.convtr.convtr.bias"] = (0.05 * rng.standard_normal(cin // 2)).astype(np.float32)
        conv(p + "residuals.0.block.0.conv.conv", cin // 2 // cfg.compress, cfg.residual_kernel_size, cin // 2)
        conv(p + "residuals.0.block.1.conv.conv", cin // 2, 1, cin // 2 // cfg.compress)
    conv("decoder.final_conv1d.conv.conv", 1, cfg.last_kernel_size, nf)
    return W


def _t(W, k) -> torch.Tensor:
    return torch.as_tensor(np.asarray(W[k])).to(DT)


# ---------------------------------------------------------------- building blocks (NCL, float64)
def codebook(W, name: str, i: int) -> torch.Tensor:
    p = f"quantizer.{name}.vq.layers.{i}.codebook."
    return _t(W, p + "embedding_sum") / torch.clamp(_t(W, p + "cluster_usage"), min=1e-5)[:, None]


def quantizer_decode(cfg: MimiConfig, W, codes) -> torch.Tensor:
    """SplitResidualVectorQuantizer.decode on codes [B, K, T] -> [B, D, T] (trap 5)."""
    codes = torch.as_tensor(np.asarray(codes), dtype=torch.long)
    K = codes.shape[1]
    assert 1 <= K <= cfg.num_codebooks
    out = codebook(W, "rvq_first", 0)[codes[:, 0]] @ _t(W, "quantizer.rvq_first.output_proj.weight")[:, 0, :].T
    if K > 1:
        rest = sum(codebook(W, "rvq_rest", i)[codes[:, 1 + i]] for i in range(K - 1))
        out = out + rest @ _t(W, "quantizer.rvq_rest.output_proj.weight")[:, 0, :].T
    return out.transpose(1, 2)


def _convtr_full(W, x: torch.Tensor, prefix: str, stride: int, depthwise: bool = False) -> torch.Tensor:
    """MLX convTransposed1d + bias, untrimmed: output length (T - 1) stride + k."""
    w = _t(W, prefix + ".weight")
    b = _t(W, prefix + ".bias") if prefix + ".bias" in W else None
    if depthwise:                                   # MLX [C, k, 1] -> torch [C, 1, k], groups = C
        return F.conv_transpose1d(x, w.permute(0, 2, 1), b, stride=stride, groups=w.shape[0])
    return F.conv_transpose1d(x, w.permute(2, 0, 1), b, stride=stride)      # MLX [out, k, in] -> torch [in, out, k]


def _conv(W, x: torch.Tensor, prefix: str) -> torch.Tensor:
    """stride-1 conv, MLX [out, k, in], no padding."""
    w = _t(W, prefix + ".weight")
    b = _t(W, prefix + ".bias") if prefix + ".bias" in W else None
    return F.conv1d(x, w.permute(0, 2, 1), b)


def rope(x: torch.Tensor, offset: int, base: float) -> torch.Tensor:
    """MLX RoPE(traditional: true) on [B, heads, T, hd] at positions offset .. offset + T - 1 (trap 1)."""
    hd, T = x.shape[-1], x.shape[-2]
    inv = base ** (-torch.arange(0, hd, 2, dtype=DT) / hd)
    ang = torch.arange(offset, offset + T, dtype=DT)[:, None] * inv[None, :]
    c, s = torch.cos(ang), torch.sin(ang)
    x1, x2 = x[..., 0::2], x[..., 1::2]
    out = torch.empty_like(x)
    out[..., 0::2] = x1 * c - x2 * s
    out[..., 1::2] = x1 * s + x2 * c
    return out


class KVCache:
    """KVCacheSimple: keys / values appended per call; offset = positions seen."""

    def __init__(self):
        self.k: Optional[torch.Tensor] = None
        self.v: Optional[torch.Tensor] = None
        self.offset = 0

    def update(self, k, v):
        self.k = k if self.k is None else torch.cat([self.k, k], 2)
        self.v = v if self.v is None else torch.cat([self.v, v], 2)
        self.offset += k.shape[2]
        return self.k, self.v


def transformer(cfg: MimiConfig, W, prefix: str, x: torch.Tensor, caches: List[KVCache]) -> torch.Tensor:
    """ProjectedTransformer (no projections at dimension == dModel) on [B, T, D] over the caches (trap 2)."""
    B, T, D = x.shape
    nh, hd = cfg.num_heads, cfg.head_dim
    for l, cache in enumerate(caches):
        p = f"{prefix}.transformer.layers.{l}."
        h = F.layer_norm(x, (D,), _t(W, p + "norm1.weight"), _t(W, p + "norm1.bias"), 1e-5)
        qkv = (h @ _t(W, p + "self_attn.in_proj.weight").T).reshape(B, T, 3, nh, hd)
        q, k, v = (qkv[:, :, i].transpose(1, 2) for i in range(3))
        p0 = cache.offset
        q, k = rope(q, p0, float(cfg.max_period)), rope(k, p0, float(cfg.max_period))
        k, v = cache.update(k, v)
        k_len = k.shape[2]
        target = T + min(cfg.context, k_len - T)
        k, v = k[:, :, k_len - target:], v[:, :, k_len - target:]
        s = (q @ k.transpose(-1, -2)) / np.sqrt(hd)
        if T > 1:                                    # MLXFast causal mask, aligned bottom-right
            kl = k.shape[2]
            allowed = torch.arange(kl)[None, :] <= torch.arange(T)[:, None] + (kl - T)
            s = s.masked_fill(~allowed, float("-inf"))
        a = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B, T, D) @ _t(W, p + "self_attn.out_proj.weight").T
        x = x + _t(W, p + "layer_scale_1.scale") * a
        h = F.layer_norm(x, (D,), _t(W, p + "norm2.weight"), _t(W, p + "norm2.bias"), 1e-5)
        m = F.gelu(h @ _t(W, p + "gating.linear1.weight").T) @ _t(W, p + "gating.linear2.weight").T
        x = x + _t(W, p + "layer_scale_2.scale") * m
    return x


# ---------------------------------------------------------------- one-shot decode (Mimi.decode, :178-186)
def _conv_causal(W, x, prefix):
    k = np.asarray(W[prefix + ".weight"]).shape[1]
    return _conv(W, F.pad(x, (k - 1, 0)), prefix)


def seanet_decode(cfg: MimiConfig, W, z: torch.Tensor) -> torch.Tensor:
    """SeanetDecoder.callAsFunction on [B, D, T25] -> [B, 1, T25 * hop] (non-streaming convs, zero causal padding)."""
    x = _conv_causal(W, z, "decoder.init_conv1d.conv.conv")
    for i, r in enumerate(cfg.ratios):
        p = f"decoder.layers.{i}."
        y = _convtr_full(W, F.elu(x), p + "upsample.convtr.convtr", r)
        x = y[..., : y.shape[-1] - r]                # causal: unpad k - stride = r on the right
        h = _conv_causal(W, F.elu(x), p + "residuals.0.block.0.conv.conv")
        x = x + _conv_causal(W, F.elu(h), p + "residuals.0.block.1.conv.conv")
    return _conv_causal(W, F.elu(x), "decoder.final_conv1d.conv.conv")


def decode(cfg: MimiConfig, W, codes) -> np.ndarray:
    """Mimi.decode: codes [B, K, T] -> [B, 1, T * samples_per_frame]."""
    z = quantizer_decode(cfg, W, codes)
    s = cfg.downsample_stride
    y = _convtr_full(W, z, "upsample.convtr.convtr.convtr", s, depthwise=True)
    z = y[..., : y.shape[-1] - s]
    z = transformer(cfg, W, "decoder_transformer", z.transpose(1, 2), [KVCache() for _ in range(cfg.num_layers)]).transpose(1, 2)
    return seanet_decode(cfg, W, z).numpy()


# ---------------------------------------------------------------- streaming (decodeStep, :196-202) with every state
class _StreamConv:
    """StreamableConv1d.step at stride 1, dilation 1: left pad k - 1 zeros on the first call, prevXs carried."""

    def __init__(self, W, prefix):
        self.W, self.prefix, self.k = W, prefix, np.asarray(W[prefix + ".weight"]).shape[1]
        self.prev: Optional[torch.Tensor] = None
        self.padded = False

    def __call__(self, x):
        if not self.padded:
            self.padded = True
            x = F.pad(x, (self.k - 1, 0))
        if self.prev is not None:
            x = torch.cat([self.prev, x], 2)
        L = x.shape[2]
        nframes = max(L + 1 - self.k, 0)
        if nframes == 0:
            self.prev = x
            return torch.zeros(x.shape[0], np.asarray(self.W[self.prefix + ".weight"]).shape[0], 0, dtype=DT)
        self.prev = x[..., nframes:]
        return _conv(self.W, x[..., : nframes - 1 + self.k], self.prefix)


class _StreamConvTr:
    """StreamableConvTranspose1d.step: the carried tail gets the bias subtracted before the overlap-add (trap 3)."""

    def __init__(self, W, prefix, stride, depthwise=False):
        self.W, self.prefix, self.stride, self.depthwise = W, prefix, stride, depthwise
        self.k = 2 * stride
        self.prev: Optional[torch.Tensor] = None

    def __call__(self, x):
        y = _convtr_full(self.W, x, self.prefix, self.stride, self.depthwise)
        ot = y.shape[2]
        if self.prev is not None:
            prev = self.prev
            if self.prefix + ".bias" in self.W:
                prev = prev - _t(self.W, self.prefix + ".bias")[None, :, None]
            pt = prev.shape[2]
            y = torch.cat([y[..., :pt] + prev, y[..., pt:]], 2)
        cut = max(ot - (self.k - self.stride), 0)
        self.prev = y[..., cut:]
        return y[..., :cut]


class _StreamingAdd:
    """StreamingAdd.step (trap 4)."""

    def __init__(self):
        self.lhs: Optional[torch.Tensor] = None
        self.rhs: Optional[torch.Tensor] = None

    def __call__(self, l, r):
        if self.lhs is not None:
            l, self.lhs = torch.cat([self.lhs, l], 2), None
        if self.rhs is not None:
            r, self.rhs = torch.cat([self.rhs, r], 2), None
        ll, rl = l.shape[2], r.shape[2]
        if ll < rl:
            self.rhs = r[..., ll:]
            return l + r[..., :ll]
        if rl < ll:
            self.lhs = l[..., rl:]
            return l[..., :rl] + r
        return l + r


class MimiStreamer:
    """Mimi.decodeStep / MimiStreamingDecoder on one Mimi: the upsample tail, every decoder conv's state and the KV caches."""

    def __init__(self, cfg: MimiConfig, W):
        self.cfg, self.W = cfg, W
        self.reset()

    def reset(self):
        """MimiStreamingDecoder.reset: decoder convs, upsample tail, KV caches (trap 6)."""
        cfg, W = self.cfg, self.W
        self.up = _StreamConvTr(W, "upsample.convtr.convtr.convtr", cfg.downsample_stride, depthwise=True)
        self.caches = [KVCache() for _ in range(cfg.num_layers)]
        self.init = _StreamConv(W, "decoder.init_conv1d.conv.conv")
        self.layers = []
        for i, r in enumerate(cfg.ratios):
            p = f"decoder.layers.{i}."
            self.layers.append((_StreamConvTr(W, p + "upsample.convtr.convtr", r), _StreamConv(W, p + "residuals.0.block.0.conv.conv"),
                                _StreamConv(W, p + "residuals.0.block.1.conv.conv"), _StreamingAdd()))
        self.final = _StreamConv(W, "decoder.final_conv1d.conv.conv")

    def decode_step(self, codes) -> np.ndarray:
        """codes [B, K, T] -> [B, 1, T * samples_per_frame]."""
        z = self.up(quantizer_decode(self.cfg, self.W, codes))
        z = transformer(self.cfg, self.W, "decoder_transformer", z.transpose(1, 2), self.caches).transpose(1, 2)
        x = self.init(z)
        for ct, c1, c2, add in self.layers:
            x = ct(F.elu(x))
            x = add(c2(F.elu(c1(F.elu(x)))), x)
        return self.final(F.elu(x)).numpy()

    def decode_frames(self, tokens) -> np.ndarray:
        """decodeFrames: [K, T] or [B, K, T] -> T single-frame steps, concatenated."""
        tok = np.asarray(tokens)
        if tok.ndim == 2:
            tok = tok[None]
        return np.concatenate([self.decode_step(tok[:, :, t:t + 1]) for t in range(tok.shape[2])], 2)


# ---------------------------------------------------------------- encode (Mimi.encode, :168-176): the Qwen3 encoder's reference
def encode(cfg: MimiConfig, W, audio) -> np.ndarray:
    """[B, 1, n] -> codes [B, nq, T] (float64 search)."""
    import qwen3_encoder_reference as qer
    return qer.encode_codes(cfg, W, qer.latent(cfg, W, audio))


def encoded_length(cfg: MimiConfig, n: int) -> int:
    import qwen3_encoder_reference as qer
    return qer.encoded_length(n, list(cfg.ratios), cfg.downsample_stride)


# ---------------------------------------------------------------- sanitize (Mimi.swift:337-413), restated
def _swap_last(v: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(np.swapaxes(v, -1, -2)) if v.ndim >= 2 else v


def sanitize(weights: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    out: Dict[str, np.ndarray] = {}
    for raw, v in weights.items():
        k = ".".join(s[1:] if s.startswith("_") else s for s in raw.split("."))
        if k.startswith("encoder.model."):
            k = k.replace("encoder.model.", "encoder.")
        if k.startswith("decoder.model."):
            k = k.replace("decoder.model.", "decoder.")
        if k.endswith(".in_proj_weight"):
            k = k.replace(".in_proj_weight", ".in_proj.weight")
        if k.endswith(".linear1.weight"):
            k = k.replace(".linear1.weight", ".gating.linear1.weight")
        if k.endswith(".linear2.weight"):
            k = k.replace(".linear2.weight", ".gating.linear2.weight")
        for l, d in enumerate([2, 5, 8, 11]):
            k = k.replace(f"decoder.{d}.", f"decoder.layers.{l}.upsample.")
            k = k.replace(f"decoder.{d + 1}.", f"decoder.layers.{l}.residuals.0.")
        for l, e in enumerate([1, 4, 7, 10]):
            k = k.replace(f"encoder.{e}.", f"encoder.layers.{l}.residuals.0.")
            k = k.replace(f"encoder.{e + 2}.", f"encoder.layers.{l}.downsample.")
        k = k.replace("decoder.0.", "decoder.init_conv1d.").replace("decoder.14.", "decoder.final_conv1d.")
        k = k.replace("encoder.0.", "encoder.init_conv1d.").replace("encoder.14.", "encoder.final_conv1d.")
        k = k.replace(".block.1.", ".block.0.").replace(".block.3.", ".block.1.")
        v = np.asarray(v)
        if k.endswith(".conv.weight") or k.endswith(".output_proj.weight") or k.endswith(".input_proj.weight"):
            v = _swap_last(v)
        if k.endswith(".convtr.weight") and v.ndim == 3:
            v = np.ascontiguousarray(np.swapaxes(v, 1, 2) if v.shape[1] == 1 else v.transpose(1, 2, 0))
        out[k] = v
    return out


def unsanitize(W: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    """The restated map inverted over the oracle's key set: MLX names and layouts -> a moshi-named PyTorch-layout checkpoint
    (the codebooks under "_codebook", the spelling of the released checkpoints' EuclideanCodebook buffers)."""
    out: Dict[str, np.ndarray] = {}
    for k, v in W.items():
        v = np.asarray(v)
        if k.endswith(".conv.weight") or k.endswith(".output_proj.weight") or k.endswith(".input_proj.weight"):
            v = _swap_last(v)
        if k.endswith(".convtr.weight") and v.ndim == 3:
            v = np.ascontiguousarray(np.swapaxes(v, 1, 2) if v.shape[2] == 1 else v.transpose(2, 0, 1))
        m = k.replace(".block.1.", ".block.3.").replace(".block.0.", ".block.1.")
        for side in ("encoder", "decoder"):
            m = m.replace(f"{side}.init_conv1d.", f"{side}.model.0.").replace(f"{side}.final_conv1d.", f"{side}.model.14.")
        m = re.sub(r"^decoder\.layers\.(\d)\.upsample\.", lambda g: f"decoder.model.{2 + 3 * int(g.group(1))}.", m)
        m = re.sub(r"^decoder\.layers\.(\d)\.residuals\.0\.", lambda g: f"decoder.model.{3 + 3 * int(g.group(1))}.", m)
        m = re.sub(r"^encoder\.layers\.(\d)\.residuals\.0\.", lambda g: f"encoder.model.{1 + 3 * int(g.group(1))}.", m)
        m = re.sub(r"^encoder\.layers\.(\d)\.downsample\.", lambda g: f"encoder.model.{3 + 3 * int(g.group(1))}.", m)
        m = m.replace(".gating.linear1.weight", ".linear1.weight").replace(".gating.linear2.weight", ".linear2.weight")
        m = m.replace(".in_proj.weight", ".in_proj_weight").replace(".codebook.", "._codebook.")
        out[m] = v
    return out
