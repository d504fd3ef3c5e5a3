"""float64 reference of Encodec with norm_type "time_group_norm" (the 48 kHz stereo model) for the 48 kHz tests and
tests/golden/make_golden_encodec_48khz.py.  Test infrastructure only: the layers are oracle.encodec's and the chunk loop, code
search and bandwidth rule are tests/encodec_encoder_reference.py's, with a GroupNorm(1, C_out) added after every conv.

Follows (paths relative to the reference checkout):
  Sources/MLXAudioCodecs/Encodec/EncodecLayers.swift:128-132, 189-210   EncodecConv1d: pad, conv, GroupNorm(1, C, pytorchCompatible)
  Sources/MLXAudioCodecs/Encodec/EncodecLayers.swift:244-248, 251-272   EncodecConvTranspose1dLayer: conv, GroupNorm, then trim
  Sources/MLXAudioCodecs/Encodec/EncodecLayers.swift:319-336            EncodecResnetBlock: shortcut(x) + block(x), each conv normed
  Sources/MLXAudioCodecs/Encodec/Encodec.swift:294-301                  decodeFrame: the chunk scale after the decoder

GroupNorm(1, C): per batch row, mean and biased variance over all T x C elements, eps 1e-5, affine norm.weight / norm.bias [C].
Weights use the checkpoint's keys: ``<conv prefix>norm.weight`` next to ``<conv prefix>conv.weight``.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence

import numpy as np

import encodec_encoder_reference as eer
from oracle import encodec as oe
from oracle.encodec import EncodecConfig, elu, lstm_block

EPS = 1e-5


def add_norm_weights(W: Dict[str, np.ndarray], seed: int = 99) -> Dict[str, np.ndarray]:
    """W plus ``norm.weight`` / ``norm.bias`` for every conv in it: gamma = +-U(0.5, 1.5), beta = +-U(0.1, 0.5), away from 1 and
    0 so that a dropped or swapped affine shows."""
    rng = np.random.default_rng(seed)
    out = dict(W)
    for k in sorted(W):
        if k.endswith("conv.weight"):
            pre, c = k[: -len("conv.weight")], W[k].shape[0]
            out[pre + "norm.weight"] = (np.where(rng.random(c) < 0.5, -1.0, 1.0) * rng.uniform(0.5, 1.5, c)).astype(np.float32)
            out[pre + "norm.bias"] = (np.where(rng.random(c) < 0.5, -1.0, 1.0) * rng.uniform(0.1, 0.5, c)).astype(np.float32)
    return out


def weights(cfg: EncodecConfig, n_codebooks: int, seed: int = 7, encoder: bool = True) -> Dict[str, np.ndarray]:
    """Decoder + codebooks (oe.init_weights), encoder (eer.init_encoder_weights) and every conv's norm."""
    W = oe.init_weights(cfg, seed, n_codebooks=n_codebooks)
    if encoder:
        W.update(eer.init_encoder_weights(cfg, seed + 1))
    return add_norm_weights(W, seed + 2)


def group_norm(x: np.ndarray, g: np.ndarray, b: np.ndarray) -> np.ndarray:
    """GroupNorm(1, C) on x [B, T, C] in float64."""
    x = np.asarray(x, dtype=np.float64)
    mu = x.mean(axis=(1, 2), keepdims=True)
    var = ((x - mu) ** 2).mean(axis=(1, 2), keepdims=True)
    return (x - mu) / np.sqrt(var + EPS) * g.astype(np.float64) + b.astype(np.float64)


def norm(W, pre, x):
    return group_norm(x, W[pre + "norm.weight"], W[pre + "norm.bias"])


def conv1d(cfg: EncodecConfig, W, pre: str, x: np.ndarray, stride: int = 1) -> np.ndarray:
    return norm(W, pre, oe.conv1d(cfg, x, W[pre + "conv.weight"], W[pre + "conv.bias"], stride=stride))


def conv_transpose1d_untrimmed(x: np.ndarray, w: np.ndarray, b: np.ndarray, stride: int) -> np.ndarray:
    """EncodecBaseConvTranspose1d (EncodecLayers.swift:371-450): [B, L, in] -> [B, (L - 1) * s + k, out]."""
    cout, k, _ = w.shape
    B, L, _ = x.shape
    y = np.zeros((B, (L - 1) * stride + k, cout), dtype=np.float64)
    w64 = w.astype(np.float64)
    for kk in range(k):
        y[:, kk: kk + (L - 1) * stride + 1: stride, :] += x @ w64[:, kk, :].T
    return y + b.astype(np.float64)


def trim(cfg: EncodecConfig, y: np.ndarray, k: int, stride: int) -> np.ndarray:
    padding_total = k - stride
    pr = math.ceil(padding_total * cfg.trim_right_ratio) if cfg.use_causal_conv else padding_total // 2
    pl = padding_total - pr
    end = y.shape[1] - pr
    return y[:, pl:end, :] if end > pl else y


def conv_transpose1d(cfg: EncodecConfig, W, pre: str, x: np.ndarray, stride: int) -> np.ndarray:
    """conv, then the norm over every output row, then the trim: the statistics include the trimmed samples."""
    w = W[pre + "conv.weight"]
    return trim(cfg, norm(W, pre, conv_transpose1d_untrimmed(x, w, W[pre + "conv.bias"], stride)), w.shape[1], stride)


def resnet_block(cfg: EncodecConfig, W, pre: str, x: np.ndarray) -> np.ndarray:
    h = conv1d(cfg, W, pre + "block.1.", elu(x))
    h = conv1d(cfg, W, pre + "block.3.", elu(h))
    return (conv1d(cfg, W, pre + "shortcut.", x) if cfg.use_conv_shortcut else x) + h


def decoder(cfg: EncodecConfig, W, emb: np.ndarray) -> np.ndarray:
    h = np.asarray(emb, dtype=np.float64)
    for idx, kind, p in oe.decoder_layout(cfg):
        pre = f"decoder.layers.{idx}."
        if kind == "conv":
            h = conv1d(cfg, W, pre, h)
        elif kind == "lstm":
            h = lstm_block(cfg, W, pre, h)
        elif kind == "elu":
            h = elu(h)
        elif kind == "convt":
            h = conv_transpose1d(cfg, W, pre, h, p["stride"])
        elif kind == "resnet":
            h = resnet_block(cfg, W, pre, h)
    return h


def decode(cfg: EncodecConfig, W, audio_codes: np.ndarray, audio_scales: Optional[Sequence] = None) -> np.ndarray:
    """Encodec.decode: [n_chunks, B, n_q, T] -> [B, samples, channels]; each chunk's scale multiplies its normed output."""
    scales = list(audio_scales) if audio_scales is not None else [None] * audio_codes.shape[0]

    def frame(i):
        y = decoder(cfg, W, oe.quantizer_decode(W, audio_codes[i]))
        return y if scales[i] is None else y * np.asarray(scales[i], dtype=np.float64).reshape(-1, 1, 1)

    if cfg.chunk_length is None:
        assert audio_codes.shape[0] == 1, "Expected one frame"
        return frame(0)
    return oe.linear_overlap_add([frame(i) for i in range(audio_codes.shape[0])], cfg.chunk_stride or 1)


def encoder(cfg: EncodecConfig, W, x: np.ndarray) -> np.ndarray:
    h = np.asarray(x, dtype=np.float64)
    for idx, kind, p in eer.encoder_layout(cfg):
        pre = f"encoder.layers.{idx}."
        if kind == "conv":
            h = conv1d(cfg, W, pre, h, stride=p["stride"])
        elif kind == "resnet":
            h = resnet_block(cfg, W, pre, h)
        elif kind == "elu":
            h = elu(h)
        elif kind == "lstm":
            h = lstm_block(cfg, W, pre, h)
    return h


def encode(cfg: EncodecConfig, W, x: np.ndarray, bandwidth: Optional[float] = None):
    """Encodec.encode: x [B, L, C] -> (codes [n_chunks, B, n_q, T], scales [n_chunks] of [B] or None, z [n_chunks, B, T, D])."""
    bw = cfg.target_bandwidths[0] if bandwidth is None else bandwidth
    if bw not in cfg.target_bandwidths:
        raise ValueError(f"bandwidth {bw} not in {cfg.target_bandwidths}")
    n_q = eer.num_quantizers_for_bandwidth(cfg, bw)
    offsets, clen = eer.chunk_offsets(cfg, x.shape[1])
    codes, scales, zs = [], [], []
    for o in offsets:
        v = np.asarray(x[:, o:o + clen], dtype=np.float64)
        scale = None
        if cfg.normalize:
            mono = v.sum(axis=2, keepdims=True) / v.shape[2]
            scale = np.sqrt((mono ** 2).mean(axis=1, keepdims=True)) + 1e-8
            v = v / scale
        z = encoder(cfg, W, v)
        codes.append(eer.rvq_encode(W, z, n_q)); scales.append(None if scale is None else scale.reshape(-1)); zs.append(z)
    return np.stack(codes, 0), scales, np.stack(zs, 0)


def config_48khz(**kw) -> EncodecConfig:
    """The 48 kHz model's geometry (facebook/encodec_48khz): stereo, non-causal reflect, normalize, 1 s chunks with 1 % overlap."""
    base = dict(audio_channels=2, use_causal_conv=False, normalize=True, norm_type="time_group_norm", sampling_rate=48000,
                chunk_length_s=1.0, overlap=0.01, target_bandwidths=[3.0, 6.0, 12.0, 24.0])
    base.update(kw)
    return EncodecConfig(**base)
