"""float64 reference of the Encodec encode path for the encoder tests and tests/golden/make_golden_encodec_encode.py.  Test
infrastructure only: the layers are oracle.encodec's (conv1d, elu, lstm_block, resnet_block), so the encoder follows exactly
the layer semantics the decoder tests pin.

Follows (paths relative to the reference checkout):
  Sources/MLXAudioCodecs/Encodec/Encodec.swift:17-88                 EncodecEncoder (module array, ELU slots counted)
  Sources/MLXAudioCodecs/Encodec/Encodec.swift:212-291               encodeFrame (normalize, scale) / encode (chunk loop)
  Sources/MLXAudioCodecs/Encodec/Encodec.swift:457-460               encodeAudio
  Sources/MLXAudioCodecs/Encodec/EncodecQuantization.swift:22-38     EncodecEuclideanCodebook.quantize (argMax of -dist)
  Sources/MLXAudioCodecs/Encodec/EncodecQuantization.swift:90-115    getNumQuantizersForBandwidth / residual encode
  Sources/MLXAudioCodecs/Encodec/EncodecLayers.swift:92-211          EncodecConv1d (padding_total = k - stride + extra right pad)

Weights use the checkpoint's keys ``encoder.layers.{i}.…`` in the decoder's MLX layouts.  At 24 kHz the module array is
0 conv, then per reversed ratio (2, 4, 5, 8) resnet, ELU, strided conv k = 2r, then 13 LSTM, 14 ELU, 15 conv.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np

from oracle import encodec as oe
from oracle.encodec import EncodecConfig, conv1d, elu, lstm_block, resnet_block


def encoder_layout(cfg: EncodecConfig):
    """EncodecEncoder's `layers` (Encodec.swift:20-70) as (index, kind, params); indices are the weight-key slots."""
    out = []
    i = 0
    out.append((i, "conv", dict(cin=cfg.audio_channels, cout=cfg.num_filters, k=cfg.kernel_size, stride=1))); i += 1
    scaling = 1
    for ratio in reversed(cfg.upsampling_ratios):
        cur = scaling * cfg.num_filters
        for j in range(cfg.num_residual_layers):
            out.append((i, "resnet", dict(dim=cur, dilations=[cfg.dilation_growth_rate ** j, 1]))); i += 1
        out.append((i, "elu", {})); i += 1
        out.append((i, "conv", dict(cin=cur, cout=2 * cur, k=2 * ratio, stride=ratio))); i += 1
        scaling *= 2
    out.append((i, "lstm", dict(dim=scaling * cfg.num_filters))); i += 1
    out.append((i, "elu", {})); i += 1
    out.append((i, "conv", dict(cin=scaling * cfg.num_filters, cout=cfg.hidden_size, k=cfg.last_kernel_size, stride=1))); i += 1
    return out


def init_encoder_weights(cfg: EncodecConfig, seed: int = 4321) -> Dict[str, np.ndarray]:
    """Random-init encoder weights (``encoder.*`` keys only; merge with ``oe.init_weights`` for a full codec), drawn like
    ``oe.init_weights``: U(+-1/sqrt(fan_in)) convs and LSTM."""
    rng = np.random.default_rng(seed)
    w: Dict[str, np.ndarray] = {}

    def u(shape, fan):
        s = (1.0 / fan) ** 0.5
        return rng.uniform(-s, s, size=shape).astype(np.float32)

    for idx, kind, p in encoder_layout(cfg):
        pre = f"encoder.layers.{idx}."
        if kind == "conv":
            w[pre + "conv.weight"] = u((p["cout"], p["k"], p["cin"]), p["k"] * p["cin"])
            w[pre + "conv.bias"] = u((p["cout"],), p["k"] * p["cin"])
        elif kind == "lstm":
            d = p["dim"]
            for l in range(cfg.num_lstm_layers):
                w[pre + f"lstm.{l}.Wx"] = u((4 * d, d), d)
                w[pre + f"lstm.{l}.Wh"] = u((4 * d, d), d)
                w[pre + f"lstm.{l}.bias"] = u((4 * d,), d)
        elif kind == "resnet":
            dim, hid = p["dim"], p["dim"] // cfg.compress
            w[pre + "block.1.conv.weight"] = u((hid, cfg.residual_kernel_size, dim), cfg.residual_kernel_size * dim)
            w[pre + "block.1.conv.bias"] = u((hid,), cfg.residual_kernel_size * dim)
            w[pre + "block.3.conv.weight"] = u((dim, 1, hid), hid)
            w[pre + "block.3.conv.bias"] = u((dim,), hid)
            if cfg.use_conv_shortcut:
                w[pre + "shortcut.conv.weight"] = u((dim, 1, dim), dim)
                w[pre + "shortcut.conv.bias"] = u((dim,), dim)
    return w


def encoder(cfg: EncodecConfig, W: Dict[str, np.ndarray], x: np.ndarray) -> np.ndarray:
    """EncodecEncoder.callAsFunction (Encodec.swift:73-87): [B, L, audio_channels] -> z [B, ceil(L / hop), hidden]."""
    h = np.asarray(x, dtype=np.float64)
    for idx, kind, p in encoder_layout(cfg):
        pre = f"encoder.layers.{idx}."
        if kind == "conv":
            h = conv1d(cfg, h, W[pre + "conv.weight"], W[pre + "conv.bias"], stride=p["stride"])
        elif kind == "resnet":
            h = resnet_block(cfg, W, pre, h, p["dilations"])
        elif kind == "elu":
            h = elu(h)
        elif kind == "lstm":
            h = lstm_block(cfg, W, pre, h)
    return h


def num_quantizers_for_bandwidth(cfg: EncodecConfig, bandwidth: Optional[float]) -> int:
    """getNumQuantizersForBandwidth (EncodecQuantization.swift:90-97); float32 arithmetic like the reference's Float."""
    bw_per_q = np.float32(math.log2(cfg.codebook_size)) * np.float32(cfg.frame_rate)
    n = cfg.num_quantizers
    if bandwidth is not None and bandwidth > 0.0:
        n = max(1, int(math.floor(np.float32(bandwidth) * np.float32(1000) / bw_per_q)))
    return n


def rvq_encode(W: Dict[str, np.ndarray], z: np.ndarray, n_q: int, with_gaps: bool = False):
    """EncodecResidualVectorQuantizer.encode (EncodecQuantization.swift:100-115) in float64: z [B, T, D] -> codes [B, n_q, T];
    with_gaps also returns, per level, the gap between the two smallest distances [B, n_q, T]."""
    res = np.asarray(z, dtype=np.float64)
    codes, gaps = [], []
    for q in range(n_q):
        e = W[f"quantizer.layers.{q}.codebook.embed"].astype(np.float64)
        d = (res ** 2).sum(-1, keepdims=True) - 2 * res @ e.T + (e ** 2).sum(1)
        idx = d.argmin(-1)                      # first minimum == the reference's argMax(-dist)
        codes.append(idx.astype(np.int32))
        part = np.partition(d, 1, axis=-1)
        gaps.append(part[..., 1] - part[..., 0])
        res = res - e[idx]
    codes = np.stack(codes, axis=1)
    return (codes, np.stack(gaps, axis=1)) if with_gaps else codes


def ordered_fp32_search(embed: np.ndarray, x: np.ndarray) -> np.ndarray:
    """The device's code search, restated: x [F, D] float32 rows, embed [K, D].  dot, |x|^2 and |e|^2 are each summed over
    d = 0..D-1 as acc = fl(acc + fl(a * b)) (no FMA), dist = fl(fl(xx - 2 dot) + ee), first index of the minimum."""
    x = np.asarray(x, dtype=np.float32)
    e = np.asarray(embed, dtype=np.float32)
    F, D = x.shape
    dot = np.zeros((F, e.shape[0]), np.float32)
    xx = np.zeros((F, 1), np.float32)
    ee = np.zeros((1, e.shape[0]), np.float32)
    for d in range(D):
        dot = dot + x[:, d:d + 1] * e[None, :, d]
        xx = xx + x[:, d:d + 1] * x[:, d:d + 1]
        ee = ee + e[None, :, d] * e[None, :, d]
    dist = (xx - np.float32(2) * dot) + ee
    return dist.argmin(-1).astype(np.int32)


def rvq_encode_fp32(W: Dict[str, np.ndarray], z: np.ndarray, n_q: int) -> np.ndarray:
    """The residual encode with ordered_fp32_search and float32 residual updates: z [B, T, D] float32 -> codes [B, n_q, T]."""
    B, T, D = z.shape
    res = np.asarray(z, dtype=np.float32).reshape(B * T, D).copy()
    codes = []
    for q in range(n_q):
        e = W[f"quantizer.layers.{q}.codebook.embed"].astype(np.float32)
        idx = ordered_fp32_search(e, res)
        codes.append(idx.reshape(B, T))
        res = res - e[idx]
    return np.stack(codes, axis=1)


def chunk_offsets(cfg: EncodecConfig, length: int) -> Tuple[List[int], int]:
    """Encodec.encode's chunk loop (Encodec.swift:267-287): (offsets, chunk length).  Raises ValueError where the reference's
    MLX.stacked would fail: chunks of different lengths (or none)."""
    chunk_len = cfg.chunk_length if cfg.chunk_length is not None else length
    stride = cfg.chunk_stride if cfg.chunk_stride is not None else length
    step = chunk_len - stride
    if cfg.chunk_length is None:
        chunk_len = length
    offsets = list(range(0, max(0, length - step), stride)) if stride > 0 else []
    lens = {min(chunk_len, length - o) for o in offsets}
    if not offsets or len(lens) != 1:
        raise ValueError("chunks of unequal length cannot be stacked")
    return offsets, lens.pop()


def encode_frame(cfg: EncodecConfig, W: Dict[str, np.ndarray], x: np.ndarray, mask: np.ndarray, n_q: int):
    """encodeFrame (Encodec.swift:212-235): x [B, L, C] -> (codes [B, n_q, T], scale [B] or None, z [B, T, D])."""
    v = np.asarray(x, dtype=np.float64)
    scale = None
    if cfg.normalize:
        v = v * mask[..., None]
        mono = v.sum(axis=2, keepdims=True) / v.shape[2]
        scale = np.sqrt((mono ** 2).mean(axis=1, keepdims=True)) + 1e-8
        v = v / scale
    z = encoder(cfg, W, v)
    return rvq_encode(W, z, n_q), (None if scale is None else scale.reshape(-1)), z


def encode(cfg: EncodecConfig, W: Dict[str, np.ndarray], x: np.ndarray, padding_mask: Optional[np.ndarray] = None,
           bandwidth: Optional[float] = None, return_latent: bool = False):
    """Encodec.encode (Encodec.swift:245-291): x [B, L, C] -> (codes [n_chunks, B, n_q, T], scales [n_chunks] of [B] or None);
    return_latent adds the per-chunk z [n_chunks, B, T, D]."""
    bw = cfg.target_bandwidths[0] if bandwidth is None else bandwidth
    if bw not in cfg.target_bandwidths:
        raise ValueError(f"bandwidth {bw} not in {cfg.target_bandwidths}")
    B, L, Cn = x.shape
    if not 1 <= Cn <= 2:
        raise ValueError("audio channels must be 1 or 2")
    n_q = num_quantizers_for_bandwidth(cfg, bw)
    mask = np.ones((B, L), bool) if padding_mask is None else np.asarray(padding_mask, bool)
    offsets, clen = chunk_offsets(cfg, L)
    codes, scales, zs = [], [], []
    for o in offsets:
        c, s, z = encode_frame(cfg, W, x[:, o:o + clen], mask[:, o:o + clen], n_q)
        codes.append(c); scales.append(s); zs.append(z)
    out = (np.stack(codes, 0), scales)
    return (*out, np.stack(zs, 0)) if return_latent else out


def synth_clip(batch: int, n: int, seed: int = 0, channels: int = 1, sr: int = 24000) -> np.ndarray:
    """[B, n, C] float32: 0.5 sin(2 pi 220 t) + 0.1 N(0, 1), seeded."""
    t = np.arange(n) / sr
    rng = np.random.default_rng(seed)
    return (0.5 * np.sin(2 * np.pi * 220.0 * t)[None, :, None] + 0.1 * rng.standard_normal((batch, n, channels))).astype(np.float32)
