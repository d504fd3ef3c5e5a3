"""float64 reference of the Qwen3-TTS speech-tokenizer ENCODER for the encoder tests and
tests/golden/make_golden_qwen3_encode.py.  Test infrastructure only: the conv primitives and GELU are oracle/qwen3_tts_codec.py's
(conv1d_mlx, extra_padding, gelu_exact).

Follows (paths relative to the reference checkout):
  Sources/MLXAudioTTS/Models/Qwen3TTS/Qwen3TTSSpeechTokenizer.swift:790-884   Qwen3TTSSpeechTokenizerEncoder (init, encode)
  Sources/MLXAudioTTS/Models/Qwen3TTS/Qwen3TTSSpeechTokenizer.swift:1093-1440 sanitize (the encoder keys)
  Sources/MLXAudioCodecs/Mimi/Seanet.swift:157-257, Conv.swift:150-221        SEANet encoder, StreamableConv1d (constant padding)
  Sources/MLXAudioCodecs/Mimi/Transformer.swift:110-369                       pre-norm LayerNorm layers, RoPE(traditional: true)
  Sources/MLXAudioCodecs/Mimi/Conv.swift:333-347                              ConvDownsample1d (k = 2s, no bias, EDGE padding)
  Sources/MLXAudioCodecs/Mimi/Quantization.swift:7-211                        split RVQ encode: argMin(|e|^2/2 - x.e)

Restatement traps (DESIGN.md section N1e):
  1. RoPE is interleaved (pairs 2i, 2i+1) with base Float(Int(rope_theta)); the sanitize concatenates q|k|v rows unpermuted.
     transformers.MimiModel uses rotate-half, so a checkpoint reads the same in both only after its q / k rows are permuted per
     head (hf_qk_permutation).
  2. One-shot encode attends full-causal.  encode() trims every KVCacheSimple to empty and passes the whole clip at once, so in
     Attention.callAsFunction kLen == t and kTargetLen = t + min(context, 0) == kLen: no key is dropped, and the mask is
     createAttentionMask(h:cache:)'s plain causal mask (the pinned mlx-swift-lm returns .causal for a multi-token input and
     applies no window of its own when none is passed).  The sliding_window of 250 never applies.  transformers.MimiModel does
     apply it, so the two agree only up to 250 encoder frames (10 s at 25 Hz).
  3. The SEANet convs pad with zeros, the downsample with the edge value (left pad and right extra pad alike).
  4. The code search distance is c2 - x.e with c2 = |e|^2 / 2 (not |x|^2 - 2 x.e + |e|^2); argMin keeps the lowest index on ties.
"""
from __future__ import annotations

import re
from typing import Dict, List, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle.qwen3_tts_codec import conv1d_mlx, extra_padding, gelu_exact

DT = torch.float64


def synth_clip(B: int, n: int, seed: int = 0) -> np.ndarray:
    """[B, 1, n] float32 test audio: a few partials with a slow envelope plus noise, peak ~0.5."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 24000.0
    out = np.empty((B, 1, n), np.float32)
    for b in range(B):
        f = rng.uniform(80, 2000, 4)
        y = sum(np.sin(2 * np.pi * fi * t + rng.uniform(0, 6.3)) for fi in f) / 4
        y = y * (0.6 + 0.4 * np.sin(2 * np.pi * 1.3 * t + b)) + 0.05 * rng.standard_normal(n)
        out[b, 0] = 0.5 * y
    return out


def encoded_length(n: int, ratios: List[int], ds: int) -> int:
    """StreamableConv1d output lengths chained (Conv.swift:150-156, 205-221): ceil(ceil(n / prod(ratios)) / ds)."""
    L = n
    for r in list(reversed(ratios)) + [ds]:
        L = (L + r + extra_padding(L, 2 * r, r) - 2 * r) // r + 1
    return L


def _t(W, k) -> torch.Tensor:
    return torch.as_tensor(np.asarray(W[k])).to(DT)


def _conv(W, x: torch.Tensor, prefix: str, stride: int = 1, mode: str = "constant") -> torch.Tensor:
    """StreamableConv1d, causal: pad kEff - stride on the left and the extra padding on the right, then the conv."""
    w = _t(W, prefix + ".weight")
    b = _t(W, prefix + ".bias") if prefix + ".bias" in W else None
    k = w.shape[1]
    x = F.pad(x, (k - stride, extra_padding(x.shape[-1], k, stride)), mode=mode)
    return conv1d_mlx(x, w, b, stride)


def seanet(cfg, W, audio) -> torch.Tensor:
    """SeanetEncoder (Seanet.swift:157-257): [B, 1, n] -> [B, hidden, T25] (NCL)."""
    x = _conv(W, torch.as_tensor(np.asarray(audio)).to(DT), "encoder.init_conv1d.conv.conv")
    for i, r in enumerate(reversed(cfg.upsampling_ratios)):
        p = f"encoder.layers.{i}."
        h = _conv(W, F.elu(x), p + "residuals.0.block.0.conv.conv")
        x = x + _conv(W, F.elu(h), p + "residuals.0.block.1.conv.conv")          # trueSkip: identity
        x = _conv(W, F.elu(x), p + "downsample.conv.conv", stride=r)
    return _conv(W, F.elu(x), "encoder.final_conv1d.conv.conv")


def rope_interleaved(x: torch.Tensor, base: float) -> torch.Tensor:
    """MLX RoPE(traditional: true) at offset 0 on [B, heads, T, hd]: frequency i rotates (x[2i], x[2i+1])."""
    hd, T = x.shape[-1], x.shape[-2]
    inv = base ** (-torch.arange(0, hd, 2, dtype=DT) / hd)
    ang = torch.arange(T, dtype=DT)[:, None] * inv[None, :]
    c, s = torch.cos(ang), torch.sin(ang)
    x1, x2 = x[..., 0::2], x[..., 1::2]
    out = torch.empty_like(x)
    out[..., 0::2] = x1 * c - x2 * s
    out[..., 1::2] = x1 * s + x2 * c
    return out


def transformer(cfg, W, x: torch.Tensor, window: int = 0) -> torch.Tensor:
    """The encoder transformer on [B, T, H] (Transformer.swift:110-369); window > 0 additionally drops keys more than `window`
    positions back (what transformers.MimiModel does; the reference's one-shot encode does not, trap 2)."""
    B, T, H = x.shape
    nh = cfg.num_attention_heads
    hd = H // nh
    base = float(int(cfg.rope_theta))
    mask = torch.ones(T, T, dtype=torch.bool).tril()
    if window > 0:
        mask &= ~torch.ones(T, T, dtype=torch.bool).tril(-window)
    for l in range(cfg.num_hidden_layers):
        p = f"encoder_transformer.transformer.layers.{l}."
        h = F.layer_norm(x, (H,), _t(W, p + "norm1.weight"), _t(W, p + "norm1.bias"), 1e-5)
        qkv = (h @ _t(W, p + "self_attn.in_proj.weight").T).reshape(B, T, 3, nh, hd)
        q, k, v = (qkv[:, :, i].transpose(1, 2) for i in range(3))
        q, k = rope_interleaved(q, base), rope_interleaved(k, base)
        s = (q @ k.transpose(-1, -2)) / np.sqrt(hd)
        a = torch.softmax(s.masked_fill(~mask, float("-inf")), -1) @ v
        a = a.transpose(1, 2).reshape(B, T, H) @ _t(W, p + "self_attn.out_proj.weight").T
        x = x + _t(W, p + "layer_scale_1.scale") * a
        h = F.layer_norm(x, (H,), _t(W, p + "norm2.weight"), _t(W, p + "norm2.bias"), 1e-5)
        m = gelu_exact(h @ _t(W, p + "gating.linear1.weight").T) @ _t(W, p + "gating.linear2.weight").T
        x = x + _t(W, p + "layer_scale_2.scale") * m
    return x


def latent(cfg, W, audio, window: int = 0) -> np.ndarray:
    """z [B, T, hidden]: SEANet -> transformer -> edge-padded downsample (the code search's input)."""
    x = seanet(cfg, W, audio).transpose(1, 2)
    x = transformer(cfg, W, x, window).transpose(1, 2)
    z = _conv(W, x, "downsample.conv.conv.conv", stride=cfg.downsample_stride, mode="replicate")
    return z.transpose(1, 2).numpy()


def codebook(W, name: str, i: int) -> np.ndarray:
    p = f"quantizer.{name}.vq.layers.{i}.codebook."
    return np.asarray(W[p + "embedding_sum"], np.float64) / np.maximum(np.asarray(W[p + "cluster_usage"], np.float64), 1e-5)[:, None]


def _levels(cfg, W):
    G = cfg.num_code_groups
    return [("rvq_first", 0)] + [("rvq_rest", i) for i in range(G - 1)]


def encode_codes(cfg, W, z: np.ndarray, with_gaps: bool = False):
    """Split RVQ encode in float64 on z [B, T, H] -> codes [B, G, T] (and, per level, the gap between the best and second-best
    distance and |residual|^2 + 1, for near-tie checks)."""
    z = np.asarray(z, np.float64)
    B, T, _ = z.shape
    G = cfg.num_code_groups
    codes = np.zeros((B, G, T), np.int32)
    gaps, scale = np.zeros((B, G, T)), np.zeros((B, G, T))
    xf = z @ np.asarray(W["quantizer.rvq_first.input_proj.weight"], np.float64)[:, 0, :].T
    res = z @ np.asarray(W["quantizer.rvq_rest.input_proj.weight"], np.float64)[:, 0, :].T if G > 1 else None
    for q, (name, i) in enumerate(_levels(cfg, W)):
        e = codebook(W, name, i)
        x = xf if q == 0 else res
        d = 0.5 * (e ** 2).sum(-1)[None, None, :] - x @ e.T
        idx = np.argmin(d, -1)
        codes[:, q] = idx
        srt = np.sort(d, -1)
        gaps[:, q] = srt[..., 1] - srt[..., 0]
        scale[:, q] = (x ** 2).sum(-1) + 1.0
        if q > 0:
            res = res - e[idx]
    return (codes, gaps, scale) if with_gaps else codes


def encode_codes_fp32(cfg, W, z: np.ndarray) -> np.ndarray:
    """The device's ordered-fp32 contract on z [B, T, H]: both input projections and every dot summed over d in order as
    acc = fl(acc + fl(a * b)); c2 = fl(ordered |e|^2) / 2; dist = fl(c2 - dot); lowest index on ties; residual -= e[idx]."""
    z = np.asarray(z, np.float32)
    B, T, H = z.shape
    G = cfg.num_code_groups
    rows = z.reshape(-1, H)

    def proj(w):
        w = np.asarray(w, np.float32)[:, 0, :]
        acc = np.zeros((rows.shape[0], w.shape[0]), np.float32)
        for d in range(H):
            acc = acc + rows[:, d:d + 1] * w[None, :, d]
        return acc

    xf = proj(W["quantizer.rvq_first.input_proj.weight"])
    res = proj(W["quantizer.rvq_rest.input_proj.weight"]) if G > 1 else None
    codes = np.zeros((rows.shape[0], G), np.int32)
    for q, (name, i) in enumerate(_levels(cfg, W)):
        p = f"quantizer.{name}.vq.layers.{i}.codebook."
        e = (np.asarray(W[p + "embedding_sum"], np.float32) / np.maximum(np.asarray(W[p + "cluster_usage"], np.float32), np.float32(1e-5))[:, None]).astype(np.float32)
        c2 = np.zeros(e.shape[0], np.float32)
        for d in range(e.shape[1]):
            c2 = c2 + e[:, d] * e[:, d]
        c2 = c2 * np.float32(0.5)
        x = xf if q == 0 else res
        dot = np.zeros((x.shape[0], e.shape[0]), np.float32)
        for d in range(e.shape[1]):
            dot = dot + x[:, d:d + 1] * e[None, :, d]
        idx = np.argmin(c2[None, :] - dot, -1)
        codes[:, q] = idx
        if q > 0:
            res = res - e[idx]
    return codes.reshape(B, T, G).transpose(0, 2, 1).copy()


# ---------------------------------------------------------------- sanitize (the encoder half), restated
_CONV_MAP = {0: "encoder.init_conv1d", 3: "encoder.layers.0.downsample", 6: "encoder.layers.1.downsample",
             9: "encoder.layers.2.downsample", 12: "encoder.layers.3.downsample", 14: "encoder.final_conv1d"}
_RES_LAYER = {1: 0, 4: 1, 7: 2, 10: 3}
_RES_BLOCK = {1: 0, 3: 1}
_TLAYER = [("self_attn.out_proj.weight", "self_attn.out_proj.weight"), ("self_attn.o_proj.weight", "self_attn.out_proj.weight"),
           ("mlp.fc1.weight", "gating.linear1.weight"), ("mlp.fc2.weight", "gating.linear2.weight"),
           ("input_layernorm.weight", "norm1.weight"), ("input_layernorm.bias", "norm1.bias"),
           ("post_attention_layernorm.weight", "norm2.weight"), ("post_attention_layernorm.bias", "norm2.bias"),
           ("self_attn_layer_scale.scale", "layer_scale_1.scale"), ("mlp_layer_scale.scale", "layer_scale_2.scale")]


def _quant_prefix(rest: str, contains: bool) -> str:
    test = (lambda x: x in rest) if contains else rest.startswith
    return "quantizer.rvq_first" if test("semantic_residual_vector_quantizer") or test("rvq_first.") else "quantizer.rvq_rest"


def sanitize_encoder(weights: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    """Qwen3TTSSpeechTokenizer.sanitize (:1093-1440), the encoder keys, without the "encoder_model." prefix and without the
    codebooks' "initialized" flags.  PyTorch-layout checkpoint -> MLX layouts."""
    out: Dict[str, np.ndarray] = {}
    qkv: Dict[int, Dict[str, np.ndarray]] = {}
    books: Dict[str, Dict[str, np.ndarray]] = {}
    for raw, v in weights.items():
        k = raw
        while True:
            for p in ("speech_tokenizer.", "encoder_model.", "decoder_model."):
                if k.startswith(p):
                    k = k[len(p):]
                    break
            else:
                break
        parts = k.split(".")
        if k in ("", "encoder_model", "decoder_model", "speech_tokenizer") or ("speaker_encoder" in parts and parts.index("speaker_encoder") + 1 < len(parts)):
            continue
        if "_codebook.cluster_usage" in k or "_codebook.embedding_sum" in k or "_codebook.initialized" in k or ".codebook.initialized" in k:
            continue
        if not k.startswith("encoder."):
            continue
        v = np.asarray(v)
        if k.startswith("encoder.encoder.layers."):
            if len(parts) < 4 or not parts[3].isdigit():
                continue
            n = int(parts[3])
            if ".block." in k:
                if n not in _RES_LAYER or len(parts) <= 5 or not parts[5].isdigit() or int(parts[5]) not in _RES_BLOCK:
                    continue
                key = f"encoder.layers.{_RES_LAYER[n]}.residuals.0.block.{_RES_BLOCK[int(parts[5])]}.conv." + ".".join(parts[6:])
            elif n in _CONV_MAP:
                key = _CONV_MAP[n] + ".conv." + ".".join(parts[4:])
            else:
                continue
            out[key] = np.ascontiguousarray(v.transpose(0, 2, 1)) if key.endswith("weight") and v.ndim == 3 else v
        elif k.startswith("encoder.encoder_transformer.layers.") or k.startswith("encoder.encoder_transformer.transformer.layers."):
            off = 4 if len(parts) >= 5 and parts[2] == "transformer" and parts[3] == "layers" else 3
            if len(parts) <= off or not parts[off].isdigit():
                continue
            l, sfx = int(parts[off]), ".".join(parts[off + 1:])
            p = f"encoder_transformer.transformer.layers.{l}."
            for n in "qkv":
                if f"self_attn.{n}_proj.weight" in sfx:
                    qkv.setdefault(l, {})[n] = v
                    break
            else:
                if "self_attn.qkv.weight" in sfx and v.ndim == 2:
                    third = v.shape[0] // 3
                    if v.shape[0] % 3 == 0 and third > 0:
                        for i, n in enumerate("qkv"):
                            qkv.setdefault(l, {})[n] = v[i * third:(i + 1) * third]
                    continue
                for src, dst in _TLAYER:
                    if src in sfx:
                        out[p + dst] = v
                        break
        elif k.startswith("encoder.downsample."):
            sfx = k[len("encoder.downsample."):]
            out["downsample.conv.conv." + sfx] = np.ascontiguousarray(v.transpose(0, 2, 1)) if sfx.endswith("weight") and v.ndim == 3 else v
        elif k.startswith("encoder.quantizer."):
            rest = k[len("encoder.quantizer."):]
            if ".codebook.embed.weight" in rest or rest.endswith("codebook.embed"):
                continue
            if "codebook.cluster_usage" in rest or "codebook.embed_sum" in rest or "codebook.embedding_sum" in rest:
                base = rest[: rest.rfind(".codebook.")] if ".codebook." in rest else rest
                books.setdefault(base, {})["cluster_usage" if "cluster_usage" in rest else "embedding_sum"] = v
                continue
            if "codebook.initialized" in rest:
                continue
            if "input_proj.weight" in rest or "output_proj.weight" in rest:
                if rest.endswith("weight") and v.ndim == 3:
                    v = np.ascontiguousarray(v.transpose(0, 2, 1))
                out[_quant_prefix(rest, False) + (".input_proj.weight" if "input_proj" in rest else ".output_proj.weight")] = v
            if "codebook." not in rest and (rest.startswith("layers.") or ".layers." in rest):
                for pre, grp in (("rvq_first.", "rvq_first"), ("rvq_rest.", "rvq_rest"), ("semantic_residual_vector_quantizer.", "rvq_first"),
                                 ("acoustic_residual_vector_quantizer.", "rvq_rest")):
                    if rest.startswith(pre):
                        out[f"quantizer.{grp}.vq." + rest[len(pre):]] = v
                        break
                else:
                    if rest.startswith("layers."):
                        out["quantizer.rvq_rest.vq." + rest] = v
    for l, d in qkv.items():
        if all(n in d for n in "qkv"):
            out[f"encoder_transformer.transformer.layers.{l}.self_attn.in_proj.weight"] = np.concatenate([d["q"], d["k"], d["v"]], 0)
    for base, d in books.items():
        m = re.search(r"(?:^|\.)layers\.(\d+)(?:\.|$)", base)
        if "cluster_usage" in d and "embedding_sum" in d and m:
            p = _quant_prefix(base, True) + f".vq.layers.{int(m.group(1))}.codebook."
            out[p + "cluster_usage"], out[p + "embedding_sum"] = d["cluster_usage"], d["embedding_sum"]
    return out


def hf_qk_permutation(n_heads: int, head_dim: int) -> np.ndarray:
    """Row order that turns a rotate-half q / k projection into the interleaved one: new row h*hd + 2i (+1) = old row
    h*hd + i (+ hd/2)."""
    half = head_dim // 2
    idx = np.empty(n_heads * head_dim, np.int64)
    for h in range(n_heads):
        for i in range(half):
            idx[h * head_dim + 2 * i] = h * head_dim + i
            idx[h * head_dim + 2 * i + 1] = h * head_dim + i + half
    return idx
