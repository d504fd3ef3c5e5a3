"""float64 reference of the 32 / 44 kHz SNAC models (LocalMHA, odd strides) for tests/test_oracle_snac_44khz.py,
tests/test_gpu_snac_44khz.py and tests/golden/make_golden_snac_44khz.py.  Test infrastructure only: composed from oracle.snac's
layers and snac_encoder_reference's encoder blocks, so everything but LocalMHA follows the semantics the 24 kHz tests pin.

LocalMHA (Attention.swift:14-95), keys <prefix>.norm.weight|bias, .to_qkv.weight [3 dim, dim], .to_out.weight [dim, dim] (no
biases), .rel_pos.inv_freq [32]:
  LayerNorm(dim, eps 1e-5) over channels -> q | k | v -> heads of 64 over windows of `window` consecutive frames -> rotary with
  angles pos * inv_freq, pos = 0 .. window - 1 within each window, [freqs, freqs] -> softmax(q k^T / 8) v -> to_out -> + residual.
  The reference's rotateHalf keeps an extra unit axis and cannot run as written (DESIGN.md 3.2c); this is the only reading under
  which its next line is well-formed: standard rotate-half, cat(-x[d/2:], x[:d/2]).
Placement: decoder.model.layers.2 (after the depthwise + 1x1 input convs; DecoderBlocks then start at 3) and
encoder.block.layers.{n+1} (after the last EncoderBlock; the final depthwise conv moves to n + 2).
Transposed convs keep oracle.snac's F.conv_transpose1d(..., output_padding=0): the reference drops DecoderBlock's outputPadding, so
a stage of odd stride s yields s T - 1 frames.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

import snac_encoder_reference as ser
from oracle import snac
from oracle.snac import SNACConfig

HEAD = 64


def init_attn_weights(prefix: str, dim: int, rng: np.random.Generator) -> Dict[str, np.ndarray]:
    """LocalMHA weights drawn like oracle.snac.init_weights: projections U(+-1/sqrt(dim)), LayerNorm gain U(0.8, 1.2) and small
    shift, inv_freq = 1 / 10000^(2i / 64) (SinusoidalEmbeddings)."""
    s = math.sqrt(1.0 / dim)
    return {
        prefix + ".norm.weight": rng.uniform(0.8, 1.2, size=dim).astype(np.float32),
        prefix + ".norm.bias": rng.uniform(-0.05, 0.05, size=dim).astype(np.float32),
        prefix + ".to_qkv.weight": rng.uniform(-s, s, size=(3 * dim, dim)).astype(np.float32),
        prefix + ".to_out.weight": rng.uniform(-s, s, size=(dim, dim)).astype(np.float32),
        prefix + ".rel_pos.inv_freq": (1.0 / 10000.0 ** (np.arange(0, HEAD, 2) / HEAD)).astype(np.float32),
    }


def init_weights(cfg: SNACConfig, seed: int = 1234, encoder: bool = True) -> Dict[str, np.ndarray]:
    """A full attention codec: oracle.snac.init_weights' decoder + quantizer with the DecoderBlocks shifted up by one behind
    LocalMHA, snac_encoder_reference's encoder with its final conv shifted behind LocalMHA.  The attention tensors come from their
    own generator (seed + 7)."""
    base = snac.init_weights(SNACConfig(**{**cfg.__dict__, "attn_window_size": None}), seed)
    w: Dict[str, np.ndarray] = {}
    p = "decoder.model.layers."
    for k, v in base.items():
        if k.startswith(p):
            i, rest = k[len(p):].split(".", 1)
            k = p + str(int(i) + (1 if int(i) >= 2 else 0)) + "." + rest
        w[k] = v
    rng = np.random.default_rng(seed + 7)
    w.update(init_attn_weights(p + "2", cfg.decoder_dim, rng))
    if encoder:
        n = len(cfg.encoder_rates)
        e = ser.init_encoder_weights(SNACConfig(**{**cfg.__dict__, "attn_window_size": None}), seed + 3)
        fin = f"encoder.block.layers.{n + 1}."
        w.update({(f"encoder.block.layers.{n + 2}." + k[len(fin):] if k.startswith(fin) else k): v for k, v in e.items()})
        w.update(init_attn_weights(f"encoder.block.layers.{n + 1}", cfg.latent, rng))
    return w


def rotate_half(x: torch.Tensor) -> torch.Tensor:
    h = x.shape[-1] // 2
    return torch.cat([-x[..., h:], x[..., :h]], dim=-1)


def local_mha(w: Dict, prefix: str, x: torch.Tensor, window: int) -> torch.Tensor:
    """Attention.swift:33-64 on x [B, C, T] (T a multiple of window) -> [B, C, T]."""
    B, C, T = x.shape
    H, Wn = C // HEAD, T // window
    h = F.layer_norm(x.transpose(1, 2), (C,), snac._t(w[prefix + ".norm.weight"]), snac._t(w[prefix + ".norm.bias"]), eps=1e-5)
    qkv = h @ snac._t(w[prefix + ".to_qkv.weight"]).T

    def heads(t):                                                   # b (w n) (h d) -> b h w n d
        return t.reshape(B, Wn, window, H, HEAD).permute(0, 3, 1, 2, 4)

    q, k, v = (heads(t) for t in qkv.split(C, dim=-1))
    pos = torch.arange(window, dtype=snac.DTYPE)
    freqs = pos[:, None] * snac._t(w[prefix + ".rel_pos.inv_freq"])[None]
    freqs = torch.cat([freqs, freqs], dim=-1)                       # [window, 64]
    q = q * freqs.cos() + rotate_half(q) * freqs.sin()
    k = k * freqs.cos() + rotate_half(k) * freqs.sin()
    att = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(HEAD), dim=-1) @ v
    out = att.permute(0, 2, 3, 1, 4).reshape(B, T, C) @ snac._t(w[prefix + ".to_out.weight"]).T
    return out.transpose(1, 2) + x


def stage_lengths(cfg: SNACConfig, t_latent: int) -> List[int]:
    """Frames out of each DecoderBlock: F.conv_transpose1d with k = 2s, pad = ceil(s/2), output_padding 0 gives s T - (s mod 2)."""
    out, t = [], t_latent
    for s in cfg.decoder_rates:
        t = (t - 1) * s - 2 * math.ceil(s / 2) + 2 * s
        out.append(t)
    return out


def noise_shapes(cfg: SNACConfig, batch: int, t_latent: int) -> List[tuple]:
    return [(batch, 1, t) for t in stage_lengths(cfg, t_latent)]


def decoder(cfg: SNACConfig, w: Dict, z: torch.Tensor, noise: Optional[List[np.ndarray]]) -> torch.Tensor:
    """Layers.swift:364-421 with LocalMHA when cfg.attn_window_size (depthwise decoders): z [B, latent, T] -> [B, 1, samples]."""
    assert cfg.depthwise
    p = "decoder.model.layers"
    x = snac.wn_conv1d(w, f"{p}.0", z, padding=3, groups=cfg.latent)
    x = snac.wn_conv1d(w, f"{p}.1", x)
    li = 2
    if cfg.attn_window_size:
        x = local_mha(w, f"{p}.2", x, cfg.attn_window_size)
        li = 3
    for i, s in enumerate(cfg.decoder_rates):
        cout = cfg.decoder_dim // 2 ** (i + 1)
        b = f"{p}.{li}.block.layers"
        x = snac.snake(x, snac._t(w[f"{b}.0.alpha"]))
        x = snac.wn_conv_transpose1d(w, f"{b}.1", x, stride=s, padding=math.ceil(s / 2))
        j = 2
        if cfg.noise:
            h = snac.wn_conv1d(w, f"{b}.2.linear", x)
            if noise is not None and noise[i] is not None:
                x = x + snac._t(noise[i]) * h
            j = 3
        for dil in (1, 3, 9):
            x = snac.residual_unit(w, f"{b}.{j}", x, dil, cout)
            j += 1
        li += 1
    x = snac.snake(x, snac._t(w[f"{p}.{li}.alpha"]))
    x = snac.wn_conv1d(w, f"{p}.{li + 1}", x, padding=3)
    return torch.tanh(x)


def decode(cfg: SNACConfig, w: Dict, codes: List[np.ndarray], noise: Optional[List[np.ndarray]] = None) -> np.ndarray:
    """SNACDecoder.swift:127-131 -> waveform [B, 1, stage_lengths(T)[-1]] float64."""
    with torch.no_grad():
        return decoder(cfg, w, snac.from_codes(cfg, w, codes), noise).numpy()


def pad_multiple(cfg: SNACConfig) -> int:
    """SNACDecoder.swift:86-100: hop_length * lcm(vq_strides, attn_window_size)."""
    return cfg.hop_length * math.lcm(*cfg.vq_strides, *([cfg.attn_window_size] if cfg.attn_window_size else []))


def preprocess(cfg: SNACConfig, x: np.ndarray) -> np.ndarray:
    n, m = x.shape[-1], pad_multiple(cfg)
    return np.pad(x, [(0, 0)] * (x.ndim - 1) + [(0, -(-n // m) * m - n)])


def encoder(cfg: SNACConfig, w: Dict, x: torch.Tensor) -> torch.Tensor:
    """Layers.swift:319-360: [B, 1, n] -> z [B, latent, n / hop]."""
    n = len(cfg.encoder_rates)
    x = ser.encoder_blocks(cfg, w, x)
    f = n + 1
    if cfg.attn_window_size:
        x = local_mha(w, f"encoder.block.layers.{n + 1}", x, cfg.attn_window_size)
        f = n + 2
    return snac.wn_conv1d(w, f"encoder.block.layers.{f}", x, padding=3, groups=cfg.latent if cfg.depthwise else 1)


def encode_latent(cfg: SNACConfig, w: Dict, audio: np.ndarray) -> np.ndarray:
    """preprocess -> encoder: audio [B, 1, n] -> z [B, latent, t_latent] float64."""
    with torch.no_grad():
        return encoder(cfg, w, snac._t(preprocess(cfg, np.asarray(audio)))).numpy()


def encode(cfg: SNACConfig, w: Dict, audio: np.ndarray) -> List[np.ndarray]:
    return snac.quantize(cfg, w, encode_latent(cfg, w, audio))[1]


# the released 32 / 44 kHz geometry (model cards), and the small one the tests and the golden run
def published(sampling_rate: int = 44100) -> SNACConfig:
    return SNACConfig(sampling_rate=sampling_rate, encoder_dim=64, encoder_rates=(2, 3, 8, 8), decoder_dim=1536,
                      decoder_rates=(8, 8, 3, 2), attn_window_size=32, codebook_size=4096, codebook_dim=8, vq_strides=(8, 4, 2, 1))


def small() -> SNACConfig:
    """Odd strides in the encoder (3) and the decoder (3), a decoder stage of 96 channels (run zero-padded to 128), window 16,
    2 heads in both LocalMHA blocks."""
    return SNACConfig(sampling_rate=44100, encoder_dim=16, encoder_rates=(3, 2, 2), decoder_dim=384, decoder_rates=(2, 3, 2),
                      attn_window_size=16, codebook_size=256, codebook_dim=8, vq_strides=(4, 2, 1))
