"""float64 reference of the SNAC encode path (SNACDecoder.swift:86-105,120-125; Layers.swift:236-259,319-360) for the encoder
tests and tests/golden/make_golden_snac_encode.py.  Test infrastructure only: it is built from oracle.snac's primitives
(wn_conv1d, residual_unit, snake, quantize), so the encoder follows exactly the layer semantics the decoder tests pin.

Weights use the checkpoint's keys (MLX ``Sequential`` naming, conv layout ``[out, k, in/groups]``):
  encoder.block.layers.0                         stem WNConv1d(1 -> d, k7, pad 3)
  encoder.block.layers.{1..n}.block.layers.{0,1,2}  ResidualUnits (dil 1, 3, 9), the decoder's inner keys
  encoder.block.layers.{1..n}.block.layers.3.alpha  Snake
  encoder.block.layers.{1..n}.block.layers.4     WNConv1d(C -> 2C, k 2s, stride s, pad ceil(s/2))
  encoder.block.layers.{n+1}                     WNConv1d(latent -> latent, k7, pad 3, groups latent when depthwise)
"""
from __future__ import annotations

import math
from typing import Dict, List

import numpy as np
import torch

from oracle import snac
from oracle.snac import SNACConfig


def init_encoder_weights(cfg: SNACConfig, seed: int = 4321) -> Dict[str, np.ndarray]:
    """Random-init encoder weights (``encoder.*`` keys only; merge with ``snac.init_weights`` for a full codec), drawn like
    ``snac.init_weights``: conv v ~ U(+-1/sqrt(fan_in)), g = ||v|| perturbed, small biases, Snake alpha ~ U(0.5, 1.5)."""
    rng = np.random.default_rng(seed)
    w: Dict[str, np.ndarray] = {}

    def wn(prefix, shape, fan):
        s = math.sqrt(1.0 / fan)
        v = rng.uniform(-s, s, size=shape).astype(np.float32)
        g = np.sqrt((v.astype(np.float64) ** 2).sum(axis=(1, 2), keepdims=True))
        w[prefix + ".weight_v"] = v
        w[prefix + ".weight_g"] = (g * rng.uniform(0.8, 1.2, size=g.shape)).astype(np.float32)
        w[prefix + ".bias"] = rng.uniform(-0.05, 0.05, size=shape[0]).astype(np.float32)

    p = "encoder.block.layers"
    d = cfg.encoder_dim
    wn(f"{p}.0", (d, 7, 1), 7)
    for i, s in enumerate(cfg.encoder_rates):
        b = f"{p}.{i + 1}.block.layers"
        g = d if cfg.depthwise else 1
        for j in range(3):
            r = f"{b}.{j}.block.layers"
            w[f"{r}.0.alpha"] = rng.uniform(0.5, 1.5, size=(1, d, 1)).astype(np.float32)
            wn(f"{r}.1", (d, 7, d // g), 7 * (d // g))
            w[f"{r}.2.alpha"] = rng.uniform(0.5, 1.5, size=(1, d, 1)).astype(np.float32)
            wn(f"{r}.3", (d, 1, d), d)
        w[f"{b}.3.alpha"] = rng.uniform(0.5, 1.5, size=(1, d, 1)).astype(np.float32)
        wn(f"{b}.4", (2 * d, 2 * s, d), 2 * s * d)
        d *= 2
    wn(f"{p}.{len(cfg.encoder_rates) + 1}", (d, 7, 1 if cfg.depthwise else d), 7 * (1 if cfg.depthwise else d))
    return w


def pad_multiple(cfg: SNACConfig) -> int:
    """SNACDecoder.swift:86-100: audio is right-padded to a multiple of hop_length * lcm(vq_strides)."""
    assert cfg.attn_window_size is None, "LocalMHA only exists in the 32/44 kHz models"
    return cfg.hop_length * math.lcm(*cfg.vq_strides)


def preprocess(cfg: SNACConfig, x: np.ndarray) -> np.ndarray:
    """SNACDecoder.swift:86-105: zero right-padding of [B, 1, n] to the next multiple of pad_multiple(cfg)."""
    n, m = x.shape[-1], pad_multiple(cfg)
    return np.pad(x, [(0, 0)] * (x.ndim - 1) + [(0, -(-n // m) * m - n)])


def encoder_blocks(cfg: SNACConfig, w: Dict, x: torch.Tensor) -> torch.Tensor:
    """Stem + the EncoderBlocks (Layers.swift:236-259, 328-337): [B, 1, n] -> [B, latent, n / hop]."""
    p = "encoder.block.layers"
    x = snac.wn_conv1d(w, f"{p}.0", x, padding=3)
    d = cfg.encoder_dim
    for i, s in enumerate(cfg.encoder_rates):
        b = f"{p}.{i + 1}.block.layers"
        for j, dil in enumerate((1, 3, 9)):
            x = snac.residual_unit(w, f"{b}.{j}", x, dil, d if cfg.depthwise else 1)
        x = snac.snake(x, snac._t(w[f"{b}.3.alpha"]))
        x = snac.wn_conv1d(w, f"{b}.4", x, stride=s, padding=math.ceil(s / 2))
        d *= 2
    return x


def encoder(cfg: SNACConfig, w: Dict, x: torch.Tensor) -> torch.Tensor:
    """Layers.swift:319-360 (Encoder, no LocalMHA): [B, 1, n] -> z [B, latent, n / hop]."""
    assert cfg.attn_window_size is None, "LocalMHA only exists in the 32/44 kHz models"
    d = cfg.encoder_dim * 2 ** len(cfg.encoder_rates)
    return snac.wn_conv1d(w, f"encoder.block.layers.{len(cfg.encoder_rates) + 1}", encoder_blocks(cfg, w, x), padding=3,
                          groups=d if cfg.depthwise else 1)


def encode_latent(cfg: SNACConfig, w: Dict, audio: np.ndarray) -> np.ndarray:
    """preprocess -> encoder: audio [B, 1, n] -> z [B, latent, t_latent] float64."""
    with torch.no_grad():
        return encoder(cfg, w, snac._t(preprocess(cfg, np.asarray(audio)))).numpy()


def encode(cfg: SNACConfig, w: Dict, audio: np.ndarray) -> List[np.ndarray]:
    """SNACDecoder.swift:120-125 (SNAC.encode): audio [B, 1, n] -> codes [B, t_latent / stride_i]."""
    return snac.quantize(cfg, w, encode_latent(cfg, w, audio))[1]


def synth_clip(batch: int, n: int, seed: int = 0, sr: int = 24000) -> np.ndarray:
    """[B, 1, n] float32: 0.5 sin(2 pi 220 t) + 0.1 N(0, 1), seeded (the encode benchmark's signal)."""
    t = np.arange(n) / sr
    rng = np.random.default_rng(seed)
    return (0.5 * np.sin(2 * np.pi * 220.0 * t)[None, None] + 0.1 * rng.standard_normal((batch, 1, n))).astype(np.float32)


def prepare_input_ids_ref(prompts: List[List[int]], ref_text_ids: List[int], ref_code_list: List[int]) -> np.ndarray:
    """LlamaTTS.swift:446-553 with refAudio / refText: per row padding, then
    [SOH] refText [EOT EOH] [audioStart SOS] codes + 128266 [EOS audioEnd], then [SOH] prompt [EOT EOH]."""
    soh, eot, eoh, sos, eos, pad, a_start, a_end, off = 128259, 128009, 128260, 128257, 128258, 128263, 128261, 128262, 128266
    ref = [soh] + list(ref_text_ids) + [eot, eoh] + [a_start, sos] + [c + off for c in ref_code_list] + [eos, a_end]
    mx = max(len(p) for p in prompts)
    return np.asarray([[pad] * (mx - len(p)) + ref + [soh] + list(p) + [eot, eoh] for p in prompts], dtype=np.int32)
