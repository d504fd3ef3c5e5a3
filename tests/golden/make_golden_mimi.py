"""Writes tests/golden/mimi.npz from the float64 oracle (oracle/mimi.py) at the small test geometry: a one-shot decode and a
frame-by-frame stream of 140 code frames (past the 125-frame attention window, where the two differ), every STRIDE-th sample, and
the codes of a 1.5 s clip.  Run from the repository root: python tests/golden/make_golden_mimi.py"""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

from oracle import mimi as om  # noqa: E402

SEED, CODE_SEED, CLIP_SEED, FRAMES, STRIDE = 21, 22, 23, 140, 97


def inputs():
    cfg = om.small_config()
    W = om.init_weights(cfg, SEED)
    codes = np.random.default_rng(CODE_SEED).integers(0, cfg.codebook_size, (1, cfg.num_codebooks, FRAMES)).astype(np.int32)
    return cfg, W, codes


def clip():
    import qwen3_encoder_reference as qer
    return qer.synth_clip(1, 36000, CLIP_SEED)


if __name__ == "__main__":
    cfg, W, codes = inputs()
    one = om.decode(cfg, W, codes)
    stream = om.MimiStreamer(cfg, W).decode_frames(codes)
    np.savez_compressed(Path(__file__).with_name("mimi.npz"), codes_in=codes, decode=one[..., ::STRIDE].astype(np.float64),
                        stream=stream[..., ::STRIDE].astype(np.float64), codes=om.encode(cfg, W, clip()))
    print("wrote mimi.npz")
