"""Generates tests/golden/snac_44khz.npz from the float64 reference of the 32 / 44 kHz SNAC models (run from the repo root:
`python tests/golden/make_golden_snac_44khz.py`), at the small attention geometry of snac_attention_reference.small() (odd strides,
a zero-padded decoder width, window 16, 2 heads).  First-N values + mean / abs-mean / min / max of the decoded waveform (explicit
noise) and of the encoder's latent, plus the encoded codes."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from oracle import snac  # noqa: E402
import snac_attention_reference as sar  # noqa: E402
import snac_encoder_reference as ser  # noqa: E402

OUT = Path(__file__).resolve().parent
SEED, T_LATENT, BATCH, N_SAMPLES = 11, 32, 2, 700


def stats(x):
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    return np.array([x.mean(), np.abs(x).mean(), x.min(), x.max()])


def inputs():
    cfg = sar.small()
    W = sar.init_weights(cfg, SEED)
    codes = snac.synth_codes(cfg, BATCH, T_LATENT, seed=2)
    rng = np.random.default_rng(5)
    noise = [rng.standard_normal(s).astype(np.float32) for s in sar.noise_shapes(cfg, BATCH, T_LATENT)]
    audio = ser.synth_clip(BATCH, N_SAMPLES, 3, sr=cfg.sampling_rate)
    return cfg, W, codes, noise, audio


def compute():
    cfg, W, codes, noise, audio = inputs()
    y = sar.decode(cfg, W, codes, noise)
    z = sar.encode_latent(cfg, W, audio)
    _, ec = snac.quantize(cfg, W, z)
    return dict(y_first=y.reshape(-1)[:16], y_stats=stats(y), y_shape=np.array(y.shape), z_first=z.reshape(-1)[:16],
                z_stats=stats(z), z_shape=np.array(z.shape), **{f"codes{i}": c for i, c in enumerate(ec)})


def main():
    np.savez_compressed(OUT / "snac_44khz.npz", **compute())


if __name__ == "__main__":
    main()
