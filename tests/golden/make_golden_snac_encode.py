"""Generates tests/golden/snac_encode.npz from the float64 encoder reference (run from the repo root:
`python tests/golden/make_golden_snac_encode.py`).  Kept apart from make_golden.py so that the other fixtures are never
rewritten by it.  Same style: first-N values + mean / abs-mean / min / max of the latent z, plus the codes."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from oracle import snac  # noqa: E402
import snac_encoder_reference as ser  # noqa: E402

OUT = Path(__file__).resolve().parent
N_SAMPLES, BATCH, CLIP_SEED = 5000, 2, 3


def stats(x):
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    return np.array([x.mean(), np.abs(x).mean(), x.min(), x.max()])


def weights():
    cfg = snac.SNACConfig()
    return cfg, {**snac.init_weights(cfg, 1234), **ser.init_encoder_weights(cfg, 4321)}


def main():
    cfg, W = weights()
    audio = ser.synth_clip(BATCH, N_SAMPLES, CLIP_SEED)
    z = ser.encode_latent(cfg, W, audio)
    _, codes = snac.quantize(cfg, W, z)
    np.savez_compressed(OUT / "snac_encode.npz", z_first=z.reshape(-1)[:16].astype(np.float32), z_stats=stats(z),
                        z_shape=np.array(z.shape), **{f"codes{i}": c for i, c in enumerate(codes)})


if __name__ == "__main__":
    main()
