"""Generates tests/golden/encodec_encode.npz from the float64 encoder reference (run from the repo root:
`python tests/golden/make_golden_encodec_encode.py`).  Kept apart from make_golden.py so that the other fixtures are never
rewritten by it.  Same style: first-N values + mean / abs-mean / min / max of the latent z, plus the codes."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from oracle import encodec as oe  # noqa: E402
import encodec_encoder_reference as eer  # noqa: E402

OUT = Path(__file__).resolve().parent
N_SAMPLES, BATCH, CLIP_SEED, BANDWIDTH = 5000, 2, 3, 6.0


def stats(x):
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    return np.array([x.mean(), np.abs(x).mean(), x.min(), x.max()])


def weights():
    cfg = oe.EncodecConfig()
    return cfg, {**oe.init_weights(cfg, 7, n_codebooks=8), **eer.init_encoder_weights(cfg, 4321)}


def compute():
    """The 24 kHz geometry at 6 kbps: z [1, B, 16, 128] and codes [1, B, 8, 16]."""
    cfg, W = weights()
    audio = eer.synth_clip(BATCH, N_SAMPLES, CLIP_SEED)
    codes, _, z = eer.encode(cfg, W, audio, bandwidth=BANDWIDTH, return_latent=True)
    return z, codes


def main():
    z, codes = compute()
    np.savez_compressed(OUT / "encodec_encode.npz", z_first=z.reshape(-1)[:16].astype(np.float32), z_stats=stats(z),
                        z_shape=np.array(z.shape), codes=codes)


if __name__ == "__main__":
    main()
