"""Generates tests/golden/encodec_48khz.npz from the float64 time_group_norm reference (run from the repo root:
`python tests/golden/make_golden_encodec_48khz.py`).  Kept apart from the other generators so that their fixtures are never
rewritten by it.  Same style as make_golden_encodec_encode.py: first / last values + mean / abs-mean / min / max of a 48 kHz-geometry
decode (two 1 s chunks with scales), and the latent z, codes and scales of a short stereo encode."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import encodec_encoder_reference as eer  # noqa: E402
import encodec_gn_reference as gnr  # noqa: E402

OUT = Path(__file__).resolve().parent
CODE_SEED, N_CHUNKS, N_Q, FRAMES = 1, 2, 4, 150
DECODE_SCALES = (0.5, 2.0)
N_SAMPLES, BATCH, CLIP_SEED, BANDWIDTH = 5000, 2, 3, 6.0


def stats(x):
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    return np.array([x.mean(), np.abs(x).mean(), x.min(), x.max()])


def weights():
    cfg = gnr.config_48khz()
    return cfg, gnr.weights(cfg, 16, seed=7)


def decode_inputs():
    codes = np.random.default_rng(CODE_SEED).integers(0, 1024, size=(N_CHUNKS, 1, N_Q, FRAMES)).astype(np.int32)
    return codes, [np.array([s], np.float32) for s in DECODE_SCALES]


def compute():
    """y [1, 95520, 2] of the chunked decode; z [1, B, 16, 128], codes [1, B, 4, 16] and scales [1, B] of the encode."""
    cfg, W = weights()
    codes, scales = decode_inputs()
    y = gnr.decode(cfg, W, codes, scales)
    audio = eer.synth_clip(BATCH, N_SAMPLES, CLIP_SEED, channels=2, sr=48000)
    audio[1] *= 0.3
    c, s, z = gnr.encode(cfg, W, audio, bandwidth=BANDWIDTH)
    return y, z, c, np.stack(s)


def main():
    y, z, codes, scales = compute()
    np.savez_compressed(OUT / "encodec_48khz.npz", y_first=y[:, :64].reshape(-1).astype(np.float32),
                        y_last=y[:, -64:].reshape(-1).astype(np.float32), y_stats=stats(y), y_shape=np.array(y.shape),
                        z_first=z.reshape(-1)[:16].astype(np.float32), z_stats=stats(z), z_shape=np.array(z.shape), codes=codes,
                        scales=scales)


if __name__ == "__main__":
    main()
