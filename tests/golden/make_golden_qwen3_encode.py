"""Generates tests/golden/qwen3_encode.npz from the float64 Qwen3-TTS speech-tokenizer encoder reference (run from the repo root:
`python tests/golden/make_golden_qwen3_encode.py`).  Kept apart from make_golden.py so that the other fixtures are never
rewritten by it.  Tiny geometry; first-N values + mean / abs-mean / min / max of the latent z, plus the codes."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import qwen3_encoder_reference as qer  # noqa: E402
from mlx_audio_swift_b200.qwen3_tts_codec import Qwen3TTSTokenizerEncoderConfig, random_init_encoder_weights  # noqa: E402

OUT = Path(__file__).resolve().parent
N_SAMPLES, BATCH, CLIP_SEED = 9000, 2, 5


def stats(x):
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    return np.array([x.mean(), np.abs(x).mean(), x.min(), x.max()])


def weights():
    cfg = Qwen3TTSTokenizerEncoderConfig(hidden_size=64, num_filters=8, num_attention_heads=2, num_key_value_heads=2, intermediate_size=128,
                                         num_hidden_layers=2, codebook_size=64, codebook_dim=16, num_quantizers=8, valid_num_quantizers=8)
    return cfg, random_init_encoder_weights(cfg, seed=77, layer_scale=0.3)


def compute():
    """z [B, 5, 64] and codes [B, 8, 5]."""
    cfg, W = weights()
    z = qer.latent(cfg, W, qer.synth_clip(BATCH, N_SAMPLES, CLIP_SEED))
    return z, qer.encode_codes(cfg, W, z)


def main():
    z, codes = compute()
    np.savez_compressed(OUT / "qwen3_encode.npz", z_first=z.reshape(-1)[:32].astype(np.float32), z_stats=stats(z),
                        z_shape=np.array(z.shape), codes=codes)


if __name__ == "__main__":
    main()
