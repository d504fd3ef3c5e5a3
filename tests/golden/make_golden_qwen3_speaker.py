"""Generates tests/golden/qwen3_speaker.npz from the float64 Qwen3-TTS speaker-encoder reference (run from the repo root:
`python tests/golden/make_golden_qwen3_speaker.py`).  Kept apart from make_golden.py so that the other fixtures are never rewritten
by it.  The small geometry, the seeds of the weights and of the clip, and the float64 embedding."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import qwen3_speaker_encoder_reference as ser  # noqa: E402
from mlx_audio_swift_b200.qwen3_tts import Qwen3SpeakerEncoderConfig, random_init_speaker_encoder_weights  # noqa: E402

OUT = Path(__file__).resolve().parent
N_SAMPLES, BATCH, CLIP_SEED, WEIGHT_SEED = 12000, 2, 9, 31
SMALL = dict(enc_channels=[96, 96, 96, 192], enc_kernel_sizes=[5, 3, 3, 3], enc_dilations=[1, 2, 3, 1], enc_attention_channels=80,
             enc_res2net_scale=4, enc_se_channels=72, enc_dim=48)


def weights():
    cfg = Qwen3SpeakerEncoderConfig(**SMALL)
    return cfg, random_init_speaker_encoder_weights(cfg, seed=WEIGHT_SEED)


def clip():
    return ser.synth_clip(BATCH, N_SAMPLES, CLIP_SEED)


def main():
    cfg, W = weights()
    x = clip()
    np.savez_compressed(OUT / "qwen3_speaker.npz", embedding=ser.embed(cfg, W, x), clip=np.array([BATCH, N_SAMPLES, CLIP_SEED]),
                        weight_seed=np.array(WEIGHT_SEED), **{k: np.array(v) for k, v in SMALL.items()})


if __name__ == "__main__":
    main()
