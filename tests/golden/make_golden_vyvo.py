"""Generates tests/golden/vyvo_tiny.npz from the CPU oracle (run from the repo root: `python tests/golden/make_golden_vyvo.py`): a tiny
VyvoTTS stack (Qwen3 with q/k norm, untied head, linear RoPE scaling 2), a framed prompt pair, the fp32-activation logits of the last prompt
position and 24 greedy tokens per row (repetition penalty 1.3 over 20 tokens)."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
from oracle import vyvo  # noqa: E402

OUT = Path(__file__).resolve().parent

TINY = dict(hidden_size=256, num_hidden_layers=2, intermediate_size=512, num_attention_heads=2, num_key_value_heads=1, head_dim=128,
            vocab_size=2048, rope_scaling={"type": "linear", "factor": 2.0})
SEED, STD = 1234, 0.08


def main():
    cfg = vyvo.Qwen3Config(**TINY)
    W = vyvo.init_weights(cfg, SEED, std=STD)
    ids, _ = vyvo.prepare_input_ids([[11, 22, 33, 44, 55, 66, 77], [101, 102, 103]])
    ids = np.where(ids >= cfg.vocab_size, ids % 997, ids).astype(np.int32)      # the tiny vocabulary: fold the special ids into it
    logits = vyvo.VyvoOracle(cfg, W).forward(ids).numpy()
    greedy = vyvo.generate_tokens(vyvo.VyvoOracle(cfg, W), ids, 24, rep_penalty=1.3, rep_context=20)
    np.savez_compressed(OUT / "vyvo_tiny.npz", ids=ids, logits_last=logits[:, -1].astype(np.float32), greedy=np.asarray(greedy, dtype=np.int32),
                        seed=SEED, std=STD)
    print("vyvo_tiny.npz", ids.shape, logits.shape, np.asarray(greedy).shape)


if __name__ == "__main__":
    main()
