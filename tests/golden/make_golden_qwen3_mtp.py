"""Generates tests/golden/qwen3_talker_mtp.npz from the float64 oracle (run from the repo root:
`python tests/golden/make_golden_qwen3_mtp.py`): a Qwen3-TTS talker whose code predictor is narrower than the talker (talker 384,
predictor 256, head_dim 128, 4 code groups), so every predictor input goes through code_predictor.small_to_mtp_projection, as in the
1.7B checkpoints.  Weights are bf16-valued (what a checkpoint holds).  Stored: stats and top-8 of the first talker logits and the
first five greedy frames, in the style of qwen3_talker_hd128.npz."""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
from oracle import qwen3_tts as ot  # noqa: E402

OUT = Path(__file__).resolve().parent
SEED = 17
CHAT = [151, 12, 13, 40, 41, 42, 43, 44, 45, 46, 47, 152, 14, 151, 12, 13]
TTS = dict(tts_bos=160, tts_eos=161, tts_pad=162)


def config(talker_hidden=384, cp_hidden=256):
    """Talker and predictor widths differ; heads are sized so q heads x 128 = hidden (GQA 3 : 1 at 384, 2 : 1 at 256)."""
    def heads(h):
        return h // 128, 1
    cq, ckv = heads(cp_hidden)
    tq, tkv = heads(talker_hidden)
    cp = ot.CodePredictorConfig(vocab_size=2048, hidden_size=cp_hidden, intermediate_size=2 * cp_hidden, num_hidden_layers=2,
                                num_attention_heads=cq, num_key_value_heads=ckv, head_dim=128, num_code_groups=4)
    return ot.TalkerConfig(vocab_size=3072, hidden_size=talker_hidden, intermediate_size=2 * talker_hidden, num_hidden_layers=3,
                           num_attention_heads=tq, num_key_value_heads=tkv, head_dim=128, num_code_groups=4, text_hidden_size=128,
                           text_vocab_size=200, codec_eos_token_id=2150, code_predictor=cp)


def weights(cfg, seed=SEED, std=0.05):
    return {k: v.to(torch.bfloat16).to(torch.float64) for k, v in ot.init_weights(cfg, seed, std=std).items()}


def make():
    cfg = config()
    W = weights(cfg)
    inp, trail, pad = ot.prepare_generation_inputs(cfg, W, CHAT, **TTS, language_id=2160)
    logits, _ = ot.Talker(cfg, W)(inp, None)
    codes = ot.generate_codes(cfg, W, inp, trail, pad, max_tokens=5, temperature=0.0, repetition_penalty=1.05, stop_on_eos=False)
    x = logits[0, -1].numpy()
    return dict(first_logits_stats=np.array([x.mean(), np.abs(x).mean(), x.min(), x.max()]),
                first_logits_top=np.argsort(-x)[:8].astype(np.int32), codes=codes.numpy().astype(np.int32))


if __name__ == "__main__":
    np.savez_compressed(OUT / "qwen3_talker_mtp.npz", **make())
