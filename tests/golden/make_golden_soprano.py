"""Generates tests/golden/soprano_tiny.npz from the CPU oracle (run from the repo root: `python tests/golden/make_golden_soprano.py`): a tiny
Soprano (Qwen3 with q/k norm, untied head; a 2-layer Vocos decoder, input kernel 3), a prompt pair whose greedy rows (repetition penalty 1.5
over the last 30 generated tokens) repeat tokens, so that the per-occurrence, generated-only penalty gives other tokens than a per-unique
penalty or one that also counts the prompt.  Stored: the prompts, the stop token (row 1 stops on it, row 0 runs to max_tokens), the tokens,
the fp32-activation hidden states (1 + n per row) and the float64 waveforms (decoded from those states, cut)."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
from oracle import soprano as so  # noqa: E402

OUT = Path(__file__).resolve().parent

TINY = dict(hidden_size=256, num_hidden_layers=2, intermediate_size=512, num_attention_heads=2, num_key_value_heads=1, head_dim=128,
            vocab_size=512, decoder_num_layers=2, decoder_dim=128, decoder_intermediate_dim=256, hop_length=64, n_fft=256, upscale=4,
            input_kernel=3, dw_kernel=3, token_size=256)
SEED, STD, MAX_TOKENS = 8, 0.02, 24
IDS = [[369, 170, 236, 236, 236, 165, 330, 404, 328], [445, 28, 328, 328, 328, 201, 193, 24, 58]]


def main():
    cfg = so.SopranoConfig(**TINY)
    W = so.init_weights(cfg, SEED, std=STD)
    ids = np.asarray(IDS, dtype=np.int32)
    free, _ = so.generate(so.SopranoLM(cfg, W), ids, MAX_TOKENS, stop_token=-1)
    # row 1 stops on a token it first emits at step 10 and row 0 never emits; row 0 (whose 21st token tells the penalties apart) runs on
    stop = next(t for i, t in enumerate(free[1]) if i >= 10 and t not in free[1][:i] and t not in free[0])
    toks, hid = so.generate(so.SopranoLM(cfg, W), ids, MAX_TOKENS, stop_token=stop)
    for v in ("unique", "prompt"):
        assert so.generate(so.SopranoLM(cfg, W), ids, MAX_TOKENS, stop_token=stop, variant=v)[0] != toks, v
    assert len(toks[1]) < MAX_TOKENS == len(toks[0])
    waves = [so.decode(cfg, W, h[None])[0] for h in hid]
    n = np.asarray([len(t) for t in toks], dtype=np.int32)
    tok = np.full((2, MAX_TOKENS), -1, dtype=np.int32)
    hs = np.zeros((2, MAX_TOKENS + 1, cfg.hidden_size), dtype=np.float32)
    wl = np.asarray([len(w) for w in waves], dtype=np.int64)
    wv = np.zeros((2, int(wl.max())), dtype=np.float32)
    for b in range(2):
        tok[b, :n[b]] = toks[b]
        hs[b, :n[b] + 1] = hid[b]
        wv[b, :wl[b]] = waves[b]
    np.savez_compressed(OUT / "soprano_tiny.npz", ids=ids, stop=stop, max_tokens=MAX_TOKENS, tokens=tok, n_tokens=n, hidden=hs, wave=wv,
                        wave_len=wl, seed=SEED, std=STD)
    print("soprano_tiny.npz", n.tolist(), wl.tolist(), "stop", stop)


if __name__ == "__main__":
    main()
