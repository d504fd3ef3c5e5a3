"""VyvoTTS (Qwen3.swift) on the CPU: the oracle's Qwen3 forward pinned against transformers.Qwen3ForCausalLM in float64, the prompt
framing, parse rule, decode chunking and config parsing of the oracle and of the library's host entry points, and the committed golden."""
import json

import numpy as np
import pytest
import torch

from conftest import GOLDEN, rel_err
from oracle import vyvo

SMALL = dict(hidden_size=128, num_hidden_layers=2, intermediate_size=256, num_attention_heads=4, head_dim=128, vocab_size=512)


def _hf_logits(cfg: vyvo.Qwen3Config, W, ids):
    from transformers import Qwen3Config, Qwen3ForCausalLM
    kw = dict(hidden_size=cfg.hidden_size, num_hidden_layers=cfg.num_hidden_layers, intermediate_size=cfg.intermediate_size,
              num_attention_heads=cfg.num_attention_heads, num_key_value_heads=cfg.num_key_value_heads, head_dim=cfg.head_dim,
              vocab_size=cfg.vocab_size, rms_norm_eps=cfg.rms_norm_eps, tie_word_embeddings=cfg.tie_word_embeddings,
              max_position_embeddings=4096, attention_bias=False)
    rope = {"rope_type": "linear", "factor": cfg.rope_linear_factor} if cfg.rope_linear_factor != 1.0 else {"rope_type": "default"}
    hc = Qwen3Config(**kw, rope_parameters={**rope, "rope_theta": cfg.rope_theta})
    hc._attn_implementation = "eager"
    m = Qwen3ForCausalLM(hc).to(torch.float64).eval()
    sd = {k: v.to(torch.float64) for k, v in W.items()}
    if cfg.tie_word_embeddings:
        sd["lm_head.weight"] = sd["model.embed_tokens.weight"]
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all("rotary" in k for k in missing), (missing, unexpected)
    with torch.no_grad():
        return m(torch.as_tensor(ids, dtype=torch.long)).logits


@pytest.mark.parametrize("tied", [False, True])
@pytest.mark.parametrize("rope_scaling", [None, {"type": "linear", "factor": 4.0}])
@pytest.mark.parametrize("nkv", [2, 1])
def test_forward_matches_transformers_qwen3(tied, rope_scaling, nkv):
    cfg = vyvo.Qwen3Config(**SMALL, num_key_value_heads=nkv, tie_word_embeddings=tied, rope_scaling=rope_scaling)
    W = vyvo.init_weights(cfg, 7, std=0.05)
    ids = np.random.default_rng(1).integers(0, cfg.vocab_size, size=(2, 37))
    ours = vyvo.VyvoOracle(cfg, W, dtype=torch.float64).forward(ids)
    assert rel_err(ours.numpy(), _hf_logits(cfg, W, ids).numpy()) < 1e-6       # transformers builds its RoPE inv_freq in float32
    # incremental (KV cache) == full
    o = vyvo.VyvoOracle(cfg, W, dtype=torch.float64)
    a, b = o.forward(ids[:, :20]), o.forward(ids[:, 20:])
    assert rel_err(torch.cat([a, b], 1).numpy(), ours.numpy()) < 1e-12


def test_rope_scaling_other_than_linear_is_ignored():
    assert vyvo.Qwen3Config(rope_scaling={"type": "dynamic", "factor": 8.0}).rope_linear_factor == 1.0
    assert vyvo.Qwen3Config(rope_scaling={"rope_type": "linear", "factor": 8.0}).rope_linear_factor == 1.0   # the key is "type"
    assert vyvo.Qwen3Config(rope_scaling={"type": "linear", "factor": 8.0}).rope_linear_factor == 8.0


def _swift_rows(prompts, text=None, codes=None):
    """Qwen3.swift:417-464 written out literally."""
    mx = max(len(p) for p in prompts)
    rows = []
    for p in prompts:
        r = [151676] * (mx - len(p))
        if text is not None and codes is not None:
            r += [151672, *text, 151645, 151673, 151674, 151670, *[c + 151679 for c in codes], 151671, 151675]
        rows.append(r + [151672, *p, 151645, 151673])
    return np.asarray(rows, dtype=np.int32)


def test_prompt_framing(b2a):
    rng = np.random.default_rng(5)
    codes = rng.integers(0, 7 * 4096, size=21).tolist()
    for prompts in ([[5, 6, 7], [1], [2, 3]], [[42]]):
        plain = _swift_rows(prompts)
        assert np.array_equal(vyvo.prepare_input_ids(prompts)[0], plain)
        ids, mask = b2a.Qwen3Model.prepare_input_ids(prompts)
        assert np.array_equal(ids, plain) and np.array_equal(mask, plain != 151676)
        ref = _swift_rows(prompts, [9, 8, 7], codes)
        assert np.array_equal(vyvo.prepare_input_ids(prompts, [9, 8, 7], codes)[0], ref)
        assert np.array_equal(b2a.Qwen3Model.prepare_input_ids(prompts, codes, [9, 8, 7])[0], ref)
    # an empty transcript; a missing piece frames the prompts alone; bad codes are refused
    assert np.array_equal(b2a.Qwen3Model.prepare_input_ids([[1]], codes, [])[0], _swift_rows([[1]], [], codes))
    assert np.array_equal(b2a.Qwen3Model.prepare_input_ids([[1]], codes, None)[0], _swift_rows([[1]]))
    with pytest.raises(b2a.AudioGenerationError):
        b2a.Qwen3Model.prepare_input_ids([[1]], codes[:5], [1])
    with pytest.raises(b2a.AudioGenerationError):
        b2a.Qwen3Model.prepare_input_ids([[1]], [7 * 4096] * 7, [1])


A = 151679          # audio offset
SOS, EOS, SOAI = 151670, 151671, 151674
PARSE_CASES = {
    # the last start-of-speech wins; stop tokens dropped; trimmed to 7
    "last_sos": ([1, SOS, A + 1, A + 2, SOS, *[A + i for i in range(7)], EOS, A + 9, A + 10], list(range(7))),
    # no start-of-speech: from the first audio token after the LAST start-of-AI
    "soai_fallback": ([SOAI, A + 5, 3, SOAI, 7, 8, *[A + 100 + i for i in range(8)]], [100 + i for i in range(7)]),
    # start-of-AI without an audio token after it, and no marker at all: the whole row
    "soai_no_audio": ([*[A + i for i in range(7)], SOAI, 5], list(range(7))),
    "neither": ([*[A + i for i in range(14)], EOS], list(range(14))),
    "short": ([SOS, A, A + 1, EOS], []),
}


@pytest.mark.parametrize("case", sorted(PARSE_CASES))
def test_parse_rule(b2a, case):
    row, want = PARSE_CASES[case]
    assert vyvo.parse_output_row(row) == want
    assert b2a.Qwen3Model.parse_output(np.asarray([row], dtype=np.int32)) == [want]


def test_parse_rows_are_independent(b2a):
    rows = np.asarray([[SOS] + [A + i for i in range(7)], [SOAI] + [A + 20 + i for i in range(7)]], dtype=np.int32)
    assert b2a.Qwen3Model.parse_output(rows) == [vyvo.parse_output_row(r) for r in rows] == [list(range(7)), list(range(20, 27))]


@pytest.mark.parametrize("frames,want", [(1, [(0, 1)]), (49, [(0, 49)]), (50, [(0, 50)]), (51, [(0, 50), (50, 1)]),
                                         (120, [(0, 50), (50, 50), (100, 20)])])
def test_decode_chunks(frames, want):
    assert vyvo.decode_chunks(7 * frames) == want


def test_config_parsing_with_defaults(b2a, tmp_path):
    base = dict(hidden_size=1024, num_hidden_layers=28, intermediate_size=3072, num_attention_heads=16, num_key_value_heads=8,
                head_dim=128, vocab_size=180352, rms_norm_eps=1e-6)
    p = tmp_path / "config.json"
    p.write_text(json.dumps(base))
    c, gs, bits = b2a.Qwen3Model.config_from_json(p, 4, 512)
    o = vyvo.load_config(p)
    assert (c.rope_theta, c.rope_linear_factor, c.tie_word_embeddings, c.max_position_embeddings, c.sample_rate, c.eos_token_id) == \
           (1e6, 1.0, 0, 32768, 24000, 151645) == (o.rope_theta, o.rope_linear_factor, int(o.tie_word_embeddings),
                                                   o.max_position_embeddings, o.sample_rate, o.eos_token_id)
    assert (c.hidden_size, c.vocab_size, c.head_dim, c.max_batch, c.max_context, gs, bits) == (1024, 180352, 128, 4, 512, 0, 0)
    p.write_text(json.dumps({**base, "rope_theta": 10000.0, "rope_scaling": {"type": "linear", "factor": 2.0}, "tie_word_embeddings": True,
                             "quantization": {"group_size": 32, "bits": 8}}))
    c, gs, bits = b2a.Qwen3Model.config_from_json(p)
    assert (c.rope_theta, c.rope_linear_factor, c.tie_word_embeddings, gs, bits) == (10000.0, 2.0, 1, 32, 8)
    p.write_text(json.dumps({**base, "rope_scaling": {"type": "yarn", "factor": 4.0}}))
    assert b2a.Qwen3Model.config_from_json(p)[0].rope_linear_factor == 1.0 == vyvo.load_config(p).rope_linear_factor
    for k in ("head_dim", "num_key_value_heads"):
        p.write_text(json.dumps({kk: v for kk, v in base.items() if kk != k}))
        with pytest.raises(b2a.AudioGenerationError, match=k):
            b2a.Qwen3Model.config_from_json(p)
        with pytest.raises(KeyError):
            vyvo.load_config(p)


def test_golden_is_the_oracle():
    g = np.load(GOLDEN / "vyvo_tiny.npz")
    from golden.make_golden_vyvo import TINY
    cfg = vyvo.Qwen3Config(**TINY)
    W = vyvo.init_weights(cfg, int(g["seed"]), std=float(g["std"]))
    lg = vyvo.VyvoOracle(cfg, W).forward(g["ids"]).numpy()[:, -1]
    assert rel_err(lg, g["logits_last"]) < 1e-6
    assert vyvo.generate_tokens(vyvo.VyvoOracle(cfg, W), g["ids"], 24, rep_penalty=1.3, rep_context=20) == g["greedy"].tolist()
