"""Soprano's oracle on the CPU: interpolate1d against torch's align-corners linear interpolation, the language model and its hidden states
against transformers.Qwen3ForCausalLM, the sampler's traps (unnormalised top-p, per-occurrence penalty over generated tokens only, greedy
penalised), sanitize key for key against the library's, and the decoder rule of fromModelDirectory in the library's config parser."""
import ctypes as C
import json

import numpy as np
import pytest
import torch
from safetensors.numpy import save_file

from conftest import GOLDEN
from oracle import soprano as so


@pytest.mark.parametrize("n,T", [(7, 25), (2, 5), (1, 1), (5, 5), (1, 4), (3, 9)])
def test_interpolate1d_matches_torch(n, T):
    x = torch.randn(2, 6, n, dtype=torch.float64)
    ref = torch.nn.functional.interpolate(x, size=T, mode="linear", align_corners=True)
    assert torch.allclose(so.interpolate1d(x, T), ref, atol=1e-12)


def test_lm_and_hidden_states_match_transformers():
    transformers = pytest.importorskip("transformers")
    cfg = so.SopranoConfig(hidden_size=256, num_hidden_layers=2, intermediate_size=512, num_attention_heads=2, num_key_value_heads=1,
                           vocab_size=300)
    W = so.init_weights(cfg, 5, std=0.05)
    hf = transformers.Qwen3ForCausalLM(transformers.Qwen3Config(
        vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size, num_hidden_layers=cfg.num_hidden_layers,
        num_attention_heads=cfg.num_attention_heads, num_key_value_heads=cfg.num_key_value_heads, head_dim=cfg.head_dim,
        rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta, tie_word_embeddings=False, attention_bias=False)).double().eval()
    sd = {k: v.double() for k, v in W.items() if not k.startswith("decoder.")}
    hf.load_state_dict(sd, strict=False)
    ids = np.random.default_rng(0).integers(0, cfg.vocab_size, size=(2, 7))
    with torch.no_grad():
        out = hf(torch.as_tensor(ids), output_hidden_states=True)
    lm = so.SopranoLM(cfg, W, dtype=torch.float64)
    lg, hid = lm.forward_hidden(ids[:, :5])
    lg2, hid2 = lm.forward_hidden(ids[:, 5:])            # through the KV cache
    def rel(a, b):     # transformers builds its RoPE frequencies in float32: differences of a few 1e-7 remain
        return float((a - b).abs().max() / b.abs().max())
    assert rel(torch.cat([lg, lg2], 1), out.logits) < 1e-5
    assert rel(torch.cat([hid, hid2], 1), out.hidden_states[-1]) < 1e-5


def test_top_p_is_unnormalised():
    l = np.array([-3.0, -2.0, -1.0, -0.5, -4.0])
    a, b = so.top_p_keep(l, 0.8), so.top_p_keep(l + 2.0, 0.8)
    assert not np.array_equal(a, b)                      # a constant shift changes the kept set; normalised top-p would not
    assert so.top_p_keep(l, 0.9999).sum() >= a.sum()
    # no token passes when sum exp(l) <= 1 - top_p: the argmax alone
    probs = so.sample_probs(np.full(4, -5.0) + np.arange(4), 1.0, 0.2)
    assert probs[3] == 1.0 and probs.sum() == 1.0


def test_penalty_per_occurrence_generated_only():
    lg = np.array([2.0, -1.0, 0.5, 3.0], dtype=np.float32)
    out = so.repetition_penalty(lg, [0, 0, 0, 1], 1.5, 30)
    assert out[0] == np.float32(np.float32(np.float32(2.0) / np.float32(1.5)) / np.float32(1.5)) / np.float32(1.5)
    assert out[1] == np.float32(-1.5) and out[2] == lg[2] and out[3] == lg[3]
    assert np.array_equal(so.repetition_penalty(lg, [], 1.5, 30), lg)                 # nothing generated yet: no penalty
    assert so.repetition_penalty(lg, [3] + [2] * 30, 1.5, 30)[3] == lg[3]            # only the last 30 generated tokens


def _golden():
    from golden.make_golden_soprano import TINY
    g = np.load(GOLDEN / "soprano_tiny.npz")
    cfg = so.SopranoConfig(**TINY)
    return g, cfg, so.init_weights(cfg, int(g["seed"]), std=float(g["std"]))


def test_golden_matches_oracle():
    g, cfg, W = _golden()
    toks, hid = so.generate(so.SopranoLM(cfg, W), g["ids"], int(g["max_tokens"]), stop_token=int(g["stop"]))
    n = g["n_tokens"]
    assert [len(t) for t in toks] == n.tolist() and n[0] != n[1]
    for b in range(2):
        assert toks[b] == g["tokens"][b, :n[b]].tolist()
        assert np.array_equal(hid[b], g["hidden"][b, :n[b] + 1])
        w = so.decode(cfg, W, hid[b][None])[0]
        assert len(w) == g["wave_len"][b] and np.abs(w - g["wave"][b, :len(w)]).max() <= 1e-6 * np.abs(w).max()


def test_greedy_is_penalised_and_prompt_is_not():
    """The golden's prompts and model make greedy rows repeat tokens: the reference's penalty gives other tokens than a penalty applied
    once per unique token, or one whose window also holds the prompt, and other tokens than no penalty at all."""
    g, cfg, W = _golden()
    ids, mt = g["ids"], int(g["max_tokens"])
    pen = so.generate(so.SopranoLM(cfg, W), ids, mt, stop_token=-1)[0]
    free = so.generate(so.SopranoLM(cfg, W), ids, mt, stop_token=-1, rep_penalty=1.0)[0]
    unique = so.generate(so.SopranoLM(cfg, W), ids, mt, stop_token=-1, variant="unique")[0]
    prompt = so.generate(so.SopranoLM(cfg, W), ids, mt, stop_token=-1, variant="prompt")[0]
    assert pen != free and pen != unique and pen != prompt
    assert len(pen[0]) - len(set(pen[0])) >= 1                     # a token repeats inside the 30-token window
    assert pen[0][0] == free[0][0] != prompt[0][0]                  # the prompt is never penalised: the first token is the free one


def _published_keys():
    return ["language_model.embed_tokens.weight", "language_model.layers.0.self_attn.q_proj.weight", "language_model.norm.weight",
            "language_model.lm_head.weight", "model.language_model.layers.0.mlp.down_proj.weight", "layers.1.input_layernorm.weight",
            "decoder.decoder.embed.weight", "decoder.head.out.bias", "model.decoder.decoder.convnext.0.gamma", "lm_head.bias"]


@pytest.mark.parametrize("tied", [False, True])
def test_sanitize_key_for_key(b2a, tmp_path, tied):
    from mlx_audio_swift_b200 import _ffi
    cfg = so.SopranoConfig(tie_word_embeddings=tied)
    tensors = {k: np.full(4, i, np.float32) for i, k in enumerate(_published_keys())}
    save_file(tensors, str(tmp_path / "model.safetensors"))
    (tmp_path / "config.json").write_text(json.dumps(cfg.to_json()))
    w = C.c_void_p()
    _ffi.check(_ffi.lib().b2a_weights_load(str(tmp_path).encode(), C.byref(w)))
    try:
        _ffi.check(_ffi.lib().b2a_weights_sanitize_soprano_config(w, str(tmp_path / "config.json").encode()))
        got = {}
        for i in range(_ffi.lib().b2a_weights_count(w)):
            t = _ffi.Tensor()
            _ffi.check(_ffi.lib().b2a_weights_get(w, i, C.byref(t)))
            got[t.name.decode()] = float(np.ctypeslib.as_array(C.cast(t.data, C.POINTER(C.c_float)), shape=(4,))[0])
    finally:
        _ffi.lib().b2a_weights_free(w)
    ref = {k: float(v[0]) for k, v in so.sanitize(cfg, tensors).items()}
    assert got == ref
    assert ("lm_head.weight" in got) != tied and "model.layers.1.input_layernorm.weight" in got and "decoder.decoder.convnext.0.gamma" in got


@pytest.mark.parametrize("repo,dim,inter,k", [("mlx-community/Soprano-1.1-80M-bf16", 768, 2304, 1), ("ekwek/soprano-1.1-80M", 768, 2304, 1),
                                              ("ekwek/Soprano-80M", 512, 1536, 3), (None, 512, 1536, 3)])
def test_decoder_generation_rule(b2a, tmp_path, repo, dim, inter, k):
    from mlx_audio_swift_b200 import _ffi
    d = tmp_path / "checkpoint"
    d.mkdir()
    (d / "config.json").write_text(json.dumps({kk: v for kk, v in so.SopranoConfig().to_json().items()
                                               if not kk.startswith("decoder") and kk != "input_kernel"}))
    c = _ffi.SopranoConfig()
    _ffi.check(_ffi.lib().b2a_soprano_config_from_json(str(d / "config.json").encode(), repo.encode() if repo else None, 8, 512, C.byref(c),
                                                       None, None))
    assert (c.decoder_dim, c.decoder_intermediate_dim, c.input_kernel) == (dim, inter, k)
    assert (c.rms_norm_eps, c.rope_theta, c.sample_rate, c.stop_token_id, c.token_size, c.n_fft, c.hop_length) == (
        pytest.approx(1e-6), 1e4, 32000, 3, 2048, 2048, 512)
    ref = so.apply_repo_rule(so.SopranoConfig(), repo or "checkpoint")
    assert (ref.decoder_dim, ref.decoder_intermediate_dim, ref.input_kernel) == (dim, inter, k)
