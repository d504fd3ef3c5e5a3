"""Soprano (SopranoModel, Soprano.swift) on the H100 through the C ABI: hidden states captured in the decode graph against the fp32-activation
oracle (1 + n_gen per row, none for the stop token), greedy tokens with the 1.5 penalty bit-exact, the Vocos decode of hidden states (the
fused upsample, the cut, n = 1), batched against serial for rows that stop at different lengths, Soprano's unnormalised top-p at T > 0,
seeding, directory loading for both decoder generations and an 8-bit checkpoint, and the error cases."""
import json

import numpy as np
import pytest
import torch
from safetensors.numpy import save_file

from conftest import GOLDEN, rel_err
from golden.make_golden_soprano import TINY as GOLDEN_TINY
from oracle import soprano as so
from test_loading import mlx_affine_quantize

pytestmark = pytest.mark.gpu

TINY = dict(hidden_size=256, num_hidden_layers=2, intermediate_size=512, num_attention_heads=2, num_key_value_heads=1, head_dim=128,
            vocab_size=512, decoder_num_layers=2, decoder_dim=128, decoder_intermediate_dim=256, hop_length=64, n_fft=256, upscale=4,
            input_kernel=3, dw_kernel=3, token_size=256)


def _cfg(**kw):
    return so.SopranoConfig(**{**TINY, **kw})


def _peak_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _greedy(b2a, cfg, W, ids, max_tokens, stop):
    m = b2a.SopranoModel(cfg.to_json(), W, max_batch=8, max_context=128, stop_token_id=stop)
    P = b2a.GenerateParameters(max_tokens=max_tokens, temperature=0.0, top_p=0.95, repetition_penalty=1.5, repetition_context_size=30)
    toks, waves, _ = m.generate_batch(ids, P)
    return m, toks, waves


def _setup(seed=7):
    cfg = _cfg()
    W = so.init_weights(cfg, 1234, std=0.08)
    ids = np.random.default_rng(seed).integers(4, 512, size=(2, 9)).astype(np.int32)
    # a stop token the first row emits at its 5th step (and not before): the rows stop at different lengths
    free, _ = so.generate(so.SopranoLM(cfg, W), ids, 12, stop_token=-1)
    stop = next(t for i, t in enumerate(free[0]) if i >= 4 and t not in free[0][:i])
    return cfg, W, ids, stop


def test_hidden_states_and_greedy_tokens_vs_oracle(b2a):
    cfg, W, ids, stop = _setup()
    ref_tok, ref_hid = so.generate(so.SopranoLM(cfg, W), ids, 12, stop_token=stop)
    m, toks, _ = _greedy(b2a, cfg, W, ids, 12, stop)
    assert toks == ref_tok                                   # bit-exact greedy tokens with the per-occurrence penalty
    assert len(toks[0]) != len(toks[1]) and stop not in toks[0]
    hid = m.hidden_states(2)
    for b in range(2):
        assert hid[b].shape == (1 + len(ref_tok[b]), cfg.hidden_size)      # 1 + n_gen states, none for the stop token
        assert rel_err(hid[b], ref_hid[b]) < 1e-5, rel_err(hid[b], ref_hid[b])


def test_step_prefill_captures_the_same_states(b2a, monkeypatch):
    cfg, W, ids, stop = _setup()
    m, toks, _ = _greedy(b2a, cfg, W, ids, 12, stop)
    monkeypatch.setenv("B2A_PREFILL", "step")
    ms, toks_s, _ = _greedy(b2a, cfg, W, ids, 12, stop)
    monkeypatch.delenv("B2A_PREFILL")
    assert toks_s == toks
    for a, b in zip(ms.hidden_states(2), m.hidden_states(2)):
        assert a.shape == b.shape and rel_err(a, b) < 1e-5, rel_err(a, b)


def test_max_tokens_row_feeds_its_last_token(b2a):
    cfg, W, ids, _ = _setup()
    ref_tok, ref_hid = so.generate(so.SopranoLM(cfg, W), ids, 6, stop_token=-1)
    m, toks, waves = _greedy(b2a, cfg, W, ids, 6, -1)
    assert toks == ref_tok
    for b, h in enumerate(m.hidden_states(2)):
        assert h.shape[0] == 7 and rel_err(h, ref_hid[b]) < 1e-5, rel_err(h, ref_hid[b])
        assert len(waves[b]) == 6 * cfg.token_size


def test_decode_hidden_vs_oracle(b2a):
    cfg = _cfg()
    W = so.init_weights(cfg, 99, std=0.08)
    m = b2a.SopranoModel(cfg.to_json(), W, max_batch=8, max_context=64)
    hid = np.random.default_rng(3).standard_normal((3, 9, cfg.hidden_size)).astype(np.float32)
    got, ref = m.decode(hid), so.decode(cfg, W, hid)
    for g, r in zip(got, ref):
        assert len(g) == 8 * cfg.token_size and _peak_err(g, r) < 1e-3, _peak_err(g, r)
    one, ref1 = m.decode(hid[:1, :1]), so.decode(cfg, W, hid[:1, :1])
    assert len(one[0]) == cfg.n_fft and _peak_err(one[0], ref1[0]) < 1e-3      # n = 1: the untrimmed one-frame overlap-add


@pytest.mark.parametrize("input_kernel", [1, 3])
def test_end_to_end_waveform_and_batched_equals_serial(b2a, input_kernel):
    cfg, W0, ids, stop = _setup()
    cfg = _cfg(input_kernel=input_kernel)
    W = so.init_weights(cfg, 1234, std=0.08)
    ref_tok, ref_hid = so.generate(so.SopranoLM(cfg, W), ids, 12, stop_token=stop)
    m, toks, waves = _greedy(b2a, cfg, W, ids, 12, stop)
    assert toks == ref_tok
    for b in range(2):
        ref = so.decode(cfg, W, ref_hid[b][None])[0]
        assert _peak_err(waves[b], ref) < 1e-3, _peak_err(waves[b], ref)
        _, t1, w1 = _greedy(b2a, cfg, W, ids[b:b + 1], 12, stop)
        assert t1[0] == toks[b] and _peak_err(w1[0], waves[b]) < 1e-5


def _first_step_model(b2a, seed, total_mass):
    """A model whose first-step logits are a chosen vector: lm_head rows = l*_v hn / |hn|^2 for the prompt's last hidden state hn, with
    l* shifted so that sum exp(l*) = total_mass."""
    cfg = _cfg()
    W = so.init_weights(cfg, seed, std=0.08)
    ids = np.random.default_rng(seed).integers(4, 512, size=(1, 9)).astype(np.int32)
    _, hid = so.SopranoLM(cfg, W).forward_hidden(ids)
    hn = hid[0, -1].double()
    rng = np.random.default_rng(seed + 1)
    target = 1.5 * rng.standard_normal(cfg.vocab_size)
    target += np.log(total_mass) - np.log(np.exp(target).sum())
    W["lm_head.weight"] = (torch.as_tensor(target)[:, None] * hn[None, :] / (hn @ hn)).to(torch.bfloat16)
    m = b2a.SopranoModel(cfg.to_json(), W, max_batch=8, max_context=64, stop_token_id=-1)
    return m, np.repeat(ids, 8, axis=0)


def test_sampling_unnormalised_top_p(b2a):
    m, ids = _first_step_model(b2a, 5, 0.6)
    lg = m(ids[:1])[0, -1].astype(np.float64)
    e = np.exp(lg)
    larger = np.array([e[lg > x].sum() for x in lg])
    below = e.sum() - larger                      # ascending cumulative mass through each token
    # a threshold 1 - top_p in the widest gap between consecutive cumulative masses of the top 12 tokens: membership away from it
    top = np.sort(below)[::-1][:13]
    k = int(np.argmax(top[:-1] - top[1:]))
    thr = 0.5 * (top[k] + top[k + 1])
    keep = below > thr
    assert 1 <= keep.sum() <= 12 and not keep.all()
    for T in (1.0, 0.7):
        P = so_params(b2a, 1, T, 1.0 - thr)
        draws = []
        for seed in range(150):
            P.seed = seed
            toks, _, _ = m.generate_batch(ids, P, decode_audio=False)
            draws += [t[0] for t in toks]
        draws = np.asarray(draws)
        assert keep[draws].all()                                # never outside the unnormalised nucleus
        p = np.where(keep, np.exp((lg - lg.max()) / T), 0.0)
        p /= p.sum()
        freq = np.bincount(draws, minlength=len(lg)) / len(draws)
        assert 0.5 * np.abs(freq - p).sum() < 0.06, 0.5 * np.abs(freq - p).sum()


def test_no_token_passes_returns_argmax(b2a):
    m, ids = _first_step_model(b2a, 11, 0.3)
    lg = m(ids[:1])[0, -1]
    P = so_params(b2a, 1, 1.0, 0.5)           # 1 - top_p = 0.5 > sum exp(l) = 0.3
    for seed in range(5):
        P.seed = seed
        toks, _, _ = m.generate_batch(ids, P, decode_audio=False)
        assert all(t[0] == int(np.argmax(lg)) for t in toks)


def so_params(b2a, max_tokens, T, top_p):
    return b2a.GenerateParameters(max_tokens=max_tokens, temperature=T, top_p=top_p, repetition_penalty=1.5, repetition_context_size=30)


def test_same_seed_same_output(b2a):
    cfg, W, ids, stop = _setup()
    m = b2a.SopranoModel(cfg.to_json(), W, max_batch=8, max_context=128, stop_token_id=stop)
    P = b2a.GenerateParameters(max_tokens=10, temperature=0.7, top_p=0.95, repetition_penalty=1.5, repetition_context_size=30, seed=42)
    t1, w1, _ = m.generate_batch(ids, P)
    t2, w2, _ = m.generate_batch(ids, P)
    assert t1 == t2 and all(np.array_equal(a, b) for a, b in zip(w1, w2))


def _published(cfg, W, quant_bits=0):
    """W in the published key layout (language_model.*, decoder.*), optionally with the LM's Linears MLX-quantised."""
    out = {}
    for k, v in W.items():
        a = v.float().numpy() if isinstance(v, torch.Tensor) else np.asarray(v, np.float32)
        name = k if k.startswith("decoder.") else "language_model." + (k[len("model."):] if k.startswith("model.") else k)
        if quant_bits and a.ndim == 2 and ".layers." in k and k.endswith("_proj.weight"):
            words, scales, biases, _ = mlx_affine_quantize(a, 64, quant_bits)
            base = name[:-len(".weight")]
            out[name], out[base + ".scales"], out[base + ".biases"] = words.view(np.int32), scales, biases
        else:
            out[name] = a
    return out


@pytest.mark.parametrize("repo,bits", [("Soprano-1.1-80M", 0), ("Soprano-80M", 0), ("soprano-1.1-80m-8bit", 8)])
def test_directory_loading(b2a, tmp_path, repo, bits):
    cfg = _cfg(decoder_dim=128, decoder_intermediate_dim=256, input_kernel=1)
    eff = so.apply_repo_rule(_cfg(decoder_dim=128, decoder_intermediate_dim=256, input_kernel=1), repo)
    W = so.init_weights(eff, 21, std=0.08)
    d = tmp_path / repo
    d.mkdir()
    conf = cfg.to_json()
    if bits:
        conf["quantization"] = {"group_size": 64, "bits": bits}
    (d / "config.json").write_text(json.dumps(conf))
    (d / "tokenizer_config.json").write_text(json.dumps({"eos_token": "[STOP]"}))
    (d / "tokenizer.json").write_text(json.dumps({"added_tokens": [{"id": 7, "content": "[STOP]"}]}))
    save_file(_published(cfg, W, bits), str(d / "model.safetensors"))
    m = b2a.SopranoModel.from_model_directory(d, max_batch=2, max_context=64)
    assert m.sample_rate == 32000
    hid = np.random.default_rng(1).standard_normal((1, 5, cfg.hidden_size)).astype(np.float32)
    assert _peak_err(m.decode(hid)[0], so.decode(eff, W, hid)[0]) < 1e-3
    ids = np.random.default_rng(2).integers(8, 512, size=(1, 6)).astype(np.int32)
    if bits == 0:
        lg, ref = m(ids), so.SopranoLM(eff, W).forward_hidden(ids)[0].numpy()
        assert rel_err(lg, ref) < 1e-4
    toks, _, _ = m.generate_batch(ids, so_params(b2a, 8, 0.0, 0.95), decode_audio=False)
    assert 7 not in toks[0]                      # the tokenizer's EOS stops generation and is not kept


def test_errors(b2a):
    cfg = _cfg()
    W = so.init_weights(cfg, 3, std=0.08)
    with pytest.raises(b2a.AudioGenerationError) as e:
        b2a.SopranoModel({**cfg.to_json(), "head_dim": 64}, W, max_batch=2, max_context=64)
    assert e.value.case == "invalidInput"
    m = b2a.SopranoModel(cfg.to_json(), W, max_batch=2, max_context=32)
    ids = np.zeros((1, 20), dtype=np.int32)
    with pytest.raises(b2a.AudioGenerationError) as e:
        m.generate_batch(ids, so_params(b2a, 12, 0.0, 0.95))        # 20 + 12 + 1 > 32
    assert e.value.case == "invalidInput"
    m.generate_batch(ids, so_params(b2a, 11, 0.0, 0.95), decode_audio=False)
    import ctypes as C
    from mlx_audio_swift_b200 import _ffi
    assert _ffi.lib().b2a_soprano_decode_hidden(None, None, 1, 1, None, 0, None) != 0
    assert _ffi.lib().b2a_soprano_create(0, None, None, 0, C.byref(C.c_void_p())) != 0
    assert _ffi.lib().b2a_soprano_create_from_directory(None, None, 0, 1, 64, None) != 0


def test_golden(b2a):
    """The golden's rows repeat tokens, so its greedy tokens pin the per-occurrence, generated-only penalty (tests/test_oracle_soprano.py
    shows that a per-unique penalty or one that counts the prompt gives other tokens); row 1 stops early, row 0 runs to max_tokens."""
    g = np.load(GOLDEN / "soprano_tiny.npz")
    cfg = so.SopranoConfig(**GOLDEN_TINY)
    W = so.init_weights(cfg, int(g["seed"]), std=float(g["std"]))
    m, toks, waves = _greedy(b2a, cfg, W, g["ids"], int(g["max_tokens"]), int(g["stop"]))
    n = g["n_tokens"]
    assert toks == [g["tokens"][b, :n[b]].tolist() for b in range(2)]
    for b, h in enumerate(m.hidden_states(2)):
        assert h.shape[0] == n[b] + 1 and rel_err(h, g["hidden"][b, :n[b] + 1]) < 1e-5, rel_err(h, g["hidden"][b, :n[b] + 1])
        assert len(waves[b]) == g["wave_len"][b] and _peak_err(waves[b], g["wave"][b, :g["wave_len"][b]]) < 1e-3
