"""VyvoTTS (Qwen3Model, Qwen3.swift) on the H100 through the C ABI: logits against the fp32-activation oracle and the golden at two GQA ratios
with tied and untied heads, the batched prompt pass with q/k norm (SIMT attention up to 128 positions, wgmma beyond) against the per-position
replay (B2A_PREFILL=step) and the oracle, greedy tokens bit-exact, the stop token 151671 on the full-size vocabulary, the 50-frame chunked
SNAC decode, voice cloning from a device-encoded clip, loading a checkpoint directory and the error cases."""
import json

import numpy as np
import pytest
import torch
from safetensors.numpy import save_file
from safetensors.torch import save_file as save_file_torch

import snac_encoder_reference as ser
from conftest import GOLDEN, rel_err
from golden.make_golden_vyvo import TINY as GOLDEN_TINY
from oracle import llama as ol
from oracle import snac as osnac
from oracle import vyvo
from test_loading import mlx_affine_quantize

pytestmark = pytest.mark.gpu
TOL = 1e-3
TINY = dict(hidden_size=256, num_hidden_layers=2, intermediate_size=512, head_dim=128, vocab_size=2048)


def config(cfg: vyvo.Qwen3Config) -> dict:
    return cfg.to_json()


def _generate(b2a, model, ids, P):
    n0 = b2a.launch_count()
    toks, _, info = model.generate_batch(ids, P, decode_audio=False)
    return toks, info, b2a.launch_count() - n0


def _models(b2a, monkeypatch, cfg, W, max_batch, max_context, **kw):
    m_b = b2a.Qwen3Model(config(cfg), W, max_batch=max_batch, max_context=max_context, **kw)
    monkeypatch.setenv("B2A_PREFILL", "step")
    m_s = b2a.Qwen3Model(config(cfg), W, max_batch=max_batch, max_context=max_context, **kw)
    monkeypatch.delenv("B2A_PREFILL")
    return m_b, m_s


@pytest.mark.parametrize("nq,tied", [(2, False), (2, True), (4, False), (4, True)])
def test_logits_vs_oracle(b2a, nq, tied):
    cfg = vyvo.Qwen3Config(**TINY, num_attention_heads=nq, num_key_value_heads=1, tie_word_embeddings=tied,
                           rope_scaling={"type": "linear", "factor": 2.0})
    W = vyvo.init_weights(cfg, 1234, std=0.08)
    m = b2a.Qwen3Model(config(cfg), W, max_batch=8, max_context=256)
    ids = np.random.default_rng(nq).integers(0, 2048, size=(2, 12)).astype(np.int32)
    lg, ref = m(ids), vyvo.VyvoOracle(cfg, W).forward(ids).numpy()
    assert rel_err(lg, ref) < 1e-4, rel_err(lg, ref)
    assert np.array_equal(lg.argmax(-1), ref.argmax(-1))


def test_golden_logits_and_greedy_tokens(b2a):
    g = np.load(GOLDEN / "vyvo_tiny.npz")
    cfg = vyvo.Qwen3Config(**GOLDEN_TINY)
    W = vyvo.init_weights(cfg, int(g["seed"]), std=float(g["std"]))
    m = b2a.Qwen3Model(config(cfg), W, max_batch=2, max_context=128)
    ids = g["ids"].astype(np.int32)
    assert rel_err(m(ids)[:, -1], g["logits_last"]) < TOL
    P = b2a.GenerateParameters(max_tokens=24, temperature=0.0, top_p=1.0, repetition_penalty=1.3, repetition_context_size=20)
    toks, _, info = m.generate_batch(ids, P, decode_audio=False)
    assert toks == g["greedy"].tolist() and info.generation_token_count == 48


# (B, L, nq, max_tokens, max_context): L <= 128 takes the SIMT prompt attention, L = 300 the wgmma one
@pytest.mark.parametrize("B,L,nq,max_context", [(1, 60, 2, 96), (8, 100, 4, 160), (1, 300, 2, 336), (8, 300, 4, 336)])
def test_batched_prefill_matches_stepwise_and_oracle(b2a, monkeypatch, B, L, nq, max_context):
    cfg = vyvo.Qwen3Config(**TINY, num_attention_heads=nq, num_key_value_heads=1)
    W = vyvo.init_weights(cfg, 77, std=0.08)
    ids = np.random.default_rng(L + B).integers(0, 2048, size=(B, L)).astype(np.int32)
    P = b2a.GenerateParameters(max_tokens=12, temperature=0.0, top_p=1.0, repetition_penalty=1.0, repetition_context_size=0)
    m_b, m_s = _models(b2a, monkeypatch, cfg, W, 8, max_context)
    a, _, n_a = _generate(b2a, m_b, ids, P)
    s, _, n_s = _generate(b2a, m_s, ids, P)
    assert n_s - n_a >= L - 1, (n_a, n_s, L)          # the replay launches a graph per prompt position, the batched pass a fixed count
    ref = vyvo.generate_tokens(vyvo.VyvoOracle(cfg, W), ids, 12, rep_penalty=1.0, rep_context=0)
    assert a == s == ref
    # the caches hold the prompt and all but the last generated token: the next position's logits
    nxt = np.asarray([[t[-1]] for t in a], dtype=np.int32)
    lb, ls = m_b(nxt, reset_cache=False), m_s(nxt, reset_cache=False)
    full = np.concatenate([ids, np.asarray(a, dtype=np.int32)], axis=1)
    ref_lg = vyvo.VyvoOracle(cfg, W).forward(full, head_positions=[full.shape[1] - 1]).numpy()
    print(f"B={B} L={L} G={nq}: batched vs step {rel_err(lb, ls):.2e}, vs oracle {rel_err(lb, ref_lg):.2e}")
    assert rel_err(lb, ls) < 4e-5, rel_err(lb, ls)
    assert rel_err(lb, ref_lg) < 1e-4, rel_err(lb, ref_lg)


def _stopping_weights(cfg, seed):
    """Untied head whose stop row is twice the row of the oracle's 5th greedy token: generation ends on 151671 within a few steps."""
    W = vyvo.init_weights(cfg, seed, std=0.05)
    ids = np.asarray([[11, 22, 33, vyvo.START_OF_SPEECH]], dtype=np.int32)
    t = vyvo.generate_tokens(vyvo.VyvoOracle(cfg, W), ids, 5)[0][4]
    W["lm_head.weight"][vyvo.END_OF_SPEECH] = (2.0 * W["lm_head.weight"][t].float()).to(torch.bfloat16)
    return W, ids


def test_greedy_stops_on_end_of_speech_with_the_full_vocabulary(b2a):
    cfg = vyvo.Qwen3Config(**{**TINY, "vocab_size": 180352}, num_attention_heads=2, num_key_value_heads=1)
    W, ids = _stopping_weights(cfg, 5)
    ref = vyvo.generate_tokens(vyvo.VyvoOracle(cfg, W), ids, 32)
    assert len(ref[0]) < 32 and vyvo.END_OF_SPEECH not in ref[0]          # the oracle stops
    m = b2a.Qwen3Model(config(cfg), W, max_batch=2, max_context=64)
    P = b2a.GenerateParameters(max_tokens=32, temperature=0.0, top_p=1.0, repetition_penalty=1.0, repetition_context_size=0)
    toks, _, info = m.generate_batch(ids, P, decode_audio=False)
    assert toks == ref and info.generation_token_count == len(ref[0])
    # the bench switch masks the stop token: fixed work
    toks, _, _ = m.generate_batch(ids, b2a.GenerateParameters(max_tokens=32, temperature=0.0, top_p=1.0, repetition_penalty=1.0,
                                                                repetition_context_size=0, mask_eos=True), decode_audio=False)
    assert len(toks[0]) == 32 and vyvo.END_OF_SPEECH not in toks[0]


def _snac(b2a, noise=True, encoder=False):
    scfg = osnac.SNACConfig(noise=noise)          # without NoiseBlocks the decoder's layer indices shift: weights for that layout
    SW = osnac.init_weights(scfg, 1234)
    if encoder:
        SW = {**SW, **ser.init_encoder_weights(scfg, 4321)}
    return b2a.SNAC(noise=noise, weights=SW)


def test_waveform_is_the_concatenated_50_frame_chunk_decodes(b2a):
    snac = _snac(b2a, noise=False)
    cfg = vyvo.Qwen3Config(**TINY, num_attention_heads=2, num_key_value_heads=1)
    W = vyvo.init_weights(cfg, 9, std=0.05)
    m = b2a.Qwen3Model(config(cfg), W, snac=snac, max_batch=2, max_context=512)
    ids = np.asarray([[11, 22, 33, vyvo.START_OF_SPEECH], [44, 55, 66, vyvo.START_OF_SPEECH]], dtype=np.int32)
    P = b2a.GenerateParameters(max_tokens=7 * 57 + 3, temperature=0.0, top_p=1.0, repetition_penalty=1.3, repetition_context_size=20,
                               mask_eos=True, wrap_codes=True)
    toks, waves, _ = m.generate_batch(ids, P)
    for b in range(2):
        cl = vyvo.parse_output_row(ids[b].tolist() + toks[b])
        cl = [((c % 4096) + 4096) % 4096 + 4096 * (i % 7) for i, c in enumerate(cl)]     # wrap_codes, as the handle applies it
        pieces = vyvo.decode_chunks(len(cl))
        assert [f for _, f in pieces] == [50, 7]
        want = np.concatenate([snac.decode(ol.codes_from_code_list(cl[7 * f0:7 * (f0 + n)])) [0, 0] for f0, n in pieces])
        assert waves[b].shape == want.shape == (57 * 2048,)
        assert np.abs(waves[b] - want).max() <= 1e-5 * np.abs(want).max()
        whole = snac.decode(ol.codes_from_code_list(cl))[0, 0]
        assert np.abs(whole - want).max() > 1e-3 * np.abs(want).max()        # a one-shot decode differs at the chunk boundary


def test_voice_cloning_prompt_from_a_3s_clip(b2a, monkeypatch):
    snac = _snac(b2a, encoder=True)
    cfg = vyvo.Qwen3Config(**{**TINY, "vocab_size": 180352}, num_attention_heads=2, num_key_value_heads=1)
    W = vyvo.init_weights(cfg, 99, std=0.05)
    m_b, m_s = _models(b2a, monkeypatch, cfg, W, 2, 512, snac=snac)
    clip = ser.synth_clip(1, 3 * 24000, seed=3)[0, 0]
    code_list = m_b.encode_audio_to_code_list(clip)
    ids, _ = m_b.prepare_input_ids([[11, 22, 33, 44], [55, 66]], code_list, list(range(1000, 1040)))
    assert 280 <= ids.shape[1] <= 330, ids.shape
    P = b2a.GenerateParameters(max_tokens=16, temperature=0.0, top_p=1.0, repetition_penalty=1.3, repetition_context_size=20, mask_eos=True)
    toks, info, n_b = _generate(b2a, m_b, ids, P)
    step, _, n_s = _generate(b2a, m_s, ids, P)
    assert n_s - n_b >= ids.shape[1] - 1, (n_b, n_s)
    ref = vyvo.generate_tokens(vyvo.VyvoOracle(cfg, W), ids, 16, rep_penalty=1.3, rep_context=20, mask_eos=True)
    assert toks == step == ref and info.prompt_token_count == ids.shape[1]


@pytest.mark.parametrize("variant", ["tied", "untied", "4bit"])
def test_from_model_directory(b2a, tmp_path, variant):
    cfg = vyvo.Qwen3Config(**TINY, num_attention_heads=2, num_key_value_heads=1, tie_word_embeddings=variant == "tied")
    W = vyvo.init_weights(cfg, 7, std=0.08)
    conf = {**config(cfg), "model_type": "qwen3"}
    files = {k: v.contiguous() for k, v in W.items()}
    ref_W = dict(W)
    if variant == "tied":
        files["lm_head.weight"] = torch.zeros_like(W["model.embed_tokens.weight"])       # sanitize drops it (Qwen3.swift:520-526)
    quant = {}
    if variant == "4bit":
        qname = "model.layers.1.mlp.down_proj"
        words, scales, biases, q = mlx_affine_quantize(W[qname + ".weight"].float().numpy(), 64, 4)
        deq = (np.repeat(scales, 64, axis=1) * q + np.repeat(biases, 64, axis=1)).astype(np.float32)
        ref_W[qname + ".weight"] = torch.from_numpy(deq).to(torch.bfloat16)
        del files[qname + ".weight"]
        quant = {qname + ".weight": words.view(np.int32), qname + ".scales": scales, qname + ".biases": biases}
        conf["quantization"] = {"group_size": 64, "bits": 4}
    d = tmp_path / variant
    d.mkdir()
    (d / "config.json").write_text(json.dumps(conf))
    save_file_torch(files, str(d / "model.safetensors"))
    if quant:
        save_file(quant, str(d / "model-quant.safetensors"))
    m = b2a.Qwen3Model.from_model_directory(d, max_batch=2, max_context=64)
    ids = np.asarray([[5, 17, 99, 4, 1000, 3], [8, 8, 2000, 31, 7, 6]], dtype=np.int32)
    ref = vyvo.VyvoOracle(cfg, ref_W).forward(ids).numpy()
    assert rel_err(m(ids), ref) < 1e-4


def test_errors(b2a, tmp_path):
    cfg = vyvo.Qwen3Config(**TINY, num_attention_heads=2, num_key_value_heads=1)
    W = vyvo.init_weights(cfg, 3, std=0.05)
    with pytest.raises(b2a.AudioGenerationError) as e:
        b2a.Qwen3Model({**config(cfg), "head_dim": 64}, W, max_batch=1, max_context=32)
    assert e.value.case == "invalidInput"
    with pytest.raises(b2a.AudioGenerationError) as e:
        b2a.Qwen3Model(config(cfg), {k: v for k, v in W.items() if k != "model.layers.1.self_attn.q_norm.weight"}, max_batch=1,
                       max_context=32)
    assert e.value.case == "modelNotInitialized" and "q_norm" in e.value.message
    m = b2a.Qwen3Model(config(cfg), W, max_batch=1, max_context=32)
    with pytest.raises(b2a.AudioGenerationError) as e:
        m.generate([1, 2, 3])
    assert e.value.case == "modelNotInitialized"
    P = b2a.GenerateParameters(max_tokens=4, temperature=0.0, top_p=1.0)
    with pytest.raises(b2a.AudioGenerationError) as e:
        m.generate_batch(np.asarray([[1, 2, 3]], dtype=np.int32), P)
    assert e.value.case == "modelNotInitialized"
