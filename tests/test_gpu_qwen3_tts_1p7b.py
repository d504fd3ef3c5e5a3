"""Qwen3-TTS talkers whose code predictor has another width than the talker (the 1.7B checkpoints: talker 2048, predictor 1024)
through the C ABI, against oracle/qwen3_tts.py.  code_predictor.small_to_mtp_projection (Qwen3TTSCodePredictor.swift:200-238) maps
every predictor input to the predictor's width (Qwen3TTS.swift:433-451): the talker's hidden state at position 0, and the codec /
predictor embedding rows after it.  Checked: talker logits and hidden state (< 1e-3), greedy frames bit-exact, batched rows,
sampling, the golden, the 1.7B widths at reduced talker depth with VoiceDesign and CustomVoice prompts, an ICL prompt, the
speaker encoder at enc_dim 2048 and directory loading (bf16 and 8-bit).  Weights are bf16-valued, as a checkpoint holds them."""
import json

import numpy as np
import pytest
import torch
from safetensors.numpy import save_file
from safetensors.torch import save_file as save_file_torch

from conftest import GOLDEN, rel_err
from oracle import qwen3_tts as ot
from test_gpu_qwen3_talker import CHAT, TTS, device_model
from test_gpu_qwen3_tts_icl import REF_CHAT, TARGET_CHAT, icl_prompt, oracle_rows, ref_codes
from test_loading import mlx_affine_quantize
from test_oracle_qwen3_tts_1p7b import golden_module

pytestmark = pytest.mark.gpu
TOL = 1e-3
mg = golden_module()
GEOMETRIES = {"narrow": (384, 256), "wide": (256, 384)}       # (talker hidden, predictor hidden)


@pytest.fixture(scope="module", params=list(GEOMETRIES))
def small(request, b2a):
    cfg = mg.config(*GEOMETRIES[request.param])
    W = mg.weights(cfg)
    return request.param, cfg, W, device_model(b2a, cfg, W, max_batch=4, max_context=128)


def greedy(b2a, n, **kw):
    return b2a.Qwen3GenerateParameters(max_tokens=n, temperature=0.0, repetition_penalty=1.05, mask_eos=True, **kw)


def oracle_frames(cfg, W, ri, rt, rp, n):
    return ot.generate_codes(cfg, W, ri, rt, rp, max_tokens=n, temperature=0.0, repetition_penalty=1.05, stop_on_eos=False).numpy()


def test_logits_and_hidden_vs_oracle(small):
    _, cfg, W, m = small
    ri, _, _ = ot.prepare_generation_inputs(cfg, W, CHAT, **TTS, language_id=2160)
    logits, hidden = m(ri.numpy().astype(np.float32))
    rl, rh = ot.Talker(cfg, W)(ri, None)
    assert hidden.shape == (1, cfg.hidden_size)
    assert rel_err(logits[0], rl[0, -1].numpy()) < TOL and rel_err(hidden[0], rh[0, -1].numpy()) < TOL


def test_greedy_frames_bit_exact_batched_rows_and_golden(b2a, small):
    name, cfg, W, m = small
    ri, rt, rp = ot.prepare_generation_inputs(cfg, W, CHAT, **TTS, language_id=2160)
    x, pad = ri.numpy().astype(np.float32), rp[0, 0].numpy()
    frames = []
    codes, info = m.generate_codes(x, [rt[0].numpy()], pad, greedy(b2a, 12), on_frame=lambda b, f, c: frames.append((b, f, c)))
    ref = oracle_frames(cfg, W, ri, rt, rp, 12)
    assert codes[0].shape == ref.shape == (12, cfg.num_code_groups)
    assert np.array_equal(codes[0], ref), (codes[0], ref)
    assert [f for _, f, _ in frames] == list(range(12)) and all(np.array_equal(c, ref[f]) for _, f, c in frames)
    if name == "narrow":
        assert np.array_equal(codes[0][:5], np.load(GOLDEN / "qwen3_talker_mtp.npz")["codes"])
    rt_short = rt[:, :3]
    c2, _ = m.generate_codes(np.stack([x[0], x[0]]), [rt[0].numpy(), rt_short[0].numpy()], pad, greedy(b2a, 12))
    assert np.array_equal(c2[0], ref) and np.array_equal(c2[1], oracle_frames(cfg, W, ri, rt_short, rp, 12))


def test_sampling_semantics(b2a, small):
    _, cfg, W, m = small
    ri, rt, rp = ot.prepare_generation_inputs(cfg, W, CHAT, **TTS, language_id=2160)
    x, tr, pad = ri.numpy().astype(np.float32), [rt[0].numpy()], rp[0, 0].numpy()
    kw = dict(max_tokens=8, temperature=0.9, top_k=50, top_p=0.95, repetition_penalty=1.05, mask_eos=True)
    a, _ = m.generate_codes(x, tr, pad, b2a.Qwen3GenerateParameters(seed=11, **kw))
    b, _ = m.generate_codes(x, tr, pad, b2a.Qwen3GenerateParameters(seed=11, **kw))
    c, _ = m.generate_codes(x, tr, pad, b2a.Qwen3GenerateParameters(seed=12, **kw))
    assert np.array_equal(a[0], b[0]) and not np.array_equal(a[0], c[0])
    assert (a[0][:, 0] < cfg.vocab_size - 1024).all() and (a[0][:, 1:] < cfg.code_predictor.vocab_size).all() and (a[0] >= 0).all()
    k1, _ = m.generate_codes(x, tr, pad, b2a.Qwen3GenerateParameters(max_tokens=5, temperature=0.7, top_k=1, repetition_penalty=1.05, mask_eos=True))
    g0, _ = m.generate_codes(x, tr, pad, greedy(b2a, 5))
    assert np.array_equal(k1[0], g0[0])


def test_icl_prompt_with_talker_width_xvector(b2a):
    cfg = mg.config()
    W = mg.weights(cfg, seed=5)
    m = device_model(b2a, cfg, W, max_batch=2, max_context=128)
    rc = ref_codes(cfg, 5, seed=3)
    spk = np.random.default_rng(1).standard_normal(cfg.hidden_size).astype(np.float32)
    inp, trail, pad = m.prepare_icl_generation_inputs(rc, REF_CHAT, TARGET_CHAT, **TTS, language_id=2160, speaker_embedding=spk)
    o, o_pad = icl_prompt(*oracle_rows(cfg, W), cfg, rc, REF_CHAT, TARGET_CHAT, **TTS, language_id=2160, speaker=spk.astype(np.float64))
    assert inp.shape == o.shape and rel_err(inp, o) < 1e-5 and rel_err(pad, o_pad[0]) < 1e-5
    codes, _ = m.generate_codes(o[None].astype(np.float32), [o_pad.astype(np.float32)], o_pad[0].astype(np.float32), greedy(b2a, 10))
    ri, rp = torch.from_numpy(o)[None], torch.from_numpy(o_pad)[None]
    ref = oracle_frames(cfg, W, ri, rp, rp, 10)
    assert codes[0].shape == ref.shape == (10, cfg.num_code_groups) and np.array_equal(codes[0], ref), (codes[0], ref)


def test_1p7b_widths_at_reduced_depth(b2a):
    """The 1.7B widths (talker 2048 / MLP 6144 / 16 q : 8 kv heads; predictor 1024 / 3072 / 5 layers, 16 code groups, codec vocabulary
    3072) with 2 talker layers instead of 28, so that the float64 oracle fits in host memory; depth changes no kernel.  The text
    table is cut to 512 rows (a gather).  VoiceDesign (instruct_ids) and CustomVoice (speaker_id) prompts."""
    cfg = ot.TalkerConfig(hidden_size=2048, intermediate_size=6144, num_hidden_layers=2, text_vocab_size=512)
    assert cfg.code_predictor.hidden_size == 1024 and cfg.text_hidden_size == 2048
    W = {k: v.to(torch.bfloat16).to(torch.float64) for k, v in ot.init_weights(cfg, 23, std=0.02).items()}
    m = device_model(b2a, cfg, W, max_batch=2, max_context=64)
    chat = [300, 12, 13] + list(range(40, 52)) + [301, 14, 300, 12, 13]
    prompts = {"language": dict(language_id=2160), "voice_design": dict(language_id=2160, instruct_ids=[300, 20, 21, 22, 23, 301, 14]),
               "custom_voice": dict(language_id=2161, speaker_id=2500)}
    for label, kw in prompts.items():
        ri, rt, rp = ot.prepare_generation_inputs(cfg, W, chat, tts_bos=400, tts_eos=401, tts_pad=402, **kw)
        inp, trail, pad = m.prepare_generation_inputs(chat, tts_bos=400, tts_eos=401, tts_pad=402, **kw)
        assert rel_err(inp, ri[0].numpy()) < 1e-5 and rel_err(trail, rt[0].numpy()) < 1e-5, label
        if label == "language":
            logits, hidden = m(ri.numpy().astype(np.float32))
            rl, rh = ot.Talker(cfg, W)(ri, None)
            e_l, e_h = rel_err(logits[0], rl[0, -1].numpy()), rel_err(hidden[0], rh[0, -1].numpy())
            assert e_l < TOL and e_h < TOL, (e_l, e_h)
        codes, _ = m.generate_codes(ri.numpy().astype(np.float32), [rt[0].numpy()], rp[0, 0].numpy(), greedy(b2a, 4))
        ref = oracle_frames(cfg, W, ri, rt, rp, 4)
        assert codes[0].shape == (4, 16) and np.array_equal(codes[0], ref), (label, codes[0], ref)


def test_speaker_encoder_at_talker_width_2048(b2a):
    """A 1.7B-Base checkpoint's x-vector has the talker's width: enc_dim 2048, the rest of the shipped speaker-encoder geometry."""
    import qwen3_speaker_encoder_reference as ser
    from test_gpu_qwen3_tts_speaker import errors, model
    cfg, W, m = model(b2a, seed=13, enc_dim=2048)
    x = ser.synth_clip(2, 3 * 24000, seed=9)
    got = m.embed(x)
    assert got.shape == (2, 2048)
    errors("embed enc_dim 2048", got, ser.embed(cfg, W, x))


def talker_config_json(cfg, quant=None):
    cp = cfg.code_predictor
    conf = {"model_type": "qwen3_tts",
            "talker_config": {"vocab_size": cfg.vocab_size, "hidden_size": cfg.hidden_size, "intermediate_size": cfg.intermediate_size,
                              "num_hidden_layers": cfg.num_hidden_layers, "num_attention_heads": cfg.num_attention_heads,
                              "num_key_value_heads": cfg.num_key_value_heads, "head_dim": cfg.head_dim, "num_code_groups": cfg.num_code_groups,
                              "text_hidden_size": cfg.text_hidden_size, "text_vocab_size": cfg.text_vocab_size,
                              "code_predictor_config": {"vocab_size": cp.vocab_size, "hidden_size": cp.hidden_size, "intermediate_size": cp.intermediate_size,
                                                        "num_hidden_layers": cp.num_hidden_layers, "num_attention_heads": cp.num_attention_heads,
                                                        "num_key_value_heads": cp.num_key_value_heads, "head_dim": cp.head_dim,
                                                        "num_code_groups": cp.num_code_groups}}}
    if quant:
        conf["quantization"] = quant
    return json.dumps(conf)


@pytest.mark.parametrize("bits", [None, 8])
def test_from_model_directory(b2a, tmp_path, bits):
    cfg = mg.config()
    W = mg.weights(cfg, seed=9)
    proj = "code_predictor.small_to_mtp_projection"
    qnames = [proj, "code_predictor.lm_head.1"] if bits else []
    Wd, quant = dict(W), {}
    for qn in qnames:
        words, scales, biases, q = mlx_affine_quantize(W[qn + ".weight"].to(torch.float32).numpy(), 64, bits)
        quant[qn] = (words, scales, biases)
        deq = (np.repeat(scales, 64, axis=1) * q + np.repeat(biases, 64, axis=1)).astype(np.float32)
        Wd[qn + ".weight"] = torch.from_numpy(deq).to(torch.bfloat16).to(torch.float64)
    ref_model = device_model(b2a, cfg, Wd, max_batch=2, max_context=64)
    d = tmp_path / "qwen3_1p7b"
    d.mkdir()
    (d / "config.json").write_text(talker_config_json(cfg, {"group_size": 64, "bits": bits} if bits else None))
    plain = {"talker." + k: v.to(torch.bfloat16).contiguous() for k, v in W.items() if not any(k == qn + ".weight" for qn in qnames)}
    save_file_torch(plain, str(d / "model.safetensors"))
    if bits:
        qd = {}
        for qn, (words, scales, biases) in quant.items():
            qd["talker." + qn + ".weight"], qd["talker." + qn + ".scales"], qd["talker." + qn + ".biases"] = words.view(np.int32), scales, biases
        save_file(qd, str(d / "model-quant.safetensors"))
    m = b2a.Qwen3TTSTalker.from_model_directory(d, max_batch=2, max_context=64)
    assert (m.config.hidden_size, m.config.code_predictor.hidden_size) == (cfg.hidden_size, cfg.code_predictor.hidden_size)
    ri, rt, rp = ot.prepare_generation_inputs(cfg, Wd, CHAT, **TTS, language_id=2160)
    x = ri.numpy().astype(np.float32)
    a, _ = m.generate_codes(x, [rt[0].numpy()], rp[0, 0].numpy(), greedy(b2a, 6))
    b, _ = ref_model.generate_codes(x, [rt[0].numpy()], rp[0, 0].numpy(), greedy(b2a, 6))
    assert a[0].shape == (6, cfg.num_code_groups) and np.array_equal(a[0], b[0])
    if not bits:
        assert np.array_equal(a[0], oracle_frames(cfg, W, ri, rt, rp, 6))


def test_missing_or_misshapen_projection_is_model_not_initialized(b2a, tmp_path):
    cfg = mg.config()
    W = {k: v.to(torch.bfloat16) for k, v in mg.weights(cfg, seed=9).items()}
    p = "code_predictor.small_to_mtp_projection."
    cases = {"no_weight": {k: v for k, v in W.items() if k != p + "weight"},
             "no_bias": {k: v for k, v in W.items() if k != p + "bias"},
             "short_bias": dict(W, **{p + "bias": W[p + "bias"][:-8]})}
    for label, Wc in cases.items():
        with pytest.raises(b2a.AudioGenerationError) as e:
            device_model(b2a, cfg, {k: v.to(torch.float64) for k, v in Wc.items()}, max_batch=1, max_context=32)
        assert e.value.case == "modelNotInitialized", label
    d = tmp_path / "noproj"
    d.mkdir()
    (d / "config.json").write_text(talker_config_json(cfg))
    save_file_torch({"talker." + k: v.contiguous() for k, v in cases["no_weight"].items()}, str(d / "model.safetensors"))
    with pytest.raises(b2a.AudioGenerationError) as e:
        b2a.Qwen3TTSTalker.from_model_directory(d, max_batch=1, max_context=32)
    assert e.value.case == "modelNotInitialized"
