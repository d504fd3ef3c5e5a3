"""Qwen3-TTS 1.7B checkpoints, host side: the float64 oracle reproduces the committed golden of a talker whose code predictor is
narrower than the talker (code_predictor.small_to_mtp_projection, Qwen3TTSCodePredictor.swift:200-238); a 1.7B-style config.json
decodes to both widths; sanitize keeps the projection's keys and expands an 8-bit projection like every other Linear."""
import ctypes as C
import importlib.util
import json

import numpy as np
import torch
from safetensors.numpy import save_file

from conftest import GOLDEN
from test_loading import mlx_affine_quantize


def golden_module():
    spec = importlib.util.spec_from_file_location("make_golden_qwen3_mtp", GOLDEN / "make_golden_qwen3_mtp.py")
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
    return mg


def test_oracle_reproduces_committed_projection_golden():
    mg = golden_module()
    g = np.load(GOLDEN / "qwen3_talker_mtp.npz")
    cfg = mg.config()
    assert cfg.hidden_size != cfg.code_predictor.hidden_size
    assert "code_predictor.small_to_mtp_projection.weight" in mg.weights(cfg)
    got = mg.make()
    assert np.array_equal(got["codes"], g["codes"]) and g["codes"].shape == (5, cfg.num_code_groups)
    assert np.array_equal(got["first_logits_top"], g["first_logits_top"])
    assert np.allclose(got["first_logits_stats"], g["first_logits_stats"], rtol=1e-9, atol=1e-12)


def test_config_from_json_reads_both_widths(b2a, tmp_path):
    f = b2a._ffi
    (tmp_path / "config.json").write_text(json.dumps({
        "model_type": "qwen3_tts", "tts_model_type": "voice_design",
        "talker_config": {"hidden_size": 2048, "intermediate_size": 6144, "num_hidden_layers": 28, "num_attention_heads": 16,
                          "num_key_value_heads": 8, "text_hidden_size": 2048,
                          "code_predictor_config": {"hidden_size": 1024, "intermediate_size": 3072, "num_hidden_layers": 5}}}))
    c = f.Qwen3TalkerConfig()
    f.check(f.lib().b2a_qwen3_talker_config_from_json(str(tmp_path / "config.json").encode(), 8, 2048, C.byref(c)))
    assert (c.hidden_size, c.intermediate_size, c.num_hidden_layers, c.text_hidden_size) == (2048, 6144, 28, 2048)
    assert (c.cp_hidden_size, c.cp_intermediate_size, c.cp_num_hidden_layers, c.cp_vocab_size) == (1024, 3072, 5, 2048)


def test_sanitize_keeps_the_projection_and_expands_an_8bit_one(b2a, tmp_path):
    f = b2a._ffi
    (tmp_path / "config.json").write_text(json.dumps({"model_type": "qwen3_tts", "quantization": {"group_size": 64, "bits": 8}}))
    rng = np.random.default_rng(3)
    wp = rng.standard_normal((32, 128)).astype(np.float32)
    words, scales, biases, q = mlx_affine_quantize(wp, 64, 8)
    bias = rng.standard_normal(32).astype(np.float32)
    p = "talker.code_predictor.small_to_mtp_projection."
    save_file({p + "weight": words.view(np.int32), p + "scales": scales, p + "biases": biases, p + "bias": bias,
               "talker.code_predictor.lm_head.0.weight": np.ones((4, 32), np.float32),
               "speaker_encoder.fc.weight": np.ones((2, 2), np.float32)}, str(tmp_path / "model.safetensors"))
    w = b2a.Weights(tmp_path)
    f.check(f.lib().b2a_weights_sanitize_qwen3_talker(w._h, str(tmp_path / "config.json").encode()))
    t = w.tensors()
    assert set(t) == {"code_predictor.small_to_mtp_projection.weight", "code_predictor.small_to_mtp_projection.bias",
                      "code_predictor.lm_head.0.weight"}
    ref = (np.repeat(scales, 64, axis=1) * q + np.repeat(biases, 64, axis=1)).astype(np.float32)
    assert torch.equal(t["code_predictor.small_to_mtp_projection.weight"], torch.from_numpy(ref).to(torch.bfloat16))
    assert np.array_equal(np.asarray(t["code_predictor.small_to_mtp_projection.bias"]), bias)
