"""Qwen3-TTS speaker encoder, CPU side: the float64 reference (tests/qwen3_speaker_encoder_reference.py) against transformers'
ECAPA_TimeDelayNet (the same architecture with reflect "same" padding), the library's config parsing and sanitize (host code, no
device needed), and the golden fixture."""
import json
import types

import numpy as np
import pytest
import torch

import qwen3_speaker_encoder_reference as ser
from conftest import GOLDEN

SMALL = dict(enc_channels=[96, 96, 96, 192], enc_kernel_sizes=[5, 3, 3, 3], enc_dilations=[1, 2, 3, 1], enc_attention_channels=80,
             enc_res2net_scale=4, enc_se_channels=72, enc_dim=48)


def cfg_of(**kw):
    from mlx_audio_swift_b200.qwen3_tts import Qwen3SpeakerEncoderConfig
    return Qwen3SpeakerEncoderConfig(**kw)


def weights(cfg, seed=3):
    from mlx_audio_swift_b200.qwen3_tts import random_init_speaker_encoder_weights
    return random_init_speaker_encoder_weights(cfg, seed=seed)


@pytest.mark.parametrize("geometry", ["small", "shipped"])
def test_reference_matches_transformers_ecapa(geometry):
    from transformers.models.qwen2_5_omni.modeling_qwen2_5_omni import ECAPA_TimeDelayNet
    cfg = cfg_of(**SMALL) if geometry == "small" else cfg_of()
    W = weights(cfg)
    hf = ECAPA_TimeDelayNet(types.SimpleNamespace(**{k: getattr(cfg, k) for k in (
        "mel_dim", "enc_dim", "enc_channels", "enc_kernel_sizes", "enc_dilations", "enc_attention_channels", "enc_res2net_scale",
        "enc_se_channels")})).double().eval()
    sd = hf.state_dict()
    assert sd.keys() == W.keys()
    hf.load_state_dict({k: torch.as_tensor(v, dtype=torch.float64) for k, v in W.items()})
    x = ser.synth_clip(2, 9000, seed=1)
    mel = np.stack([ser.log_mel(r) for r in x])
    assert mel.shape == (2, ser.frames(9000), 128)
    with torch.no_grad():
        want = hf(torch.as_tensor(mel)).numpy()
    got = ser.forward(cfg, W, mel)
    assert got.shape == (2, cfg.enc_dim)
    assert np.abs(got - want).max() < 1e-9 * np.abs(want).max()


def test_shortest_input_pads_without_clamping():
    # 1024 samples -> 5 frames, the fewest the shipped geometry accepts: the widest pad (k 3, dilation 4) is 4 < T
    cfg = cfg_of()
    assert ser.frames(1023) == 4 and ser.frames(1024) == 5
    assert max((k - 1) * d // 2 for k, d in zip(cfg.enc_kernel_sizes, cfg.enc_dilations)) == 4


def test_config_from_json(b2a, tmp_path):
    from mlx_audio_swift_b200 import _ffi
    from mlx_audio_swift_b200.qwen3_tts import Qwen3SpeakerEncoderConfig
    import ctypes as C
    p = tmp_path / "config.json"
    c = _ffi.Qwen3SpeakerEncoderConfig()
    p.write_text(json.dumps({"tts_model_type": "base"}))                       # no block: every default
    _ffi.check(_ffi.lib().b2a_qwen3_speaker_encoder_config_from_json(str(p).encode(), C.byref(c)))
    assert Qwen3SpeakerEncoderConfig.from_ffi(c) == Qwen3SpeakerEncoderConfig()
    p.write_text(json.dumps({"speaker_encoder_config": {"enc_dim": 2048, "enc_channels": [256, 256, 256, 512], "enc_kernel_sizes": [5, 3, 3, 1],
                                                        "enc_dilations": [1, 2, 3, 1], "sample_rate": 16000}}))
    _ffi.check(_ffi.lib().b2a_qwen3_speaker_encoder_config_from_json(str(p).encode(), C.byref(c)))
    got = Qwen3SpeakerEncoderConfig.from_ffi(c)
    assert got == Qwen3SpeakerEncoderConfig(enc_dim=2048, enc_channels=[256, 256, 256, 512], enc_kernel_sizes=[5, 3, 3, 1],
                                            enc_dilations=[1, 2, 3, 1], sample_rate=16000)
    assert got.to_ffi().num_enc_layers == 4
    p.write_text(json.dumps({"speaker_encoder_config": {"enc_channels": [256, 256, 512]}}))        # lists of unequal length
    with pytest.raises(_ffi.AudioGenerationError) as e:
        _ffi.check(_ffi.lib().b2a_qwen3_speaker_encoder_config_from_json(str(p).encode(), C.byref(c)))
    assert e.value.case == "invalidInput"
    with pytest.raises(_ffi.AudioGenerationError) as e:
        Qwen3SpeakerEncoderConfig(enc_channels=[256, 256, 512]).to_ffi()
    assert e.value.case == "invalidInput"


@pytest.mark.parametrize("prefix", ["speaker_encoder.", "model.speaker_encoder."])
def test_sanitize_key_for_key(b2a, tmp_path, prefix):
    from safetensors.numpy import save_file
    cfg = cfg_of(**SMALL)
    W = weights(cfg)
    ck = {prefix + k: v for k, v in W.items()}
    ck["blocks.1.se_block.conv1.weight"] = np.zeros((2, 2, 1), np.float32)       # no speaker_encoder component: dropped
    ck["talker.model.norm.weight"] = np.zeros(4, np.float32)
    ck["speaker_encoder"] = np.zeros(1, np.float32)                               # nothing after the component: dropped
    mlx_layout = {prefix + "fc.weight": W["fc.weight"].transpose(0, 2, 1).copy()}  # already [out, k, in]: kept
    ref = ser.sanitize({**ck, **mlx_layout})
    assert ref.keys() == W.keys()
    for k, v in W.items():                                                        # every weight of this geometry is transposed once
        assert np.array_equal(ref[k], v.transpose(0, 2, 1) if v.ndim == 3 else v), k
    save_file({**ck, **mlx_layout}, str(tmp_path / "m.safetensors"))
    w = b2a.loading.Weights(tmp_path / "m.safetensors")
    w.sanitize_qwen3_speaker_encoder()
    got = w.tensors()
    assert got.keys() == ref.keys()
    for k, v in ref.items():
        assert got[k].shape == v.shape and np.array_equal(got[k], v.astype(np.float32)), k


def test_golden_reproduces():
    import sys
    sys.path.insert(0, str(GOLDEN))
    import make_golden_qwen3_speaker as mg
    g = np.load(GOLDEN / "qwen3_speaker.npz")
    cfg, W = mg.weights()
    assert [int(v) for v in g["clip"]] == [mg.BATCH, mg.N_SAMPLES, mg.CLIP_SEED] and list(g["enc_channels"]) == cfg.enc_channels
    got = ser.embed(cfg, W, mg.clip())
    assert np.abs(got - g["embedding"]).max() < 1e-9 * np.abs(g["embedding"]).max()
