"""The float64 Qwen3-TTS speech-tokenizer encoder reference (tests/qwen3_encoder_reference.py) pinned against
transformers.MimiModel (random init, float64) on a Qwen3-layout checkpoint run through the restated sanitize; the sanitize key
for key against the library's; the encoded-length rule; the golden fixture.  CPU only."""
import json

import numpy as np
import pytest
import torch

import qwen3_encoder_reference as qer
from conftest import GOLDEN

SMALL_HF = dict(hidden_size=64, num_filters=8, upsampling_ratios=[8, 6, 5, 4], num_attention_heads=2, num_key_value_heads=2, head_dim=32,
                intermediate_size=128, num_hidden_layers=2, codebook_size=64, codebook_dim=16, vector_quantization_hidden_dimension=16,
                num_quantizers=8, num_semantic_quantizers=1, sliding_window=250, use_causal_conv=True, frame_rate=12.5, sampling_rate=24000,
                upsample_groups=64)


def small_cfg(b2a=None, **kw):
    from mlx_audio_swift_b200.qwen3_tts_codec import Qwen3TTSTokenizerEncoderConfig
    d = dict(hidden_size=64, num_filters=8, num_attention_heads=2, num_key_value_heads=2, intermediate_size=128, num_hidden_layers=2,
             codebook_size=64, codebook_dim=16, num_quantizers=8, valid_num_quantizers=8)
    d.update(kw)
    return Qwen3TTSTokenizerEncoderConfig(**d)


def hf_model(seed=0):
    from transformers import MimiConfig, MimiModel
    torch.manual_seed(seed)
    m = MimiModel(MimiConfig(**SMALL_HF)).double().eval()
    with torch.no_grad():                   # make the layer scales and norms matter, and give the codebooks spread-out usages
        for name, p in m.named_parameters():
            if "layer_scale" in name:
                p.copy_(0.3 + 0.2 * torch.rand_like(p))
            elif "norm" in name and name.endswith("weight"):
                p.copy_(1 + 0.1 * torch.randn_like(p))
            elif "norm" in name and name.endswith("bias"):
                p.copy_(0.05 * torch.randn_like(p))
        for name, b in m.named_buffers():
            if name.endswith("cluster_usage"):
                b.copy_(0.5 + 1.5 * torch.rand_like(b))
            elif name.endswith("embed_sum"):
                b.copy_(torch.randn_like(b) * 0.5)
    return m


def qwen3_checkpoint(m, fused_qkv=False):
    """{"encoder." + k: v} over MimiModel.state_dict(), q / k rows permuted per head so that the reference's interleaved RoPE
    equals HF's rotate-half."""
    cfg = m.config
    perm = qer.hf_qk_permutation(cfg.num_attention_heads, cfg.head_dim)
    ck = {}
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    for k, v in sd.items():
        if ".self_attn.q_proj.weight" in k or ".self_attn.k_proj.weight" in k:
            v = v[perm]
        ck["encoder." + k] = v
    if fused_qkv:
        for l in range(cfg.num_hidden_layers):
            p = f"encoder.encoder_transformer.layers.{l}.self_attn."
            ck[p + "qkv.weight"] = np.concatenate([ck.pop(p + f"{n}_proj.weight") for n in "qkv"], 0)
    return ck


def test_reference_matches_transformers_mimi():
    m = hf_model()
    cfg = small_cfg(valid_num_quantizers=8)
    W = qer.sanitize_encoder(qwen3_checkpoint(m))
    x = qer.synth_clip(2, 24000 * 3 + 517, seed=3)       # 76 encoder frames (< 250: the window does not bite)
    with torch.no_grad():
        xt = torch.from_numpy(x).double()
        e = m.encoder(xt)
        e = m.encoder_transformer(e.transpose(1, 2))[0].transpose(1, 2)
        z_hf = m.downsample(e).transpose(1, 2).numpy()
        codes_hf = m.quantizer.encode(m.downsample(e), num_quantizers=8).transpose(0, 1).numpy()
    z = qer.latent(cfg, W, x)
    assert z.shape == z_hf.shape == (2, qer.encoded_length(x.shape[-1], cfg.upsampling_ratios, 2), 64)
    err = np.abs(z - z_hf).max() / np.abs(z_hf).max()
    assert err < 1e-9, err
    codes, gaps, scale = qer.encode_codes(cfg, W, z, with_gaps=True)
    diff = codes != codes_hf
    for b, t in zip(*np.nonzero(diff.any(1))):          # only float64 near-ties may flip (then finer levels are exempt)
        q = int(np.argmax(diff[b, :, t]))
        assert gaps[b, q, t] < 1e-9 * scale[b, q, t], (b, q, t)
    assert diff.any(1).mean() < 0.02


def test_transformers_applies_the_window_the_reference_does_not():
    """Past 250 encoder frames MimiModel's sliding window drops keys; the reference's one-shot encode does not (trap 2)."""
    m = hf_model(1)
    cfg = small_cfg()
    W = qer.sanitize_encoder(qwen3_checkpoint(m))
    x = qer.synth_clip(1, 960 * 300, seed=4)
    with torch.no_grad():
        e = m.encoder(torch.from_numpy(x).double())
        h_hf = m.encoder_transformer(e.transpose(1, 2))[0].numpy()
    x0 = qer.seanet(cfg, W, x).transpose(1, 2)
    full, windowed = qer.transformer(cfg, W, x0).numpy(), qer.transformer(cfg, W, x0, window=250).numpy()
    assert np.abs(windowed - h_hf).max() < 1e-9 * np.abs(h_hf).max()
    assert np.abs(full[:, :250] - h_hf[:, :250]).max() < 1e-9 * np.abs(h_hf).max()
    assert np.abs(full[:, 250:] - h_hf[:, 250:]).max() > 1e-6 * np.abs(h_hf).max()


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("prefix", ["", "speech_tokenizer."])
def test_sanitize_key_for_key(b2a, tmp_path, fused, prefix):
    from safetensors.numpy import save_file
    m = hf_model(2)
    ck = {prefix + k: np.ascontiguousarray(v, np.float32) for k, v in qwen3_checkpoint(m, fused_qkv=fused).items()}
    ck[prefix + "decoder.quantizer.rvq_first.vq.layers.0._codebook.embedding_sum"] = np.zeros((4, 2), np.float32)
    ck[prefix + "speaker_encoder.fc.weight"] = np.zeros((2, 2), np.float32)
    # the rvq_first / rvq_rest spelling of the quantizer prefixes maps to the same keys
    renamed = {k.replace("semantic_residual_vector_quantizer", "rvq_first").replace("acoustic_residual_vector_quantizer", "rvq_rest"): v
               for k, v in ck.items()}
    ref = qer.sanitize_encoder(ck)
    assert qer.sanitize_encoder(renamed).keys() == ref.keys()
    assert "encoder_transformer.transformer.layers.1.self_attn.in_proj.weight" in ref
    assert "quantizer.rvq_rest.vq.layers.6.codebook.embedding_sum" in ref and "downsample.conv.conv.conv.weight" in ref
    assert not any(k.startswith("decoder") or "speaker" in k for k in ref)
    for i, d in enumerate((ck, renamed)):
        save_file(d, str(tmp_path / f"m{i}.safetensors"))
        w = b2a.loading.Weights(tmp_path / f"m{i}.safetensors")
        w.sanitize_speech_tokenizer_encoder()
        got = w.tensors()
        assert got.keys() == ref.keys()
        for k, v in ref.items():
            assert got[k].shape == v.shape and np.array_equal(got[k], v.astype(np.float32)), k


def test_encoded_length_rule():
    for n in [1, 2, 959, 960, 961, 1919, 1920, 1921, 3839, 3840, 3841, 24000, 1920 * 375, 1920 * 375 + 1]:
        assert qer.encoded_length(n, [8, 6, 5, 4], 2) == -(-(-(-n // 960)) // 2), n


def test_config_from_json(b2a, tmp_path):
    from mlx_audio_swift_b200 import _ffi
    import ctypes as C
    p = tmp_path / "config.json"
    c = _ffi.SpeechTokenizerEncoderConfig()
    with pytest.raises(_ffi.AudioGenerationError) as e:             # no file: no encoder
        _ffi.check(_ffi.lib().b2a_speech_tokenizer_encoder_config_from_json(str(p).encode(), C.byref(c)))
    assert e.value.case == "modelNotInitialized"
    p.write_text(json.dumps({"decoder_config": {}}))
    with pytest.raises(_ffi.AudioGenerationError) as e:             # decoder-only config
        _ffi.check(_ffi.lib().b2a_speech_tokenizer_encoder_config_from_json(str(p).encode(), C.byref(c)))
    assert e.value.case == "modelNotInitialized"
    p.write_text(json.dumps({"encoder_config": {"num_filters": 32, "upsampling_ratios": [4, 4]}, "encoder_valid_num_quantizers": 8}))
    _ffi.check(_ffi.lib().b2a_speech_tokenizer_encoder_config_from_json(str(p).encode(), C.byref(c)))
    assert (c.num_filters, c.num_upsampling_ratios, list(c.upsampling_ratios)[:2], c.valid_num_quantizers) == (32, 2, [4, 4], 8)
    assert (c.hidden_size, c.head_dim, c.num_quantizers, c.codebook_dim, c.kernel_size, c.last_kernel_size) == (512, 64, 32, 256, 7, 3)
    assert abs(c.frame_rate - 12.5) < 1e-6 and c.sampling_rate == 24000 and c.use_causal_conv == 1 and c.use_conv_shortcut == 0


def test_golden_reproduces():
    import sys
    sys.path.insert(0, str(GOLDEN))
    import make_golden_qwen3_encode as mg
    g = np.load(GOLDEN / "qwen3_encode.npz")
    cfg, W = mg.weights()
    x = qer.synth_clip(mg.BATCH, mg.N_SAMPLES, mg.CLIP_SEED)
    z = qer.latent(cfg, W, x)
    assert np.abs(z.reshape(-1)[:32] - g["z_first"]).max() < 1e-6 * np.abs(g["z_first"]).max()
    assert np.array_equal(qer.encode_codes(cfg, W, z), g["codes"])
