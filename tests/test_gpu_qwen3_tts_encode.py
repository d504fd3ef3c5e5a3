"""CUDA Qwen3-TTS speech-tokenizer encode (through the C ABI) against the float64 reference (tests/qwen3_encoder_reference.py,
itself pinned against transformers.MimiModel in test_oracle_qwen3_tts_encode.py).

z (the code search's input): max |diff| / max |ref| below 1e-3.  Codes: bit-exact against the ordered-fp32 search run on the
device's own z; against the float64 end-to-end reference a frame's first differing level must be a float64 near-tie (its finer
levels then search a different residual and are exempt)."""
import json

import numpy as np
import pytest
import torch

import qwen3_encoder_reference as qer
from conftest import max_rel_to_peak, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-3
TIE_REL = 1e-4     # float64 distance gap, relative to |x|^2 + 1, below which a level's search counts as a near-tie
SMALL = dict(hidden_size=64, num_filters=8, num_attention_heads=2, num_key_value_heads=2, intermediate_size=128, num_hidden_layers=2,
             codebook_size=64, codebook_dim=16, num_quantizers=8, valid_num_quantizers=8)


def model(b2a, seed=7, **kw):
    from mlx_audio_swift_b200 import qwen3_tts_codec as q
    cfg = q.Qwen3TTSTokenizerEncoderConfig(**kw)
    W = q.random_init_encoder_weights(cfg, seed=seed, layer_scale=0.3)
    return cfg, W, q.Qwen3TTSSpeechTokenizerEncoder(cfg, weights=W)


@pytest.fixture(scope="module")
def small(b2a):
    return model(b2a, **SMALL)


@pytest.fixture(scope="module")
def shipped(b2a):
    return model(b2a, seed=11)


def assert_codes_explained(cfg, W, dev, z64):
    ref, gaps, scale = qer.encode_codes(cfg, W, z64, with_gaps=True)
    diff = dev != ref
    for b, t in zip(*np.nonzero(diff.any(1))):
        q = int(np.argmax(diff[b, :, t]))
        assert gaps[b, q, t] < TIE_REL * scale[b, q, t], (b, q, t, gaps[b, q, t], scale[b, q, t])
    return float(diff.any(1).mean())


def check_against_float64(cfg, W, m, x, label):
    z, codes = m.encode_latent(x)
    T = qer.encoded_length(x.shape[-1], cfg.upsampling_ratios, cfg.downsample_stride)
    assert z.shape == (x.shape[0], T, cfg.hidden_size) and codes.shape == (x.shape[0], cfg.num_code_groups, T)
    assert m.encoded_length(x.shape[-1]) == T
    z64 = qer.latent(cfg, W, x)
    err_peak, err_l2 = max_rel_to_peak(z, z64), rel_err(z, z64)
    print(f"{label}: z error max/peak {err_peak:.2e}, rel L2 {err_l2:.2e}")
    assert err_peak < TOL and err_l2 < TOL
    assert np.array_equal(codes, qer.encode_codes_fp32(cfg, W, z))
    frac = assert_codes_explained(cfg, W, codes, z64)
    print(f"{label}: frames whose codes differ from float64 (near-ties only): {frac:.3f}")
    assert np.array_equal(m.encode(x), codes)
    return codes


@pytest.mark.parametrize("B,n", [(2, 96000), (3, 24017), (1, 1)])
def test_small_vs_float64(b2a, small, B, n):
    cfg, W, m = small
    x = qer.synth_clip(B, n, seed=n)
    if B > 1:
        x[1] *= 0.25
    check_against_float64(cfg, W, m, x, f"small B={B} n={n}")


def test_shipped_geometry_vs_float64(b2a, shipped):
    cfg, W, m = shipped
    x = qer.synth_clip(2, 4 * 24000, seed=5)
    codes = check_against_float64(cfg, W, m, x, "shipped 2 x 4 s")
    assert codes.shape == (2, 16, 50)


def test_past_250_frames_attends_full_causal(b2a, small):
    """24 s = 600 encoder frames: the device matches the full-causal reference, not the 250-frame window of transformers."""
    cfg, W, m = small
    x = qer.synth_clip(1, 24 * 24000, seed=8)
    z, _ = m.encode_latent(x)
    z64 = qer.latent(cfg, W, x)
    err = max_rel_to_peak(z, z64)
    print(f"small 1 x 24 s: z error max/peak {err:.2e}")
    assert err < TOL
    assert max_rel_to_peak(z, qer.latent(cfg, W, x, window=250)) > 10 * err


def test_golden(b2a):
    import sys
    from conftest import GOLDEN
    sys.path.insert(0, str(GOLDEN))
    import make_golden_qwen3_encode as mg
    from mlx_audio_swift_b200 import qwen3_tts_codec as q
    g = np.load(GOLDEN / "qwen3_encode.npz")
    cfg, W = mg.weights()
    m = q.Qwen3TTSSpeechTokenizerEncoder(cfg, weights=W)
    x = qer.synth_clip(mg.BATCH, mg.N_SAMPLES, mg.CLIP_SEED)
    z, codes = m.encode_latent(x)
    assert z.shape == tuple(g["z_shape"]) and codes.shape == g["codes"].shape
    assert np.abs(z.reshape(-1)[:32] - g["z_first"]).max() < TOL * max(abs(g["z_stats"][2]), abs(g["z_stats"][3]))
    z64 = qer.latent(cfg, W, x)
    assert np.array_equal(qer.encode_codes(cfg, W, z64), g["codes"])
    assert_codes_explained(cfg, W, codes, z64)         # a code may differ from the fixture only at a float64 near-tie


def test_batched_serial_device_entry_deterministic(b2a, small):
    cfg, W, m = small
    x = qer.synth_clip(3, 40000, seed=11)
    x[2] *= 3.0
    codes = m.encode(x)
    for b in range(3):
        assert np.array_equal(m.encode(x[b:b + 1]), codes[b:b + 1])
    assert np.array_equal(m.encode(x), codes)
    d_x = torch.from_numpy(x).cuda()
    d_codes = torch.empty(codes.shape, dtype=torch.int32, device="cuda")
    m.encode_dev(d_x, d_codes)
    torch.cuda.synchronize()
    assert np.array_equal(d_codes.cpu().numpy(), codes)
    s = torch.cuda.Stream()
    d2 = torch.zeros_like(d_codes)
    m.encode_dev(d_x, d2, stream=s.cuda_stream)
    s.synchronize()
    assert torch.equal(d2, d_codes)


def test_shipped_8x30s_prefix_and_lengths(b2a, shipped):
    cfg, W, m = shipped
    n = 30 * 24000
    x = qer.synth_clip(8, n, seed=12)
    codes = m.encode(x)
    assert codes.shape == (8, 16, 375)
    K = 1920 * 100                                       # a 8 s prefix: its 100 frames see only samples inside it
    assert np.array_equal(m.encode(np.ascontiguousarray(x[:, :, :K])), codes[:, :, :100])
    y = qer.synth_clip(1, 1920 * 375 + 1, seed=14)
    for k in (1, 2, 375):
        for d in (-1, 0, 1):
            nn = 1920 * k + d
            assert m.encoded_length(nn) == -(-(-(-nn // 960)) // 2)
            assert m.encode(np.ascontiguousarray(y[:, :, :nn])).shape == (1, 16, m.encoded_length(nn))


def test_errors(b2a, small, tmp_path):
    from mlx_audio_swift_b200 import _ffi
    from mlx_audio_swift_b200 import qwen3_tts_codec as q
    cfg, W, m = small

    def case(fn):
        with pytest.raises(_ffi.AudioGenerationError) as e:
            fn()
        return e.value.case

    assert case(lambda: m.encode(np.zeros((1, 1, 0), np.float32))) == "audioEncodingFailed"
    for bad in (dict(audio_channels=2), dict(num_residual_layers=2), dict(use_conv_shortcut=True), dict(num_key_value_heads=1)):
        c = q.Qwen3TTSTokenizerEncoderConfig(**{**SMALL, **bad})
        assert case(lambda: q.Qwen3TTSSpeechTokenizerEncoder(c, weights=W)) == "invalidInput"
    dec_only = {k: v for k, v in W.items() if not k.startswith("encoder.")}
    assert case(lambda: q.Qwen3TTSSpeechTokenizerEncoder(cfg, weights=dec_only)) == "modelNotInitialized"
    # a decoder-only speech_tokenizer directory: no encoder_config, then no encoder keys
    from safetensors.numpy import save_file
    save_file({"decoder.pre_conv.conv.weight": np.zeros((4, 3, 8), np.float32)}, str(tmp_path / "model.safetensors"))
    (tmp_path / "config.json").write_text(json.dumps({"decoder_config": {}}))
    assert case(lambda: q.Qwen3TTSSpeechTokenizerEncoder.from_model_directory(tmp_path)) == "modelNotInitialized"
    (tmp_path / "config.json").write_text(json.dumps({"encoder_config": {}}))
    assert case(lambda: q.Qwen3TTSSpeechTokenizerEncoder.from_model_directory(tmp_path)) == "modelNotInitialized"
    # mismatched device tensors
    d_x = torch.zeros((1, 1, 4000), dtype=torch.float32, device="cuda")
    T = m.encoded_length(4000)
    assert case(lambda: m.encode_dev(d_x, torch.zeros((1, 8, T + 1), dtype=torch.int32, device="cuda"))) == "invalidInput"
    assert case(lambda: m.encode_dev(d_x, torch.zeros((1, 8, T), dtype=torch.int64, device="cuda"))) == "invalidInput"
    assert case(lambda: m.encode_dev(d_x.cpu(), torch.zeros((1, 8, T), dtype=torch.int32, device="cuda"))) == "invalidInput"
    assert case(lambda: m.encode(np.zeros((1, 2, 100), np.float32))) == "invalidInput"
    # sizes whose indices would overflow
    lib = _ffi.lib()
    assert case(lambda: _ffi.check(lib.b2a_speech_tokenizer_encoder_encode_dev(m._h, _ffi.ptr(d_x), 4, 1 << 30, _ffi.ptr(d_x), None))) == "invalidInput"


def test_from_directory_and_tokenizer_encode(b2a, small, tmp_path):
    """A Qwen3-layout checkpoint directory loads through the library's sanitize; Qwen3TTSSpeechTokenizer.encode takes 1-D / 2-D /
    3-D audio; encode -> decode round trip gives the decoder's length and finite audio (random weights: no meaningful audio)."""
    from safetensors.numpy import save_file
    from mlx_audio_swift_b200 import qwen3_tts_codec as q
    from test_oracle_qwen3_tts_encode import SMALL_HF, hf_model, qwen3_checkpoint
    hf = hf_model(3)
    ck = {"speech_tokenizer." + k: np.ascontiguousarray(v, np.float32) for k, v in qwen3_checkpoint(hf).items()}
    save_file(ck, str(tmp_path / "model.safetensors"))
    enc_cfg = {k: SMALL_HF[k] for k in ("hidden_size", "num_filters", "upsampling_ratios", "num_attention_heads", "num_key_value_heads",
                                        "intermediate_size", "num_hidden_layers", "codebook_size", "codebook_dim", "num_quantizers")}
    (tmp_path / "config.json").write_text(json.dumps({"encoder_config": enc_cfg, "encoder_valid_num_quantizers": 8}))
    m = q.Qwen3TTSSpeechTokenizerEncoder.from_model_directory(tmp_path)
    cfg = q.Qwen3TTSTokenizerEncoderConfig(**{**SMALL, "upsampling_ratios": [8, 6, 5, 4]})
    W = qer.sanitize_encoder(ck)
    x = qer.synth_clip(2, 30000, seed=13)
    z, codes = m.encode_latent(x)
    assert max_rel_to_peak(z, qer.latent(cfg, W, x)) < TOL
    assert np.array_equal(codes, qer.encode_codes_fp32(cfg, W, z))
    dcfg = q.Qwen3TTSTokenizerDecoderConfig(codebook_size=64, codebook_dim=32, latent_dim=64, decoder_dim=128, hidden_size=64, intermediate_size=128,
                                            num_attention_heads=2, num_key_value_heads=2, num_hidden_layers=1, num_quantizers=8,
                                            upsample_rates=[8, 5, 4, 3], upsampling_ratios=[2, 2])
    tok = q.Qwen3TTSSpeechTokenizer(dcfg, weights=q.random_init_weights(dcfg), max_batch=2, encoder=m)
    assert tok.has_encoder and not q.Qwen3TTSSpeechTokenizer(dcfg, weights=q.random_init_weights(dcfg)).has_encoder
    assert np.array_equal(tok.encode(x[0, 0]), codes[:1]) and np.array_equal(tok.encode(x[:, 0]), codes) and np.array_equal(tok.encode(x), codes)
    wav, lengths = tok.decode(codes.transpose(0, 2, 1))
    assert wav.shape == (2, codes.shape[-1] * 1920) and np.isfinite(wav).all()
