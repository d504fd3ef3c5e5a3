"""CUDA Encodec with norm_type time_group_norm (the 48 kHz stereo model) through the C ABI against the float64 reference
(tests/encodec_gn_reference.py, itself pinned against transformers' EncodecModel in test_oracle_encodec_48khz.py).

Decode and latent z: max |diff| / max |ref| below 1e-3 (the codec contract).  Codes: bit-exact against the ordered-fp32 code
search run on the device's own z; against the float64 search a frame's first differing level must be a float64 near-tie.
The group norm's statistics cover a whole chunk, so nothing is causal; what holds instead is that chunks are independent."""
import json

import numpy as np
import pytest
import torch

import encodec_encoder_reference as eer
import encodec_gn_reference as gnr
from conftest import GOLDEN, max_rel_to_peak, rel_err
from test_gpu_encodec_encode import assert_codes_explained, device_latent, fp32_codes

pytestmark = pytest.mark.gpu
TOL = 1e-3
SMALL = dict(num_filters=8, hidden_size=16, codebook_dim=16, codebook_size=64)
CHUNK, STRIDE = 48000, 47520          # 1 s chunks, overlap 0.01


def make(b2a, cfg, W):
    return b2a.Encodec(b2a.EncodecConfig(**cfg.__dict__), weights=W)


def clip(B, n, seed, channels=2):
    x = eer.synth_clip(B, n, seed=seed, channels=channels, sr=48000)
    if B > 1:
        x[1] *= 0.25
    return x


@pytest.fixture(scope="module")
def model48(b2a):
    cfg = gnr.config_48khz()              # 32 filters, ratios 8,5,4,2, 2 x LSTM(512), stereo, non-causal reflect, normalize
    W = gnr.weights(cfg, 16, seed=7)
    return cfg, W, make(b2a, cfg, W)


@pytest.mark.parametrize("n_chunks,B", [(1, 2), (3, 1)])
def test_decode_vs_float64(model48, n_chunks, B):
    cfg, W, m = model48
    rng = np.random.default_rng(n_chunks)
    codes = rng.integers(0, 1024, size=(n_chunks, B, 16, 150)).astype(np.int32)
    scales = [rng.uniform(0.2, 3.0, size=B).astype(np.float32) for _ in range(n_chunks)]
    y, ref = m.decode(codes, scales), gnr.decode(cfg, W, codes, scales)
    assert y.shape == ref.shape == (B, STRIDE * (n_chunks - 1) + CHUNK, 2)
    err = max_rel_to_peak(y, ref)
    print(f"decode {n_chunks} chunk(s) x B={B}: max/peak {err:.2e}, rel L2 {rel_err(y, ref):.2e}")
    assert err < TOL and rel_err(y, ref) < TOL
    # fewer codebooks, no scales
    y2, ref2 = m.decode(codes[:, :, :4]), gnr.decode(cfg, W, codes[:, :, :4])
    assert max_rel_to_peak(y2, ref2) < TOL


def test_encode_latent_and_codes_vs_float64(b2a, model48):
    cfg, W, m = model48
    n = STRIDE + CHUNK
    x = clip(2, n, seed=11)
    assert m.encoded_shape(n) == (2, 150)
    z = device_latent(b2a, m, x)
    codes64, scales64, z64 = gnr.encode(cfg, W, x, bandwidth=24.0)
    assert z.shape == z64.shape == (2, 2, 150, 128)
    err_peak, err_l2 = max_rel_to_peak(z, z64), rel_err(z, z64)
    print(f"z error 2 chunks x B=2: max/peak {err_peak:.2e}, rel L2 {err_l2:.2e}")
    assert err_peak < TOL and err_l2 < TOL
    codes, scales = m.encode(x, bandwidth=24.0)
    assert codes.shape == codes64.shape == (2, 2, 16, 150)
    assert np.array_equal(codes, fp32_codes(W, z, 16))
    for c in range(2):
        assert np.abs(scales[c] - scales64[c]).max() < 1e-6 * scales64[c].max()
        print(f"chunk {c}: frames whose codes differ from the float64 search (near-ties): {assert_codes_explained(W, codes[c], z64[c], 16):.3f}")


def test_batched_equals_serial_and_device_entry(b2a, model48):
    cfg, W, m = model48
    n = STRIDE + CHUNK
    x = clip(3, n, seed=12)
    x[2] *= 3.0
    codes, scales = m.encode(x, bandwidth=6.0)
    z = device_latent(b2a, m, x)
    y = m.decode(codes, scales)
    for b in range(3):
        cb, sb = m.encode(x[b:b + 1], bandwidth=6.0)
        assert np.array_equal(cb, codes[:, b:b + 1])
        assert all(np.array_equal(s1, s2[b:b + 1]) for s1, s2 in zip(sb, scales))
        assert np.array_equal(device_latent(b2a, m, x[b:b + 1]), z[:, b:b + 1])
        assert np.array_equal(m.decode(cb, sb), y[b:b + 1])
    d_x = torch.from_numpy(x).cuda()
    d_codes = torch.empty(codes.shape, dtype=torch.int32, device="cuda")
    d_scales = torch.empty((codes.shape[0], 3), dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    m.encode_dev(d_x, d_codes, d_scales, stream=s.cuda_stream, bandwidth=6.0)
    s.synchronize()
    assert np.array_equal(d_codes.cpu().numpy(), codes) and np.array_equal(d_scales.cpu().numpy(), np.stack(scales))
    d_wave = torch.empty(y.shape, dtype=torch.float32, device="cuda")
    m.decode_dev(d_codes, d_wave, d_scales, stream=s.cuda_stream)
    s.synchronize()
    assert np.array_equal(d_wave.cpu().numpy(), y)


def test_chunk_independence(b2a, model48):
    cfg, W, m = model48
    n = 2 * STRIDE + CHUNK
    x = clip(2, n, seed=13)
    codes, scales = m.encode(x, bandwidth=24.0)
    assert codes.shape == (3, 2, 16, 150)
    x2 = x.copy()
    x2[:, CHUNK:2 * STRIDE] = eer.synth_clip(2, 2 * STRIDE - CHUNK, seed=99, channels=2)     # chunk 1's exclusive span only
    codes2, scales2 = m.encode(x2, bandwidth=24.0)
    for c in (0, 2):
        assert np.array_equal(codes2[c], codes[c]) and np.array_equal(scales2[c], scales[c])
    assert not np.array_equal(codes2[1], codes[1])


@pytest.mark.parametrize("kw", [dict(use_causal_conv=True), dict(pad_mode="constant"), dict(use_conv_shortcut=False),
                                dict(audio_channels=1), dict(num_lstm_layers=0), dict(upsampling_ratios=[3, 2], compress=1)])
def test_config_variants(b2a, kw):
    cfg = gnr.config_48khz(**SMALL, **kw)
    W = gnr.weights(cfg, 6, seed=5)
    m = make(b2a, cfg, W)
    codes = np.random.default_rng(4).integers(0, 64, size=(1, 2, 3, 19)).astype(np.int32)
    y, ref = m.decode(codes, [np.array([0.5, 2.0], np.float32)]), gnr.decode(cfg, W, codes, [np.array([0.5, 2.0])])
    assert y.shape == ref.shape
    assert max_rel_to_peak(y, ref) < TOL, max_rel_to_peak(y, ref)
    x = clip(2, 3001, seed=4, channels=cfg.audio_channels)
    z = device_latent(b2a, m, x)
    codes64, scales64, z64 = gnr.encode(cfg, W, x, bandwidth=3.0)
    assert z.shape == z64.shape
    assert max_rel_to_peak(z, z64) < TOL and rel_err(z, z64) < TOL, max_rel_to_peak(z, z64)
    codes, scales = m.encode(x, bandwidth=3.0)
    assert codes.shape == codes64.shape
    assert np.array_equal(codes, fp32_codes(W, z, codes.shape[2]))
    assert_codes_explained(W, codes[0], z64[0], codes.shape[2])
    assert np.abs(scales[0] - scales64[0]).max() < 1e-6 * scales64[0].max()


def test_golden(b2a):
    import sys
    sys.path.insert(0, str(GOLDEN))
    import make_golden_encodec_48khz as mg
    g = np.load(GOLDEN / "encodec_48khz.npz")
    cfg, W = mg.weights()
    m = make(b2a, cfg, W)
    codes, scales = mg.decode_inputs()
    y = m.decode(codes, scales)
    assert y.shape == tuple(g["y_shape"])
    peak = max(abs(g["y_stats"][2]), abs(g["y_stats"][3]))
    assert np.abs(y[:, :64].reshape(-1) - g["y_first"]).max() < TOL * peak
    assert np.abs(y[:, -64:].reshape(-1) - g["y_last"]).max() < TOL * peak
    assert np.abs(mg.stats(y) - g["y_stats"]).max() < TOL * peak
    audio = eer.synth_clip(mg.BATCH, mg.N_SAMPLES, mg.CLIP_SEED, channels=2, sr=48000)
    audio[1] *= 0.3
    z = device_latent(b2a, m, audio)
    assert z.shape == tuple(g["z_shape"])
    zpeak = max(abs(g["z_stats"][2]), abs(g["z_stats"][3]))
    assert np.abs(z.reshape(-1)[:16] - g["z_first"]).max() < TOL * zpeak
    c, s = m.encode(audio, bandwidth=mg.BANDWIDTH)
    assert c.shape == g["codes"].shape
    assert (c != g["codes"]).mean() < 0.05              # float64 near-ties may flip a code (checked exactly above)
    assert np.abs(np.stack(s) - g["scales"]).max() < 1e-6 * g["scales"].max()


def test_full_size_8x30s_at_24kbps(b2a):
    base = gnr.config_48khz()
    W = b2a.Encodec.random_init_weights(b2a.EncodecConfig(**base.__dict__), seed=3, n_codebooks=16, encoder=True)
    assert "decoder.layers.0.norm.weight" in W and "encoder.layers.15.norm.bias" in W
    m = make(b2a, base, W)
    n = 30 * STRIDE + CHUNK                                # 1 473 600 samples: 31 full chunks, 30.7 s
    x = clip(8, n, seed=1)
    codes, scales = m.encode(x, bandwidth=24.0)
    assert codes.shape == (31, 8, 16, 150) and codes.min() >= 0 and codes.max() < 1024
    assert len(scales) == 31 and all(np.isfinite(s).all() and (s > 0).all() for s in scales)
    y = m.decode(codes, scales)
    assert y.shape == (8, n, 2) and np.isfinite(y).all()
    with pytest.raises(b2a.AudioGenerationError) as e:     # exactly 30 s: the last chunk would be ragged
        m.encode(np.zeros((1, 1440000, 2), np.float32), bandwidth=24.0)
    assert e.value.case == "invalidInput"


def test_errors(b2a):
    cfg = gnr.config_48khz(**SMALL)
    W = gnr.weights(cfg, 2, seed=3)
    E = b2a.AudioGenerationError
    with pytest.raises(E) as e:                            # norm_type other than weight_norm / time_group_norm -> 2
        make(b2a, gnr.config_48khz(**SMALL, norm_type="layer_norm"), W)
    assert e.value.case == "invalidInput"
    for key in ("decoder.layers.4.shortcut.norm.bias", "decoder.layers.15.norm.weight"):
        W2 = dict(W); W2.pop(key)
        with pytest.raises(E) as e:
            make(b2a, cfg, W2)
        assert e.value.case == "modelNotInitialized" and key in str(e.value)
    W2 = dict(W); W2.pop("encoder.layers.3.norm.weight")   # a missing encoder norm leaves the decoder usable
    bad = make(b2a, cfg, W2)
    with pytest.raises(E) as e:
        bad.encode(clip(1, 640, seed=0))
    assert e.value.case == "modelNotInitialized"
    m = make(b2a, cfg, W)
    for bw in (1.5, 2.0):                                   # not one of [3, 6, 12, 24]
        with pytest.raises(E) as e:
            m.encode(clip(1, 640, seed=0), bandwidth=bw)
        assert e.value.case == "invalidInput"


def test_from_model_directory(b2a, tmp_path):
    from safetensors.numpy import save_file
    cfg = gnr.config_48khz(**SMALL)
    W = gnr.weights(cfg, 4, seed=8)
    conf = dict(cfg.__dict__, model_type="encodec")
    (tmp_path / "config.json").write_text(json.dumps(conf))
    save_file({k: np.ascontiguousarray(v) for k, v in W.items()}, str(tmp_path / "model.safetensors"))
    a = b2a.Encodec.from_model_directory(tmp_path)
    assert a.config.norm_type == "time_group_norm" and a.channels == 2 and a.sampling_rate == 48000
    b = make(b2a, cfg, W)
    x = clip(2, 3001, seed=6)
    ca, sa = a.encode(x, bandwidth=3.0)                     # 64-entry books at 150 frames/s: 3 codebooks
    cb, sb = b.encode(x, bandwidth=3.0)
    assert ca.shape == (1, 2, 3, 10)
    assert np.array_equal(ca, cb) and all(np.array_equal(p, q) for p, q in zip(sa, sb))
    assert np.array_equal(a.decode(ca, sa), b.decode(cb, sb))
