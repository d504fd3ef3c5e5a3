"""CUDA SNAC for the 32 / 44 kHz models (LocalMHA, odd strides, a zero-padded decoder width) through the C ABI against the float64
reference (tests/snac_attention_reference.py) and its golden.  Waveforms and latents: max |diff| / max |ref| below 1e-3 (the
project's fp32 contract; the observed errors are in DESIGN.md 3.2c).  Codes as tests/test_gpu_snac_encode.py checks them."""
import json

import numpy as np
import pytest
import torch

import snac_attention_reference as sar
import snac_encoder_reference as ser
from conftest import GOLDEN, max_rel_to_peak, rel_err
from oracle import snac as osnac
from test_gpu_snac_encode import assert_codes_explained, search_gaps

pytestmark = pytest.mark.gpu
TOL = 1e-3


def make(b2a, cfg, W, **kw):
    return b2a.SNAC(cfg.sampling_rate, cfg.encoder_dim, cfg.encoder_rates, cfg.latent_dim, cfg.decoder_dim, cfg.decoder_rates,
                    cfg.attn_window_size, cfg.codebook_size, cfg.codebook_dim, cfg.vq_strides, cfg.noise, cfg.depthwise,
                    weights=W, **kw)


@pytest.fixture(scope="module")
def small(b2a):
    cfg = sar.small()
    W = sar.init_weights(cfg, 11)
    return cfg, W, make(b2a, cfg, W)


@pytest.fixture(scope="module")
def published(b2a):
    cfg = sar.published(44100)
    W = sar.init_weights(cfg, 5, encoder=False)
    return cfg, W, make(b2a, cfg, W)


def noise_for(cfg, B, T, seed):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal(s).astype(np.float32) for s in sar.noise_shapes(cfg, B, T)]


def device_latent(b2a, m, cfg, audio):
    a = np.ascontiguousarray(audio[:, 0], dtype=np.float32)
    B, n = a.shape
    z = np.empty((B, cfg.latent, m.encoded_length(n)), dtype=np.float32)
    b2a._ffi.check(b2a._ffi.lib().b2a_snac_encode_latent_test(m._h, b2a._ffi.ptr(a), B, n, b2a._ffi.ptr(z)))
    return z


# ---------------------------------------------------------------------------------------------------------- LocalMHA window core
def attn_core_ref(qkv, inv, B, T, dim, window):
    """float64 restatement of local_attn_kernel: rotary on q and k, softmax(q k^T / 8) v per (clip, window, head)."""
    x = torch.as_tensor(qkv, dtype=torch.float64).reshape(B, T // window, window, 3, dim // 64, 64)
    q, k, v = (x[:, :, :, i].permute(0, 3, 1, 2, 4) for i in range(3))          # [B, H, W, n, 64]
    f = torch.arange(window, dtype=torch.float64)[:, None] * torch.as_tensor(inv, dtype=torch.float64)[None]
    f = torch.cat([f, f], -1)
    q, k = (t * f.cos() + sar.rotate_half(t) * f.sin() for t in (q, k))
    o = torch.softmax(q @ k.transpose(-1, -2) / 8.0, -1) @ v
    return o.permute(0, 2, 3, 1, 4).reshape(B * T, dim).numpy()


@pytest.mark.parametrize("heads,window,B,T,scale", [(16, 32, 2, 96, 1.0), (24, 32, 3, 64, 1.0), (16, 24, 2, 72, 1.0),
                                                    (24, 16, 1, 80, 1.0), (16, 32, 2, 64, 12.0), (24, 64, 1, 128, 1.0)])
def test_local_attn_kernel_vs_float64(b2a, heads, window, B, T, scale):
    dim = heads * 64
    rng = np.random.default_rng(heads * 100 + window)
    qkv = (rng.standard_normal((B * T, 3 * dim)) * scale).astype(np.float32)
    inv = (1.0 / 10000.0 ** (np.arange(0, 64, 2) / 64.0)).astype(np.float32)
    out = np.empty((B * T, dim), dtype=np.float32)
    b2a._ffi.check(b2a._ffi.lib().b2a_snac_local_attn_test(b2a._ffi.ptr(qkv), b2a._ffi.ptr(inv), B, T, dim, window, b2a._ffi.ptr(out)))
    ref = attn_core_ref(qkv, inv, B, T, dim, window)
    assert max_rel_to_peak(out, ref) < TOL, max_rel_to_peak(out, ref)


# ---------------------------------------------------------------------------------------------------------- decode
def test_decode_published_geometry_vs_float64(published):
    cfg, W, m = published
    T = 64                                                           # two windows
    codes = osnac.synth_codes(cfg, 1, T, seed=4)
    noise = noise_for(cfg, 1, T, 6)
    y = m.decode(codes, noise=noise)
    ref = sar.decode(cfg, W, codes, noise)
    assert y.shape == ref.shape == (1, 1, 384 * T - 2)
    assert max_rel_to_peak(y, ref) < TOL, max_rel_to_peak(y, ref)


def test_decode_small_geometry_vs_float64(small):
    cfg, W, m = small
    for B, T in ((1, 16), (3, 48)):
        codes = osnac.synth_codes(cfg, B, T, seed=T)
        noise = noise_for(cfg, B, T, B)
        y = m.decode(codes, noise=noise)
        ref = sar.decode(cfg, W, codes, noise)
        assert y.shape == ref.shape
        assert max_rel_to_peak(y, ref) < TOL and rel_err(y, ref) < TOL, (max_rel_to_peak(y, ref), rel_err(y, ref))


def test_decoded_length_matches_reference(small, published):
    for cfg, _, m in (small, published):
        for T in (32, 64, 128):
            assert m.decoded_length(T) == sar.stage_lengths(cfg, T)[-1]
    assert published[2].decoded_length(32) == 384 * 32 - 2


def test_decode_batched_serial_device_bit_exact(small):
    cfg, W, m = small
    B, T = 4, 32
    codes = osnac.synth_codes(cfg, B, T, seed=9)
    full = m.decode(codes, zero_noise=True)
    for b in range(B):
        one = m.decode([c[b:b + 1] for c in codes], zero_noise=True)
        assert np.array_equal(full[b:b + 1], one)
    seeded = m.decode(codes, seed=7)
    d_codes = [torch.from_numpy(c).cuda() for c in codes]
    d_wave = torch.empty((B, 1, m.decoded_length(T)), dtype=torch.float32, device="cuda")
    m.decode_dev(d_codes, d_wave, seed=7, stream=m.stream)
    torch.cuda.synchronize()
    assert np.array_equal(seeded, d_wave.cpu().numpy())


def test_golden(b2a, small):
    cfg, W, m = small
    import importlib.util
    spec = importlib.util.spec_from_file_location("mg44", GOLDEN / "make_golden_snac_44khz.py")
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
    g = np.load(GOLDEN / "snac_44khz.npz")
    _, _, codes, noise, audio = mg.inputs()
    y = m.decode(codes, noise=noise)
    assert tuple(g["y_shape"]) == y.shape
    peak = max(abs(g["y_stats"][2]), abs(g["y_stats"][3]))
    assert np.abs(y.reshape(-1)[:16] - g["y_first"]).max() < TOL * peak
    ys = np.array([y.mean(), np.abs(y).mean(), y.min(), y.max()])
    assert np.abs(ys - g["y_stats"]).max() < TOL * peak
    z = device_latent(b2a, m, cfg, audio)
    assert tuple(g["z_shape"]) == z.shape
    zpeak = max(abs(g["z_stats"][2]), abs(g["z_stats"][3]))
    assert np.abs(z.reshape(-1)[:16] - g["z_first"]).max() < TOL * zpeak
    ec = m.encode(audio)
    _, gaps = search_gaps(cfg, W, sar.encode_latent(cfg, W, audio))
    assert_codes_explained(cfg, ec, [g[f"codes{i}"] for i in range(len(cfg.vq_strides))], gaps)


# ---------------------------------------------------------------------------------------------------------- encode
@pytest.mark.parametrize("B,n", [(1, 192), (2, 1000), (3, 5000)])
def test_encode_vs_float64(b2a, small, B, n):
    cfg, W, m = small
    audio = ser.synth_clip(B, n, seed=n, sr=cfg.sampling_rate)
    z = device_latent(b2a, m, cfg, audio)
    zr = sar.encode_latent(cfg, W, audio)
    assert z.shape == zr.shape == (B, cfg.latent, m.encoded_length(n))
    assert max_rel_to_peak(z, zr) < TOL and rel_err(z, zr) < TOL, (max_rel_to_peak(z, zr), rel_err(z, zr))
    codes = m.encode(audio)
    _, from_z = osnac.quantize(cfg, W, z)
    assert all(np.array_equal(a, b) for a, b in zip(codes, from_z))
    ref, gaps = search_gaps(cfg, W, zr)
    assert_codes_explained(cfg, codes, ref, gaps)


def test_encode_batched_serial_device_and_round_trip(small):
    cfg, W, m = small
    n = 3000
    audio = ser.synth_clip(3, n, seed=2, sr=cfg.sampling_rate)
    full = m.encode(audio)
    for b in range(3):
        one = m.encode(audio[b:b + 1])
        assert all(np.array_equal(f[b:b + 1], o) for f, o in zip(full, one))
    T = m.encoded_length(n)
    assert T % cfg.attn_window_size == 0 and T * cfg.hop_length >= n
    d_codes = [torch.empty((3, T // s), dtype=torch.int32, device="cuda") for s in cfg.vq_strides]
    m.encode_dev(torch.from_numpy(audio).cuda(), d_codes, stream=m.stream)
    torch.cuda.synchronize()
    assert all(np.array_equal(h, d.cpu().numpy()) for h, d in zip(full, d_codes))
    y = m.decode(full)
    assert y.shape == (3, 1, m.decoded_length(T)) and np.isfinite(y).all()


def test_published_encode_length(b2a):
    cfg = sar.published(32000)
    W = b2a.SNAC.random_init_weights(3, latent=1024, decoder_dim=1536, decoder_rates=cfg.decoder_rates, vq_strides=cfg.vq_strides,
                                     encoder=True, encoder_dim=64, encoder_rates=cfg.encoder_rates, attn_window_size=32)
    m = make(b2a, cfg, W)
    assert m.encoded_length(1) == 32 and m.encoded_length(12288) == 32 and m.encoded_length(12289) == 64
    codes = m.encode(ser.synth_clip(1, 20000, seed=1, sr=32000))
    assert [c.shape for c in codes] == [(1, 64 // s) for s in cfg.vq_strides]


# ---------------------------------------------------------------------------------------------------------- loading and errors
def test_from_model_directory(b2a, small, tmp_path):
    from safetensors.numpy import save_file
    cfg, W, m = small
    d = tmp_path / "snac_small"
    d.mkdir()
    (d / "config.json").write_text(json.dumps(dict(
        sampling_rate=cfg.sampling_rate, encoder_dim=cfg.encoder_dim, encoder_rates=list(cfg.encoder_rates), latent_dim=None,
        decoder_dim=cfg.decoder_dim, decoder_rates=list(cfg.decoder_rates), attn_window_size=cfg.attn_window_size,
        codebook_size=cfg.codebook_size, codebook_dim=cfg.codebook_dim, vq_strides=list(cfg.vq_strides), noise=True, depthwise=True)))
    save_file({k: np.ascontiguousarray(v) for k, v in W.items()}, str(d / "model.safetensors"))
    m2 = b2a.SNAC.from_model_directory(d)
    codes = osnac.synth_codes(cfg, 2, 32, seed=1)
    assert np.array_equal(m2.decode(codes, zero_noise=True), m.decode(codes, zero_noise=True))
    audio = ser.synth_clip(1, 800, seed=1, sr=cfg.sampling_rate)
    assert all(np.array_equal(a, b) for a, b in zip(m2.encode(audio), m.encode(audio)))


def expect(b2a, code, fn):
    with pytest.raises(b2a.AudioGenerationError) as e:
        fn()
    assert e.value.code == code, e.value


def test_errors(b2a, small, monkeypatch):
    cfg, W, m = small
    ffi = b2a._ffi
    bad_heads = sar.SNACConfig(**{**cfg.__dict__, "decoder_dim": 352})
    expect(b2a, ffi.ERR_INVALID_INPUT, lambda: make(b2a, bad_heads, W))
    bad_win = sar.SNACConfig(**{**cfg.__dict__, "attn_window_size": 80})
    expect(b2a, ffi.ERR_INVALID_INPUT, lambda: make(b2a, bad_win, W))
    codes = osnac.synth_codes(cfg, 1, 24, seed=1)                     # 24 % 16 != 0
    expect(b2a, ffi.ERR_INVALID_INPUT, lambda: m.decode(codes))
    dec_missing = {k: v for k, v in W.items() if k != "decoder.model.layers.2.to_out.weight"}
    with pytest.raises(b2a.AudioGenerationError) as e:
        make(b2a, cfg, dec_missing)
    assert e.value.code == ffi.ERR_MODEL_NOT_INITIALIZED and "decoder.model.layers.2.to_out.weight" in e.value.message
    n = len(cfg.encoder_rates)
    enc_missing = {k: v for k, v in W.items() if k != f"encoder.block.layers.{n + 1}.rel_pos.inv_freq"}
    m3 = make(b2a, cfg, enc_missing)                                   # the decoder still works
    good = osnac.synth_codes(cfg, 1, 32, seed=1)
    assert np.array_equal(m3.decode(good, zero_noise=True), m.decode(good, zero_noise=True))
    with pytest.raises(b2a.AudioGenerationError) as e:
        m3.encode(ser.synth_clip(1, 500, seed=1))
    assert e.value.code == ffi.ERR_MODEL_NOT_INITIALIZED and "rel_pos.inv_freq" in e.value.message
    monkeypatch.setenv("B2A_SNAC", "simt")
    expect(b2a, ffi.ERR_INVALID_INPUT, lambda: make(b2a, cfg, W))


# ---------------------------------------------------------------------------------------------------------- full size
def test_full_size_8x30s_44khz(b2a):
    """8 x 30 s of 44.1 kHz audio at the published geometry: its 2-tap operands pass 2^31 elements, so the batch runs in slices of
    clips.  Finite, of the right lengths, and one clip of the batch equals its serial result."""
    cfg = sar.published(44100)
    W = b2a.SNAC.random_init_weights(1234, latent=1024, decoder_dim=1536, decoder_rates=cfg.decoder_rates, vq_strides=cfg.vq_strides,
                                     encoder=True, encoder_dim=64, encoder_rates=cfg.encoder_rates, attn_window_size=32)
    m = make(b2a, cfg, W)
    n = 30 * 44100
    audio = ser.synth_clip(8, n, seed=1, sr=44100)
    codes = m.encode(audio)
    T = m.encoded_length(n)
    assert T == 3456 and [c.shape for c in codes] == [(8, T // s) for s in cfg.vq_strides]
    one = m.encode(audio[6:7])
    assert all(np.array_equal(c[6:7], o) for c, o in zip(codes, one))
    y = m.decode(codes, zero_noise=True)
    assert y.shape == (8, 1, 384 * T - 2) and np.isfinite(y).all()
    y6 = m.decode([c[6:7] for c in codes], zero_noise=True)
    assert np.array_equal(y[6:7], y6)
