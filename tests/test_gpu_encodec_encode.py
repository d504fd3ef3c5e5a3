"""CUDA Encodec encode (through the C ABI) against the float64 reference (tests/encodec_encoder_reference.py, itself pinned against
transformers' EncodecModel.encode in test_oracle_encodec_encode.py).

Latent z: max |diff| / max |ref| and relative L2 below 1e-3 (the codec contract; the fp32 CUDA-core path measures ~1e-6).
Codes: bit-exact against the ordered-fp32 code search run on the device's own z; against the float64 end-to-end reference a
frame's first differing level must be a float64 near-tie (its finer levels then search a different residual and are exempt)."""
import numpy as np
import pytest
import torch

import encodec_encoder_reference as eer
from conftest import GOLDEN, max_rel_to_peak, rel_err
from oracle import encodec as oe

pytestmark = pytest.mark.gpu
TOL = 1e-3
TIE_REL = 1e-3     # float64 distance gap, relative to |residual|^2 + 1, below which a level's search counts as a near-tie
SMALL = dict(num_filters=8, hidden_size=16, codebook_dim=16, codebook_size=64)


def make(b2a, cfg, W):
    return b2a.Encodec(b2a.EncodecConfig(**cfg.__dict__), weights=W)


def weights(cfg, n_codebooks, seed=7):
    return {**oe.init_weights(cfg, seed, n_codebooks=n_codebooks), **eer.init_encoder_weights(cfg, seed + 1)}


def device_latent(b2a, m, x):
    """z [n_chunks, B, frames, hidden] of the device encoder (before the code search)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    nc, T = m.encoded_shape(x.shape[1])
    z = np.empty((nc, x.shape[0], T, m.config.hidden_size), dtype=np.float32)
    b2a._ffi.check(b2a._ffi.lib().b2a_encodec_encode_latent_test(m._h, b2a._ffi.ptr(x), x.shape[0], x.shape[1], b2a._ffi.ptr(z)))
    return z


def fp32_codes(W, z, n_q):
    """The ordered-fp32 search on the device's own z [n_chunks, B, T, D] -> [n_chunks, B, n_q, T]."""
    return np.stack([eer.rvq_encode_fp32(W, zc, n_q) for zc in z])


def assert_codes_explained(W, dev, z64, n_q):
    """dev [B, n_q, T] vs the float64 search on the float64 z [B, T, D]: a frame's first differing level is a near-tie."""
    ref, gaps = eer.rvq_encode(W, z64, n_q, with_gaps=True)
    res = np.asarray(z64, dtype=np.float64)
    scale = np.empty_like(gaps)
    for q in range(n_q):
        scale[:, q] = (res ** 2).sum(-1) + 1.0
        res = res - W[f"quantizer.layers.{q}.codebook.embed"].astype(np.float64)[ref[:, q]]
    diff = dev != ref
    for b, t in zip(*np.nonzero(diff.any(1))):
        q = int(np.argmax(diff[b, :, t]))
        assert gaps[b, q, t] < TIE_REL * scale[b, q, t], (b, q, t, gaps[b, q, t])
    return float(diff.any(1).mean())


@pytest.fixture(scope="module")
def model24(b2a):
    cfg = oe.EncodecConfig()                              # the 24 kHz model: 32 filters, ratios 8,5,4,2, 2 x LSTM(512)
    W = weights(cfg, 8)
    return cfg, W, make(b2a, cfg, W)


@pytest.mark.parametrize("B,n", [(1, 320), (3, 24017), (2, 72000)])
def test_latent_and_codes_24khz_vs_float64(b2a, model24, B, n):
    cfg, W, m = model24
    x = eer.synth_clip(B, n, seed=n)
    if B > 1:
        x[1] *= 0.25
    z = device_latent(b2a, m, x)
    T = -(-n // 320)
    assert z.shape == (1, B, T, 128) and m.encoded_shape(n) == (1, T)
    z64 = eer.encoder(cfg, W, x)
    err_peak, err_l2 = max_rel_to_peak(z[0], z64), rel_err(z[0], z64)
    print(f"z error B={B} n={n}: max/peak {err_peak:.2e}, rel L2 {err_l2:.2e}")
    assert err_peak < TOL and err_l2 < TOL
    codes, scales = m.encode(x, bandwidth=6.0)
    assert codes.shape == (1, B, 8, T) and scales == [None]
    assert np.array_equal(codes, fp32_codes(W, z, 8))
    assert_codes_explained(W, codes[0], z64, 8)
    # golden fixture geometry
    if (B, n) == (3, 24017):
        assert np.array_equal(m.encode(x, bandwidth=6.0)[0], codes)                  # repeated call is identical


def test_golden(b2a):
    import sys
    sys.path.insert(0, str(GOLDEN))
    import make_golden_encodec_encode as mg
    g = np.load(GOLDEN / "encodec_encode.npz")
    cfg, W = mg.weights()
    m = make(b2a, cfg, W)
    x = eer.synth_clip(mg.BATCH, mg.N_SAMPLES, mg.CLIP_SEED)
    z = device_latent(b2a, m, x)
    assert z.shape == tuple(g["z_shape"])
    peak = max(abs(g["z_stats"][2]), abs(g["z_stats"][3]))
    assert np.abs(z.reshape(-1)[:16] - g["z_first"]).max() < TOL * peak
    codes = m.encode(x, bandwidth=mg.BANDWIDTH)[0]
    assert codes.shape == g["codes"].shape
    assert (codes != g["codes"]).mean() < 0.05          # float64 near-ties may flip a code (checked exactly above)


def test_batched_equals_serial_and_device_entry(b2a, model24):
    cfg, W, m = model24
    x = eer.synth_clip(3, 8000, seed=11)
    x[2] *= 3.0
    codes, _ = m.encode(x, bandwidth=6.0)
    for b in range(3):
        assert np.array_equal(m.encode(x[b:b + 1], bandwidth=6.0)[0], codes[:, b:b + 1])
    d_x = torch.from_numpy(x).cuda()
    d_codes = torch.empty(codes.shape, dtype=torch.int32, device="cuda")
    m.encode_dev(d_x, d_codes, bandwidth=6.0)
    torch.cuda.synchronize()
    assert np.array_equal(d_codes.cpu().numpy(), codes)
    s = torch.cuda.Stream()
    d2 = torch.zeros_like(d_codes)
    m.encode_dev(d_x, d2, stream=s.cuda_stream, bandwidth=6.0)
    s.synchronize()
    assert torch.equal(d2, d_codes)


@pytest.mark.parametrize("kw", [dict(use_causal_conv=False), dict(pad_mode="constant"), dict(use_conv_shortcut=False),
                                dict(num_lstm_layers=1), dict(num_lstm_layers=0), dict(audio_channels=2),
                                dict(upsampling_ratios=[3, 2], compress=1), dict(normalize=True)])
def test_config_variants(b2a, kw):
    cfg = oe.EncodecConfig(**SMALL, **kw)
    W = weights(cfg, 6, seed=5)
    m = make(b2a, cfg, W)
    n = 3001
    x = eer.synth_clip(2, n, seed=4, channels=cfg.audio_channels)
    x[1] *= 0.2
    z = device_latent(b2a, m, x)
    codes64, scales64, z64 = eer.encode(cfg, W, x, bandwidth=3.0, return_latent=True)
    assert z.shape == z64.shape
    assert max_rel_to_peak(z, z64) < TOL and rel_err(z, z64) < TOL, max_rel_to_peak(z, z64)
    codes, scales = m.encode(x, bandwidth=3.0)
    assert codes.shape == codes64.shape
    assert np.array_equal(codes, fp32_codes(W, z, codes.shape[2]))
    assert_codes_explained(W, codes[0], z64[0], codes.shape[2])
    if cfg.normalize:
        assert np.abs(scales[0] - scales64[0]).max() < 1e-6 * scales64[0].max()
    else:
        assert scales == [None]


def test_chunked_encode_with_overlap_and_normalize(b2a):
    cfg = oe.EncodecConfig(chunk_length_s=0.04, overlap=0.5, normalize=True, **SMALL)
    W = weights(cfg, 4, seed=9)
    m = make(b2a, cfg, W)
    x = eer.synth_clip(2, 1920, seed=8)
    x[1, 1000:] *= 0.05                                    # chunks of different loudness
    assert m.encoded_shape(1920) == (3, 3)
    codes, scales = m.encode(x, bandwidth=1.5)
    codes64, scales64, z64 = eer.encode(cfg, W, x, bandwidth=1.5, return_latent=True)
    z = device_latent(b2a, m, x)
    assert codes.shape == codes64.shape == (3, 2, 3, 3)      # 1.5 kbps of 64-entry books: 3 codebooks
    assert max_rel_to_peak(z, z64) < TOL
    assert np.array_equal(codes, fp32_codes(W, z, 3))
    for c in range(3):
        assert np.abs(scales[c] - scales64[c]).max() < 1e-6 * scales64[c].max()
        assert_codes_explained(W, codes[c], z64[c], 3)
    # the padding mask multiplies the audio ahead of the normalisation
    mask = np.ones((2, 1920), bool); mask[0, 1500:] = False
    cm, sm = m.encode(x, padding_mask=mask, bandwidth=1.5)
    xm = x * mask[..., None]
    assert np.array_equal(cm, m.encode(xm, bandwidth=1.5)[0])
    with pytest.raises(b2a.AudioGenerationError) as e:       # ragged: the last chunk would be shorter
        m.encode(eer.synth_clip(1, 2000, seed=1), bandwidth=1.5)
    assert e.value.case == "invalidInput"


def test_reconstruct_round_trip(b2a, model24):
    cfg, W, m = model24
    x = eer.synth_clip(2, 6400, seed=3)
    enc = m.encode_audio(x)
    assert enc.codes.shape == (1, 2, 2, 20)                # default bandwidth 1.5 kbps: 2 codebooks
    y = m.reconstruct(x)
    ref = oe.decode(cfg, W, enc.codes, enc.scales)
    assert y.shape == ref.shape == (2, 6400, 1)
    assert max_rel_to_peak(y, ref) < TOL and rel_err(y, ref) < TOL


def test_full_size_8x30s_at_24kbps_and_causal_prefix(b2a):
    cfg = oe.EncodecConfig()
    W = b2a.Encodec.random_init_weights(b2a.EncodecConfig(), seed=3, n_codebooks=32, encoder=True)
    m = make(b2a, cfg, W)
    n = 24000 * 30
    x = eer.synth_clip(8, n, seed=1)
    z = device_latent(b2a, m, x)
    assert z.shape == (1, 8, 2250, 128) and np.isfinite(z).all()
    codes, _ = m.encode(x, bandwidth=24.0)
    assert codes.shape == (1, 8, 32, 2250) and codes.min() >= 0 and codes.max() < 1024
    # causal convs + LSTM, and 750*320 samples need no right padding anywhere: the prefix encodes to the first 750 frames
    p = 750 * 320
    zp = device_latent(b2a, m, np.ascontiguousarray(x[:, :p]))
    assert np.array_equal(zp[:, :, :750], z[:, :, :750])
    assert np.array_equal(m.encode(np.ascontiguousarray(x[:, :p]), bandwidth=24.0)[0], codes[..., :750])


def test_errors(b2a):
    cfg = oe.EncodecConfig(**SMALL)
    W = weights(cfg, 2, seed=3)
    E = b2a.AudioGenerationError
    x = eer.synth_clip(1, 640, seed=0)
    Wdec = oe.init_weights(cfg, 3, n_codebooks=2)
    dec_only = make(b2a, cfg, Wdec)
    with pytest.raises(E) as e:
        dec_only.encode(x)
    assert e.value.case == "modelNotInitialized"
    codes = np.random.default_rng(0).integers(0, 64, size=(1, 1, 2, 4))
    assert max_rel_to_peak(dec_only.decode(codes), oe.decode(cfg, Wdec, codes)) < TOL
    # a malformed encoder tensor leaves the decoder usable
    W2 = dict(W); W2["encoder.layers.3.conv.weight"] = W2["encoder.layers.3.conv.weight"][:1]
    bad = make(b2a, cfg, W2)
    with pytest.raises(E) as e:
        bad.encode(x)
    assert e.value.case == "modelNotInitialized"
    assert np.array_equal(bad.decode(codes), make(b2a, cfg, W).decode(codes))
    m = make(b2a, cfg, W)
    lib, ptr = b2a._ffi.lib(), b2a._ffi.ptr
    out = np.empty((1, 1, 8, 2), np.int32)
    for nq in (0, 3):                                    # n_q < 1, more than the 2 codebooks held
        assert lib.b2a_encodec_encode(m._h, ptr(x), 1, 640, nq, ptr(out), None) == b2a._ffi.ERR_INVALID_INPUT
    for bad_x in (eer.synth_clip(1, 640, channels=2), np.zeros((1, 0, 1), np.float32)):   # channel mismatch, empty input
        with pytest.raises(E) as e:
            m.encode(bad_x)
        assert e.value.case == "invalidInput"
    with pytest.raises(E) as e:
        m.encode(x, bandwidth=2.0)                       # not one of target_bandwidths
    assert e.value.case == "invalidInput"
    d_x = torch.from_numpy(x).cuda()
    nc, T = m.encoded_shape(640)
    for d_codes in (torch.empty((nc, 1, 2, T), dtype=torch.int64, device="cuda"), torch.empty((nc, 1, 2, T + 1), dtype=torch.int32, device="cuda"),
                    torch.empty((nc, 1, 2, T), dtype=torch.int32)):
        with pytest.raises(E) as e:
            m.encode_dev(d_x, d_codes)
        assert e.value.case == "invalidInput"
    with pytest.raises(E) as e:
        m.encode_dev(d_x.double(), torch.empty((nc, 1, 2, T), dtype=torch.int32, device="cuda"))
    assert e.value.case == "invalidInput"
