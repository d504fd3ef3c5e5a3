"""The float64 time_group_norm reference (tests/encodec_gn_reference.py) against transformers' EncodecModel with
norm_type="time_group_norm" (the 48 kHz model's layer semantics, random init with randomised norm affines, float64), the closed
form of the transposed conv's norm over the trimmed samples, and the 48 kHz golden.  CPU only."""
import numpy as np
import pytest
import torch

import encodec_encoder_reference as eer
import encodec_gn_reference as gnr
from conftest import GOLDEN
from oracle import encodec as oe


def hf_to_mlx(m) -> dict:
    """transformers EncodecModel (time_group_norm) -> checkpoint keys in MLX layouts: Conv1d [out,in,k] -> [out,k,in],
    ConvTranspose1d [in,out,k] -> [out,k,in], GroupNorm weight / bias as norm.weight / norm.bias, LSTM weight_ih/hh -> Wx/Wh."""
    W = {}
    for q, layer in enumerate(m.quantizer.layers):
        W[f"quantizer.layers.{q}.codebook.embed"] = layer.codebook.embed.detach().numpy().astype(np.float32)

    def conv(pre, mod, transposed=False):
        w = mod.conv.weight.detach()
        w = w.permute(1, 2, 0) if transposed else w.permute(0, 2, 1)
        W[pre + "conv.weight"] = w.contiguous().numpy().astype(np.float32)
        W[pre + "conv.bias"] = mod.conv.bias.detach().numpy().astype(np.float32)
        W[pre + "norm.weight"] = mod.norm.weight.detach().numpy().astype(np.float32)
        W[pre + "norm.bias"] = mod.norm.bias.detach().numpy().astype(np.float32)

    for side in ("encoder", "decoder"):
        for i, layer in enumerate(getattr(m, side).layers):
            pre = f"{side}.layers.{i}."
            name = type(layer).__name__
            if name in ("EncodecConv1d", "EncodecConvTranspose1d"):
                conv(pre, layer, transposed=name == "EncodecConvTranspose1d")
            elif name == "EncodecLSTM":
                for l in range(layer.lstm.num_layers):
                    W[pre + f"lstm.{l}.Wx"] = getattr(layer.lstm, f"weight_ih_l{l}").detach().numpy().astype(np.float32)
                    W[pre + f"lstm.{l}.Wh"] = getattr(layer.lstm, f"weight_hh_l{l}").detach().numpy().astype(np.float32)
                    W[pre + f"lstm.{l}.bias"] = (getattr(layer.lstm, f"bias_ih_l{l}") + getattr(layer.lstm, f"bias_hh_l{l}")).detach().numpy().astype(np.float32)
            elif name == "EncodecResnetBlock":
                for bi, sub in enumerate(layer.block):
                    if type(sub).__name__ == "EncodecConv1d":
                        conv(pre + f"block.{bi}.", sub)
                if type(layer.shortcut).__name__ == "EncodecConv1d":
                    conv(pre + "shortcut.", layer.shortcut)
    return W


def hf_model(**kw):
    from transformers import EncodecConfig as HC, EncodecModel
    torch.manual_seed(0)
    m = EncodecModel(HC(norm_type="time_group_norm", audio_channels=2, use_causal_conv=False, sampling_rate=48000,
                        target_bandwidths=[3.0, 6.0, 12.0, 24.0], **kw)).eval()
    with torch.no_grad():
        for layer in m.quantizer.layers:                   # codebooks are zero-initialised buffers
            layer.codebook.embed.normal_()
        for mod in m.modules():                            # GroupNorm starts at gamma 1, beta 0: draw them away from that
            if isinstance(mod, torch.nn.GroupNorm):
                mod.weight.uniform_(0.5, 1.5).mul_(torch.where(torch.rand_like(mod.weight) < 0.5, -1.0, 1.0))
                mod.bias.uniform_(0.1, 0.5).mul_(torch.where(torch.rand_like(mod.bias) < 0.5, -1.0, 1.0))
    return m.double()


@pytest.mark.parametrize("kw", [dict(), dict(use_conv_shortcut=False)])
def test_decoder_matches_transformers(kw):
    m = hf_model(**kw)
    W = hf_to_mlx(m)
    cfg = gnr.config_48khz(chunk_length_s=None, overlap=None, **kw)
    codes = np.random.default_rng(0).integers(0, 1024, size=(2, 8, 23))     # T = 23: longer than every reflect pad
    with torch.no_grad():
        emb = m.quantizer.decode(torch.from_numpy(codes).transpose(0, 1))
        ref = m.decoder(emb).numpy().transpose(0, 2, 1)                        # [B, T*320, 2]
    y = gnr.decode(cfg, W, codes[None])
    assert y.shape == ref.shape == (2, 23 * 320, 2)
    err = np.abs(y - ref).max() / np.abs(ref).max()
    assert err < 1e-5, err                                                      # fp32-rounded weights vs HF's own


@pytest.mark.parametrize("kw", [dict(), dict(use_conv_shortcut=False)])
def test_encoder_matches_transformers(kw):
    m = hf_model(**kw)
    W = hf_to_mlx(m)
    cfg = gnr.config_48khz(chunk_length_s=None, overlap=None, normalize=False, **kw)
    x = eer.synth_clip(2, 4817, seed=5, channels=2)
    x[1] *= 0.3
    with torch.no_grad():
        z_hf = m.encoder(torch.from_numpy(x.astype(np.float64)).permute(0, 2, 1)).permute(0, 2, 1).numpy()
    z = gnr.encoder(cfg, W, x)
    assert z.shape == z_hf.shape == (2, 16, 128)
    assert np.abs(z - z_hf).max() / np.abs(z_hf).max() < 1e-5
    codes, scales, z2 = gnr.encode(cfg, W, x, bandwidth=6.0)
    with torch.no_grad():
        hf_codes = m.quantizer.encode(torch.from_numpy(z_hf).permute(0, 2, 1), bandwidth=6.0).transpose(0, 1).numpy()
    assert codes.shape == (1, 2, 4, 16)                                        # 6 kbps at 150 frames/s: 4 codebooks
    assert np.array_equal(codes[0], hf_codes) and scales == [None]


@pytest.mark.parametrize("causal", [True, False])
def test_transposed_conv_norm_covers_the_trimmed_samples(causal):
    """Closed form: a constant input through a k = 2s transposed conv of ones gives s samples of 1, (L - 1) s of 2 and s of 1
    ((L + 1) s in all).  The norm takes mean 2L / (L + 1) and E[y^2] = (4L - 2) / (L + 1) over all of them, the trimmed ones
    included; statistics of the kept samples alone would differ."""
    cfg = oe.EncodecConfig(use_causal_conv=causal)
    s, L = 4, 5
    k = 2 * s
    W = {"p.conv.weight": np.ones((1, k, 1), np.float32), "p.conv.bias": np.zeros(1, np.float32),
         "p.norm.weight": np.array([1.5], np.float32), "p.norm.bias": np.array([0.25], np.float32)}
    out = gnr.conv_transpose1d(cfg, W, "p.", np.ones((1, L, 1)), s)
    pr = s if causal else s // 2                     # trim_right_ratio 1: ceil((k - s) * 1) causal, (k - s) // 2 otherwise
    pl = s - pr
    y = np.array([1.0] * s + [2.0] * ((L - 1) * s) + [1.0] * s)
    kept = y[pl:len(y) - pr]
    assert out.shape == (1, L * s, 1) and len(kept) == L * s
    mu = 2 * L / (L + 1)
    var = (4 * L - 2) / (L + 1) - mu ** 2
    assert np.allclose(out[0, :, 0], (kept - mu) / np.sqrt(var + gnr.EPS) * 1.5 + 0.25, rtol=0, atol=1e-12)
    own = (kept - kept.mean()) / np.sqrt(kept.var() + gnr.EPS) * 1.5 + 0.25
    assert np.abs(out[0, :, 0] - own).max() > 1e-2


def test_chunks_have_their_own_statistics():
    cfg = gnr.config_48khz(num_filters=8, hidden_size=16, codebook_dim=16, codebook_size=64, chunk_length_s=0.02,
                           num_lstm_layers=1)                             # 960-sample chunks, stride 950
    W = gnr.weights(cfg, 4, seed=3)
    n = cfg.chunk_stride * 2 + cfg.chunk_length
    x = eer.synth_clip(1, n, seed=2, channels=2)
    codes, scales, z = gnr.encode(cfg, W, x, bandwidth=3.0)
    assert codes.shape == (3, 1, 3, 3)
    x2 = x.copy()
    x2[:, cfg.chunk_length:2 * cfg.chunk_stride] *= -3.0                      # only chunk 1's exclusive span
    codes2, scales2, z2 = gnr.encode(cfg, W, x2, bandwidth=3.0)
    assert np.array_equal(z[0], z2[0]) and np.array_equal(z[2], z2[2]) and not np.array_equal(z[1], z2[1])
    assert np.array_equal(scales[0], scales2[0]) and np.array_equal(scales[2], scales2[2])
    assert np.array_equal(codes[0], codes2[0]) and np.array_equal(codes[2], codes2[2])


def test_golden_reproduces():
    import sys
    sys.path.insert(0, str(GOLDEN))
    import make_golden_encodec_48khz as mg
    g = np.load(GOLDEN / "encodec_48khz.npz")
    y, z, codes, scales = mg.compute()
    assert tuple(g["y_shape"]) == y.shape and tuple(g["z_shape"]) == z.shape
    assert np.abs(y[:, :64].reshape(-1) - g["y_first"]).max() < 1e-6 and np.abs(y[:, -64:].reshape(-1) - g["y_last"]).max() < 1e-6
    assert np.abs(mg.stats(y) - g["y_stats"]).max() < 1e-12
    assert np.abs(z.reshape(-1)[:16] - g["z_first"]).max() < 1e-6
    assert np.abs(mg.stats(z) - g["z_stats"]).max() < 1e-12
    assert np.array_equal(codes, g["codes"]) and np.allclose(scales, g["scales"], rtol=1e-12)
