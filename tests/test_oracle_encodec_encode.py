"""The float64 Encodec encode reference (tests/encodec_encoder_reference.py) against transformers' EncodecModel.encode (random
init, float64), its key layout against the HF module array, its chunk loop and bandwidth rule, the ordered-fp32 search
restatement, and its golden.  CPU only."""
import numpy as np
import pytest
import torch

import encodec_encoder_reference as eer
from conftest import GOLDEN
from oracle import encodec as oe


def hf_encoder_to_mlx(m) -> dict:
    """transformers EncodecModel -> encoder.* / quantizer.* keys in MLX layouts (Conv1d [out,in,k] -> [out,k,in]; LSTM
    weight_ih/hh -> Wx/Wh, bias_ih + bias_hh)."""
    W = {}
    for q, layer in enumerate(m.quantizer.layers):
        W[f"quantizer.layers.{q}.codebook.embed"] = layer.codebook.embed.detach().numpy().astype(np.float32)

    def conv(pre, mod):
        W[pre + "conv.weight"] = mod.conv.weight.detach().permute(0, 2, 1).contiguous().numpy().astype(np.float32)
        W[pre + "conv.bias"] = mod.conv.bias.detach().numpy().astype(np.float32)

    for i, layer in enumerate(m.encoder.layers):
        pre = f"encoder.layers.{i}."
        name = type(layer).__name__
        if name == "EncodecConv1d":
            conv(pre, layer)
        elif name == "EncodecLSTM":
            for l in range(layer.lstm.num_layers):
                W[pre + f"lstm.{l}.Wx"] = getattr(layer.lstm, f"weight_ih_l{l}").detach().numpy().astype(np.float32)
                W[pre + f"lstm.{l}.Wh"] = getattr(layer.lstm, f"weight_hh_l{l}").detach().numpy().astype(np.float32)
                W[pre + f"lstm.{l}.bias"] = (getattr(layer.lstm, f"bias_ih_l{l}") + getattr(layer.lstm, f"bias_hh_l{l}")).detach().numpy().astype(np.float32)
        elif name == "EncodecResnetBlock":
            for bi, sub in enumerate(layer.block):
                if type(sub).__name__ == "EncodecConv1d":
                    conv(pre + f"block.{bi}.", sub)
            conv(pre + "shortcut.", layer.shortcut)
    return W


def hf_model(normalize: bool):
    from transformers import EncodecConfig as HC, EncodecModel
    torch.manual_seed(0)
    m = EncodecModel(HC(normalize=normalize)).eval()
    for layer in m.quantizer.layers:                       # codebooks are zero-initialised buffers
        layer.codebook.embed.normal_()
    return m


@pytest.mark.parametrize("normalize,bandwidth", [(False, 6.0), (True, 1.5)])
def test_encode_matches_transformers(normalize, bandwidth):
    m = hf_model(normalize)
    W = hf_encoder_to_mlx(m)
    md = m.double()                                          # fp32-rounded weights vs HF's own: ~1e-7
    cfg = oe.EncodecConfig(normalize=normalize)
    x = eer.synth_clip(2, 24017, seed=5)                    # longer than every reflect pad (HF pads short inputs differently)
    x[1] *= 0.3
    with torch.no_grad():
        xt = torch.from_numpy(x.astype(np.float64)).permute(0, 2, 1)
        z_hf = md.encoder(xt / (xt.mean(1, keepdim=True).pow(2).mean(-1, keepdim=True).sqrt() + 1e-8) if normalize else xt)
        out = md.encode(xt, bandwidth=bandwidth, return_dict=True)
    codes, scales, z = eer.encode(cfg, W, x, bandwidth=bandwidth, return_latent=True)
    n_q = {6.0: 8, 1.5: 2}[bandwidth]
    assert codes.shape == tuple(out.audio_codes.shape) == (1, 2, n_q, 76)
    zr = z_hf.permute(0, 2, 1).numpy()
    assert np.abs(z[0] - zr).max() / np.abs(zr).max() < 1e-5
    assert np.array_equal(codes, out.audio_codes.numpy())
    if normalize:
        assert np.abs(scales[0] - out.audio_scales[0].reshape(-1).numpy()).max() < 1e-12
    else:
        assert scales == [None] and out.audio_scales[0] is None


def test_layout_and_keys_follow_the_module_array():
    from transformers import EncodecConfig as HC, EncodecModel
    cfg = oe.EncodecConfig()
    kinds = [k for _, k, _ in eer.encoder_layout(cfg)]
    assert kinds == ["conv"] + ["resnet", "elu", "conv"] * 4 + ["lstm", "elu", "conv"]
    hf = EncodecModel(HC())
    assert [type(l).__name__ for l in hf.encoder.layers] == ["EncodecConv1d"] + ["EncodecResnetBlock", "ELU", "EncodecConv1d"] * 4 + \
        ["EncodecLSTM", "ELU", "EncodecConv1d"]
    W = eer.init_encoder_weights(cfg, 0)
    assert set(W) == set(k for k in hf_encoder_to_mlx(hf) if k.startswith("encoder."))
    assert W["encoder.layers.0.conv.weight"].shape == (32, 7, 1)
    assert W["encoder.layers.3.conv.weight"].shape == (64, 4, 32)          # ratio 2: k 4, stride 2
    assert W["encoder.layers.12.conv.weight"].shape == (512, 16, 256)      # ratio 8: k 16, stride 8
    assert W["encoder.layers.13.lstm.1.Wh"].shape == (2048, 512)
    assert W["encoder.layers.15.conv.weight"].shape == (128, 7, 512)


def test_bandwidth_to_codebooks():
    cfg = oe.EncodecConfig()
    assert [eer.num_quantizers_for_bandwidth(cfg, b) for b in cfg.target_bandwidths] == [2, 4, 8, 16, 32]
    assert eer.num_quantizers_for_bandwidth(cfg, None) == 32


@pytest.mark.parametrize("n,offsets,clen", [(960, [0], 960), (1440, [0, 480], 960), (1920, [0, 480, 960], 960), (500, [0], 500)])
def test_chunk_loop(n, offsets, clen):
    cfg = oe.EncodecConfig(chunk_length_s=0.04, overlap=0.5)
    assert eer.chunk_offsets(cfg, n) == (offsets, clen)


@pytest.mark.parametrize("n", [1000, 1500, 2000])
def test_ragged_chunks_are_rejected(n):
    with pytest.raises(ValueError):
        eer.chunk_offsets(oe.EncodecConfig(chunk_length_s=0.04, overlap=0.5), n)


def test_encode_shapes_chunks_and_batched_equals_serial():
    cfg = oe.EncodecConfig(chunk_length_s=0.04, overlap=0.5, normalize=True, num_filters=8, hidden_size=16, codebook_dim=16,
                           codebook_size=64)
    W = {**oe.init_weights(cfg, 1, n_codebooks=32), **eer.init_encoder_weights(cfg, 2)}
    x = eer.synth_clip(3, 1920, seed=1)
    x[2] *= 0.1
    codes, scales = eer.encode(cfg, W, x, bandwidth=3.0)
    assert codes.shape == (3, 3, 6, 3) and len(scales) == 3 and all(s.shape == (3,) for s in scales)
    for c, o in enumerate((0, 480, 960)):
        chunk = x[:, o:o + 960].astype(np.float64)
        assert np.allclose(scales[c], np.sqrt((chunk.mean(-1) ** 2).mean(-1)) + 1e-8, rtol=1e-12)
    for b in range(3):
        cb, sb = eer.encode(cfg, W, x[b:b + 1], bandwidth=3.0)
        assert np.array_equal(cb, codes[:, b:b + 1]) and all(np.allclose(s, t[b:b + 1]) for s, t in zip(sb, scales))


def test_ordered_fp32_search_is_the_fp32_argmin():
    rng = np.random.default_rng(0)
    e = rng.standard_normal((64, 16)).astype(np.float32)
    x = rng.standard_normal((50, 16)).astype(np.float32)
    idx = eer.ordered_fp32_search(e, x)
    d64 = ((x.astype(np.float64)[:, None] - e.astype(np.float64)[None]) ** 2).sum(-1)
    assert (idx == d64.argmin(-1)).mean() > 0.95
    # ties resolve to the lowest index
    e2 = np.concatenate([e[:4], e[:4]])
    assert (eer.ordered_fp32_search(e2, x) < 4).all()


def test_golden_reproduces():
    import sys
    sys.path.insert(0, str(GOLDEN))
    import make_golden_encodec_encode as mg
    g = np.load(GOLDEN / "encodec_encode.npz")
    z, codes = mg.compute()
    assert tuple(g["z_shape"]) == z.shape
    assert np.abs(z.reshape(-1)[:16] - g["z_first"]).max() < 1e-6
    assert np.abs(mg.stats(z) - g["z_stats"]).max() < 1e-12
    assert np.array_equal(codes, g["codes"])
