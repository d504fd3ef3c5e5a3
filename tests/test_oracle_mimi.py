"""The float64 Mimi reference (oracle/mimi.py) pinned against transformers.MimiModel (random init, float64, q / k rows permuted
per head); where the per-call attention window makes them part; the streaming decodeStep against the one-shot decode; the
sanitize key for key against the library's; the default config; the golden fixture.  CPU only."""
import ctypes as C
import sys

import numpy as np
import pytest
import torch

import qwen3_encoder_reference as qer
from conftest import GOLDEN
from oracle import mimi as om

HF = dict(hidden_size=64, num_filters=16, upsampling_ratios=[8, 6, 5, 4], num_attention_heads=2, num_key_value_heads=2, head_dim=32,
          intermediate_size=128, num_hidden_layers=2, codebook_size=64, codebook_dim=16, vector_quantization_hidden_dimension=16,
          num_quantizers=8, num_semantic_quantizers=1, sliding_window=250, use_causal_conv=True, frame_rate=12.5, sampling_rate=24000,
          upsample_groups=64, kernel_size=7, last_kernel_size=3, residual_kernel_size=3, compress=2, num_residual_layers=1,
          use_conv_shortcut=False, rope_theta=10000.0, norm_eps=1e-5, trim_right_ratio=1.0)


def hf_model(seed=0):
    from transformers import MimiConfig, MimiModel
    torch.manual_seed(seed)
    m = MimiModel(MimiConfig(**HF)).double().eval()
    with torch.no_grad():                   # make the layer scales and norms matter, and give the codebooks spread-out usages
        for name, p in m.named_parameters():
            if "layer_scale" in name:
                p.copy_(0.3 + 0.2 * torch.rand_like(p))
            elif "norm" in name and name.endswith("weight"):
                p.copy_(1 + 0.1 * torch.randn_like(p))
            elif "norm" in name and name.endswith("bias"):
                p.copy_(0.05 * torch.randn_like(p))
            elif "upsample" in name:
                p.copy_(0.5 + 0.3 * torch.randn_like(p))
        for name, b in m.named_buffers():
            if name.endswith("cluster_usage"):
                b.copy_(0.5 + 1.5 * torch.rand_like(b))
            elif name.endswith("embed_sum"):
                b.copy_(torch.randn_like(b) * 0.5)
    return m


def hf_weights(m):
    """MimiModel.state_dict() -> the oracle's names and MLX layouts.  The encoder and quantizer go through the Qwen3 encoder
    reference's sanitize (the same modules); the decoder half is mapped here.  q / k rows are permuted per head (trap 1)."""
    cfg = m.config
    perm = qer.hf_qk_permutation(cfg.num_attention_heads, cfg.head_dim)
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    W = qer.sanitize_encoder({"encoder." + k: (v[perm] if (".q_proj." in k or ".k_proj." in k) else v) for k, v in sd.items()})
    W["upsample.convtr.convtr.convtr.weight"] = sd["upsample.conv.weight"].transpose(0, 2, 1)
    tl = {"self_attn.o_proj.weight": "self_attn.out_proj.weight", "mlp.fc1.weight": "gating.linear1.weight",
          "mlp.fc2.weight": "gating.linear2.weight", "input_layernorm.weight": "norm1.weight", "input_layernorm.bias": "norm1.bias",
          "post_attention_layernorm.weight": "norm2.weight", "post_attention_layernorm.bias": "norm2.bias",
          "self_attn_layer_scale.scale": "layer_scale_1.scale", "mlp_layer_scale.scale": "layer_scale_2.scale"}
    for l in range(cfg.num_hidden_layers):
        p, q = f"decoder_transformer.layers.{l}.", f"decoder_transformer.transformer.layers.{l}."
        W[q + "self_attn.in_proj.weight"] = np.concatenate([sd[p + "self_attn.q_proj.weight"][perm], sd[p + "self_attn.k_proj.weight"][perm],
                                                            sd[p + "self_attn.v_proj.weight"]], 0)
        for a, b in tl.items():
            W[q + b] = sd[p + a]
    conv = lambda k: sd[k].transpose(0, 2, 1)
    W["decoder.init_conv1d.conv.conv.weight"], W["decoder.init_conv1d.conv.conv.bias"] = conv("decoder.layers.0.conv.weight"), sd["decoder.layers.0.conv.bias"]
    for i in range(4):
        p, q = f"decoder.layers.{2 + 3 * i}.conv.", f"decoder.layers.{i}.upsample.convtr.convtr."
        W[q + "weight"], W[q + "bias"] = sd[p + "weight"].transpose(1, 2, 0), sd[p + "bias"]
        for j, blk in ((0, 1), (1, 3)):
            p, q = f"decoder.layers.{3 + 3 * i}.block.{blk}.conv.", f"decoder.layers.{i}.residuals.0.block.{j}.conv.conv."
            W[q + "weight"], W[q + "bias"] = conv(p + "weight"), sd[p + "bias"]
    W["decoder.final_conv1d.conv.conv.weight"], W["decoder.final_conv1d.conv.conv.bias"] = conv("decoder.layers.14.conv.weight"), sd["decoder.layers.14.conv.bias"]
    return W


def codes_for(cfg, B, K, T, seed=0):
    return np.random.default_rng(seed).integers(0, cfg.codebook_size, (B, K, T)).astype(np.int32)


@pytest.mark.parametrize("K", [1, 3, 8])
def test_decode_matches_transformers(K):
    m = hf_model()
    cfg, W = om.small_config(), hf_weights(m)
    assert set(W) == set(om.init_weights(cfg)), "hf_weights covers exactly the oracle's key set"
    codes = codes_for(cfg, 2, K, 60, seed=K)
    with torch.no_grad():
        ref = m.decode(torch.from_numpy(codes).long()).audio_values.numpy()
    got = om.decode(cfg, W, codes)
    assert got.shape == ref.shape == (2, 1, 60 * 1920)
    assert np.abs(got - ref).max() < 1e-6 * np.abs(ref).max()


def test_encode_matches_transformers():
    m = hf_model(1)
    cfg, W = om.small_config(), hf_weights(m)
    x = qer.synth_clip(2, 24000 * 2 + 333, seed=5)
    with torch.no_grad():
        ref = m.encode(torch.from_numpy(x).double(), num_quantizers=8).audio_codes.numpy()
    got = om.encode(cfg, W, x)
    assert got.shape == ref.shape == (2, 8, om.encoded_length(cfg, x.shape[-1]))
    assert (got != ref).mean() < 0.01                  # float64 near-ties only (the Qwen3 encoder test pins the tie rule)


def test_decode_past_the_window_parts_from_transformers():
    """Past 250 latent positions (125 code frames) transformers drops keys per query; the one-shot decode attends the whole clip."""
    m = hf_model(2)
    cfg, W = om.small_config(), hf_weights(m)
    codes = codes_for(cfg, 1, 8, 140, seed=9)
    with torch.no_grad():
        ref = m.decode(torch.from_numpy(codes).long()).audio_values.numpy()
    got = om.decode(cfg, W, codes)
    cut = 125 * 1920
    peak = np.abs(ref).max()
    assert np.abs(got[..., :cut] - ref[..., :cut]).max() < 1e-6 * peak
    assert np.abs(got[..., cut:] - ref[..., cut:]).max() > 1e-4 * peak


@pytest.mark.parametrize("chunk", [1, 3, 7])
def test_stream_equals_one_shot_within_the_window(chunk):
    cfg = om.small_config()
    W = om.init_weights(cfg, 3)
    codes = codes_for(cfg, 2, 8, 125, seed=chunk)
    ref = om.decode(cfg, W, codes)
    st = om.MimiStreamer(cfg, W)
    got = np.concatenate([st.decode_step(codes[:, :, t:t + chunk]) for t in range(0, 125, chunk)], 2)
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() < 1e-9 * np.abs(ref).max()


def test_stream_follows_the_per_call_window():
    """Frame by frame, the call at offset p0 keeps keys [p0 - 250, p0 + 1]: equal to a full-causal decode up to 125 code
    frames, different after; chunked streams see different left edges per call and differ from each other past the window."""
    cfg = om.small_config()
    W = om.init_weights(cfg, 4)
    codes = codes_for(cfg, 1, 8, 150, seed=11)
    full = om.decode(cfg, W, codes)
    s1 = om.MimiStreamer(cfg, W).decode_frames(codes[0])
    st = om.MimiStreamer(cfg, W)
    s7 = np.concatenate([st.decode_step(codes[:, :, t:t + 7]) for t in range(0, 150, 7)], 2)
    cut, peak = 125 * 1920, np.abs(full).max()
    for s in (s1, s7):
        assert np.abs(s[..., :cut] - full[..., :cut]).max() < 1e-9 * peak
        assert np.abs(s[..., cut:] - full[..., cut:]).max() > 1e-4 * peak
    assert np.abs(s1[..., cut:] - s7[..., cut:]).max() > 1e-4 * peak


def test_reset_starts_over():
    cfg = om.small_config()
    W = om.init_weights(cfg, 5)
    codes = codes_for(cfg, 1, 8, 6, seed=2)
    st = om.MimiStreamer(cfg, W)
    a = st.decode_frames(codes)
    st.decode_frames(codes)
    st.reset()
    assert np.array_equal(st.decode_frames(codes), a)


def test_sanitize_key_for_key(b2a, tmp_path):
    from safetensors.numpy import save_file
    cfg = om.small_config()
    W = om.init_weights(cfg, 6)
    ck = om.unsanitize(W)
    assert "decoder.model.2.convtr.convtr.weight" in ck and "encoder.model.14.conv.conv.weight" in ck
    assert "decoder_transformer.transformer.layers.1.self_attn.in_proj_weight" in ck and "decoder_transformer.transformer.layers.0.linear2.weight" in ck
    assert "quantizer.rvq_rest.vq.layers.6._codebook.embedding_sum" in ck and "decoder.model.12.block.3.conv.conv.bias" in ck
    assert ck["upsample.convtr.convtr.convtr.weight"].shape == (64, 1, 4) and ck["decoder.model.5.convtr.convtr.weight"].shape == (128, 64, 12)
    ref = om.sanitize(ck)
    assert ref.keys() == W.keys() and all(np.array_equal(ref[k], W[k]) for k in W)
    save_file({k: np.ascontiguousarray(v, np.float32) for k, v in ck.items()}, str(tmp_path / "m.safetensors"))
    w = b2a.loading.Weights(tmp_path / "m.safetensors")
    w.sanitize_mimi()
    got = w.tensors()
    assert got.keys() == W.keys()
    for k, v in W.items():
        assert got[k].shape == v.shape and np.array_equal(got[k], v), k


def test_config_default_is_mimi_202407(b2a):
    from mlx_audio_swift_b200 import _ffi
    c = _ffi.MimiConfig()
    _ffi.check(_ffi.lib().b2a_mimi_config_default(32, 8, 2250, C.byref(c)))
    r = om.mimi_202407(32)
    assert (c.sample_rate, c.channels, c.dimension, c.n_filters, c.n_residual_layers, list(c.ratios)[:c.num_ratios]) == \
        (r.sample_rate, 1, r.dimension, r.n_filters, 1, list(r.ratios))
    assert (c.kernel_size, c.residual_kernel_size, c.last_kernel_size, c.dilation_base, c.compress, c.causal, c.true_skip) == \
        (r.kernel_size, r.residual_kernel_size, r.last_kernel_size, 2, r.compress, 1, 1)
    assert (c.num_heads, c.num_layers, c.dim_feedforward, c.context, c.max_period, c.gating, c.norm_rms, c.kv_repeat) == \
        (r.num_heads, r.num_layers, r.dim_feedforward, r.context, r.max_period, 0, 0, 1)
    assert (c.num_codebooks, c.codebook_size, c.codebook_dim, c.max_batch, c.max_cache_frames) == (32, 2048, 256, 8, 2250)
    assert c.frame_rate == 12.5 and r.samples_per_frame == 1920 and r.downsample_stride == 2
    with pytest.raises(_ffi.AudioGenerationError) as e:
        _ffi.check(_ffi.lib().b2a_mimi_config_default(0, 8, 2250, C.byref(c)))
    assert e.value.case == "invalidInput"


def test_golden_reproduces():
    sys.path.insert(0, str(GOLDEN))
    import make_golden_mimi as mg
    g = np.load(GOLDEN / "mimi.npz")
    cfg, W, codes = mg.inputs()
    one = om.decode(cfg, W, codes)
    assert np.abs(one[..., ::mg.STRIDE] - g["decode"]).max() < 1e-6 * np.abs(g["decode"]).max()
    stream = om.MimiStreamer(cfg, W).decode_frames(codes)
    assert np.abs(stream[..., ::mg.STRIDE] - g["stream"]).max() < 1e-6 * np.abs(g["stream"]).max()
    assert np.array_equal(om.encode(cfg, W, mg.clip()), g["codes"])
