"""CPU checks of the float64 reference of the 32 / 44 kHz SNAC models (tests/snac_attention_reference.py): LocalMHA against an
independent composition (torch.nn.LayerNorm, transformers' Llama rotate_half / apply_rotary_pos_emb, F.scaled_dot_product_attention),
the 24 kHz reference unchanged without attention, odd-stride stage lengths, the preprocess multiple and the golden."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import snac_attention_reference as sar
import snac_encoder_reference as ser
from conftest import GOLDEN
from oracle import snac


def independent_local_mha(w, prefix, x, window):
    from transformers.models.llama.modeling_llama import apply_rotary_pos_emb
    B, C, T = x.shape
    H = C // 64
    ln = torch.nn.LayerNorm(C, eps=1e-5, dtype=torch.float64)
    with torch.no_grad():
        ln.weight.copy_(torch.as_tensor(w[prefix + ".norm.weight"], dtype=torch.float64))
        ln.bias.copy_(torch.as_tensor(w[prefix + ".norm.bias"], dtype=torch.float64))
    h = ln(x.transpose(1, 2))
    q, k, v = (h @ torch.as_tensor(w[prefix + ".to_qkv.weight"], dtype=torch.float64).T).split(C, dim=-1)
    # windows as batch rows: [B * W, H, window, 64]
    q, k, v = (t.reshape(B * (T // window), window, H, 64).transpose(1, 2) for t in (q, k, v))
    inv = torch.as_tensor(w[prefix + ".rel_pos.inv_freq"], dtype=torch.float64)
    f = torch.arange(window, dtype=torch.float64)[:, None] * inv[None]
    emb = torch.cat([f, f], dim=-1)
    q, k = apply_rotary_pos_emb(q, k, emb.cos()[None], emb.sin()[None])
    o = F.scaled_dot_product_attention(q, k, v)
    o = o.transpose(1, 2).reshape(B, T, C) @ torch.as_tensor(w[prefix + ".to_out.weight"], dtype=torch.float64).T
    return o.transpose(1, 2) + x


@pytest.mark.parametrize("dim,window,T", [(128, 16, 48), (256, 32, 64), (128, 7, 21)])
def test_local_mha_matches_independent_composition(dim, window, T):
    rng = np.random.default_rng(dim + window)
    w = sar.init_attn_weights("a", dim, rng)
    x = torch.as_tensor(rng.standard_normal((2, dim, T)) * 3.0, dtype=torch.float64)
    with torch.no_grad():
        ref = sar.local_mha(w, "a", x, window)
        ind = independent_local_mha(w, "a", x, window)
    assert ref.shape == x.shape
    assert torch.max(torch.abs(ref - ind)).item() < 1e-12


def test_without_attention_equals_24khz_reference():
    cfg = snac.SNACConfig()
    W = {**snac.init_weights(cfg, 1234), **ser.init_encoder_weights(cfg, 4321)}
    codes = snac.synth_codes(cfg, 1, 8, seed=5)
    rng = np.random.default_rng(1)
    noise = [rng.standard_normal(s) for s in snac.noise_shapes(cfg, 1, 8)]
    assert np.array_equal(sar.decode(cfg, W, codes, noise), snac.decode(cfg, W, codes, noise))
    audio = ser.synth_clip(1, 3000, 2)
    assert np.array_equal(sar.encode_latent(cfg, W, audio), ser.encode_latent(cfg, W, audio))
    assert sar.pad_multiple(cfg) == cfg.hop_length * math.lcm(*cfg.vq_strides)


def test_odd_stride_stage_lengths():
    cfg = sar.small()
    T = 32
    lens = sar.stage_lengths(cfg, T)
    t = T
    for s, n in zip(cfg.decoder_rates, lens):
        assert n == s * t - (s % 2)
        t = n
    W = sar.init_weights(cfg, 11)
    codes = snac.synth_codes(cfg, 1, T, seed=3)
    y = sar.decode(cfg, W, codes, None)
    assert y.shape == (1, 1, lens[-1]) and lens[-1] == 12 * T - 2
    pub = sar.published()
    assert sar.stage_lengths(pub, 64)[-1] == 384 * 64 - 2


def test_preprocess_multiple_published():
    for sr in (32000, 44100):
        cfg = sar.published(sr)
        assert cfg.latent == 1024 and cfg.hop_length == 384
        assert sar.pad_multiple(cfg) == 12288


def test_encoder_with_attention_shapes():
    cfg = sar.small()
    W = sar.init_weights(cfg, 11)
    audio = ser.synth_clip(2, 500, 4)
    z = sar.encode_latent(cfg, W, audio)
    assert z.shape == (2, cfg.latent, 192 * 3 // cfg.hop_length)
    assert np.isfinite(z).all()


def test_golden_reproduces():
    import importlib.util
    spec = importlib.util.spec_from_file_location("mg44", GOLDEN / "make_golden_snac_44khz.py")
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
    g = np.load(GOLDEN / "snac_44khz.npz")
    cur = mg.compute()
    for k in g.files:
        if g[k].dtype.kind in "iu":
            assert np.array_equal(g[k], cur[k]), k
        else:
            np.testing.assert_allclose(cur[k], g[k], rtol=1e-9, atol=1e-9, err_msg=k)
