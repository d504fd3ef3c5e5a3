"""The float64 SNAC encode reference (tests/snac_encoder_reference.py) against transformers' DAC encoder, its preprocess padding and
shapes, its golden, and the voice-cloning prompt framing of the library (b2a_tts_prepare_input_ids_ref).  CPU only."""
import ctypes as C

import numpy as np
import pytest
import torch

import snac_encoder_reference as ser
from conftest import GOLDEN
from oracle import snac


def test_dense_encoder_blocks_match_transformers_dac_encoder():
    """With depthwise = false the SNAC encoder's stem and EncoderBlocks (Layers.swift:236-259, 328-337) are DAC's conv1 + block:
    k7 stem -> per block three dilated residual units, Snake, conv k = 2s, stride s, padding ceil(s/2).  Same weights (weight norm
    folded) in float64."""
    from transformers import DacConfig
    from transformers.models.dac.modeling_dac import DacEncoder
    cfg = snac.SNACConfig(encoder_dim=8, encoder_rates=(2, 4, 8, 8), depthwise=False)
    w = ser.init_encoder_weights(cfg, 11)
    enc = DacEncoder(DacConfig(encoder_hidden_size=8, downsampling_ratios=list(cfg.encoder_rates), hidden_size=16)).double()
    p = "encoder.block.layers"
    with torch.no_grad():
        enc.conv1.weight.copy_(snac.wn_conv_weight(w, f"{p}.0")); enc.conv1.bias.copy_(snac._t(w[f"{p}.0.bias"]))
        for i, blk in enumerate(enc.block):
            b = f"{p}.{i + 1}.block.layers"
            for j, ru in enumerate((blk.res_unit1, blk.res_unit2, blk.res_unit3)):
                r = f"{b}.{j}.block.layers"
                ru.snake1.alpha.copy_(snac._t(w[f"{r}.0.alpha"])); ru.snake2.alpha.copy_(snac._t(w[f"{r}.2.alpha"]))
                ru.conv1.weight.copy_(snac.wn_conv_weight(w, f"{r}.1")); ru.conv1.bias.copy_(snac._t(w[f"{r}.1.bias"]))
                ru.conv2.weight.copy_(snac.wn_conv_weight(w, f"{r}.3")); ru.conv2.bias.copy_(snac._t(w[f"{r}.3.bias"]))
            blk.snake1.alpha.copy_(snac._t(w[f"{b}.3.alpha"]))
            blk.conv1.weight.copy_(snac.wn_conv_weight(w, f"{b}.4")); blk.conv1.bias.copy_(snac._t(w[f"{b}.4.bias"]))
    x = torch.randn(2, 1, 2048, dtype=torch.float64)
    with torch.no_grad():
        ref = enc.conv1(x)
        for blk in enc.block:
            ref = blk(ref)
        ours = ser.encoder_blocks(cfg, w, x)
    assert ours.shape == ref.shape == (2, 128, 4) and (ours - ref).abs().max() < 1e-10


@pytest.mark.parametrize("n,padded", [(1, 2048), (2047, 2048), (2048, 2048), (2049, 4096), (12000, 12288), (24000 * 30, 720896)])
def test_preprocess_padding_and_code_shapes(n, padded):
    cfg = snac.SNACConfig()
    assert ser.pad_multiple(cfg) == 512 * 4
    x = np.ones((2, 1, n), dtype=np.float32)
    y = ser.preprocess(cfg, x)
    assert y.shape == (2, 1, padded) and np.array_equal(y[..., :n], x) and not y[..., n:].any()


def test_encode_shapes_and_batched_equals_serial():
    cfg = snac.SNACConfig()
    W = {**snac.init_weights(cfg, 1234), **ser.init_encoder_weights(cfg, 4321)}
    audio = ser.synth_clip(3, 5000, seed=2)
    audio[1] *= 0.2
    z = ser.encode_latent(cfg, W, audio)
    assert z.shape == (3, 768, 12)
    codes = ser.encode(cfg, W, audio)
    assert [c.shape for c in codes] == [(3, 3), (3, 6), (3, 12)]
    assert all(c.min() >= 0 and c.max() < 4096 for c in codes)
    for b in range(3):
        assert np.abs(ser.encode_latent(cfg, W, audio[b:b + 1]) - z[b:b + 1]).max() < 1e-12
        assert all(np.array_equal(c[b:b + 1], o) for c, o in zip(codes, ser.encode(cfg, W, audio[b:b + 1])))


def test_golden_reproduces():
    g = np.load(GOLDEN / "snac_encode.npz")
    cfg = snac.SNACConfig()
    W = {**snac.init_weights(cfg, 1234), **ser.init_encoder_weights(cfg, 4321)}
    audio = ser.synth_clip(2, 5000, 3)
    z = ser.encode_latent(cfg, W, audio)
    assert tuple(g["z_shape"]) == z.shape
    assert np.abs(z.reshape(-1)[:16] - g["z_first"]).max() < 1e-6
    assert np.abs(np.array([z.mean(), np.abs(z).mean(), z.min(), z.max()]) - g["z_stats"]).max() < 1e-12
    codes = snac.quantize(cfg, W, z)[1]
    assert all(np.array_equal(c, g[f"codes{i}"]) for i, c in enumerate(codes))


def test_random_init_weights_default_is_unchanged(b2a):
    a = b2a.SNAC.random_init_weights()
    e = b2a.SNAC.random_init_weights(encoder=True)
    assert not any(k.startswith("encoder.") for k in a)
    assert set(e) - set(a) == {k for k in e if k.startswith("encoder.")} and len(e) > len(a)
    assert all(np.array_equal(a[k], e[k]) for k in a)


def _ref_ids(b2a, prompts, text, codes):
    rows = [np.ascontiguousarray(p, dtype=np.int32) for p in prompts]
    lens = np.asarray([len(r) for r in rows], dtype=np.int32)
    pp = (C.c_void_p * len(rows))(*[r.ctypes.data if len(r) else None for r in rows])
    t = np.ascontiguousarray(text, dtype=np.int32)
    c = np.ascontiguousarray(codes, dtype=np.int32)
    n = C.c_int32(0)
    lib = b2a._ffi.lib()
    st = lib.b2a_tts_prepare_input_ids_ref(pp, b2a._ffi.ptr(lens), len(rows), b2a._ffi.ptr(t), len(t), b2a._ffi.ptr(c), len(c), None,
                                          C.byref(n))
    if st != 0:
        return st, None
    out = np.empty((len(rows), n.value), dtype=np.int32)
    b2a._ffi.check(lib.b2a_tts_prepare_input_ids_ref(pp, b2a._ffi.ptr(lens), len(rows), b2a._ffi.ptr(t), len(t), b2a._ffi.ptr(c), len(c),
                                                     b2a._ffi.ptr(out), C.byref(n)))
    return st, out


def test_cloning_prompt_framing_matches_reference_restatement(b2a):
    rng = np.random.default_rng(3)
    codes = rng.integers(0, 7 * 4096, size=21).tolist()
    text = [128000, 9906, 1917, 13]
    for prompts in ([[5, 6, 7, 8, 9], [1, 2], [3]], [[42]], [[1, 2, 3], [4, 5, 6]]):
        st, ids = _ref_ids(b2a, prompts, text, codes)
        assert st == 0 and np.array_equal(ids, ser.prepare_input_ids_ref(prompts, text, codes))
        # padding comes first, then the reference block, then the prompt (LlamaTTS.swift:499-543)
        assert ids[-1, 0] == 128263 if len(set(map(len, prompts))) > 1 else ids[0, 0] == 128259
        got, mask = b2a.LlamaTTSModel.prepare_input_ids(prompts, codes, text)
        assert np.array_equal(got, ids) and np.array_equal(mask, ids != 128263)
    st, ids = _ref_ids(b2a, [[1, 2]], [], codes)                   # an empty transcript
    assert st == 0 and np.array_equal(ids, ser.prepare_input_ids_ref([[1, 2]], [], codes))
    assert ids[0, :3].tolist() == [128259, 128009, 128260]
    # with either piece missing the prompts are framed alone
    plain, _ = b2a.LlamaTTSModel.prepare_input_ids([[1, 2]], codes, None)
    assert np.array_equal(plain, b2a.LlamaTTSModel.prepare_input_ids([[1, 2]])[0])


@pytest.mark.parametrize("codes", [[1] * 6, [7 * 4096] + [0] * 6, [-1] + [0] * 6], ids=["not-7", "too-big", "negative"])
def test_cloning_prompt_errors(b2a, codes):
    st, _ = _ref_ids(b2a, [[1, 2]], [5], codes)
    assert st == b2a._ffi.ERR_INVALID_INPUT
    with pytest.raises(b2a.AudioGenerationError) as e:
        b2a.LlamaTTSModel.prepare_input_ids([[1, 2]], codes, [5])
    assert e.value.case == "invalidInput"
    n = C.c_int32(0)
    assert b2a._ffi.lib().b2a_tts_prepare_input_ids_ref(None, None, 1, None, 0, None, 0, None, C.byref(n)) == b2a._ffi.ERR_INVALID_INPUT
