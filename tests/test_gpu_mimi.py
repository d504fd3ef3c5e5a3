"""Mimi on the GPU (csrc/mimi.cu) against the float64 oracle (oracle/mimi.py): one-shot decode at the small geometry and at
mimi_202407(32) with K = 1 .. 32 codebooks, encode codes bit for bit against the oracle's ordered-fp32 search on the device's
own latent, streaming against the one-shot waveform and against the oracle's windowed stream, reset, batch determinism and the
error cases."""
import ctypes as C
import functools

import numpy as np
import pytest

import qwen3_encoder_reference as qer
from oracle import mimi as om

pytestmark = pytest.mark.gpu

SMALL = dict(dimension=64, n_filters=16, num_heads=2, num_layers=2, dim_feedforward=128, codebook_size=64, codebook_dim=16)


def small(b2a, W=None, seed=0, nq=8, **kw):
    cfg = om.small_config(nq)
    W = W if W is not None else om.init_weights(cfg, seed)
    kw.setdefault("max_cache_frames", 256)
    return cfg, W, b2a.Mimi(W, nq, **SMALL, **kw)


def codes_for(cfg, B, K, T, seed=0):
    return np.random.default_rng(seed).integers(0, cfg.codebook_size, (B, K, T)).astype(np.int32)


def peak_err(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / np.abs(b).max())


@pytest.mark.parametrize("K", [1, 3, 8])
def test_decode_small(b2a, K):
    cfg, W, m = small(b2a, seed=1)
    codes = codes_for(cfg, 2, K, 40, seed=K)
    got = m.decode(codes)
    assert got.shape == (2, 1, 40 * 1920)
    assert peak_err(got, om.decode(cfg, W, codes)) <= 1e-3


@functools.lru_cache(maxsize=1)
def full_weights():
    return om.init_weights(om.mimi_202407(32), 7)


@pytest.mark.parametrize("K", [1, 8, 32])
def test_decode_mimi_202407(b2a, K):
    cfg, W = om.mimi_202407(32), full_weights()
    m = b2a.Mimi(W, 32, max_batch=2, max_cache_frames=64)
    codes = codes_for(cfg, 2, K, 50, seed=K)             # 2 x 4 s
    assert peak_err(m.decode(codes), om.decode(cfg, W, codes)) <= 1e-3


def test_encode_codes_and_round_trip(b2a):
    from mlx_audio_swift_b200 import _ffi
    cfg, W, m = small(b2a, seed=2)
    x = qer.synth_clip(2, 24000 * 2 + 777, seed=8)
    codes = m.encode(x)
    T = om.encoded_length(cfg, x.shape[-1])
    assert codes.shape == (2, 8, T) and codes.dtype == np.int32
    # the same implementation as a standalone speech-tokenizer encoder, which exposes its latent: codes == fp32 search on it
    e = _ffi.SpeechTokenizerEncoderConfig(sampling_rate=24000, frame_rate=12.5, audio_channels=1, num_filters=16, num_residual_layers=1,
                                          num_upsampling_ratios=4, kernel_size=7, residual_kernel_size=3, last_kernel_size=3, compress=2,
                                          use_causal_conv=1, use_conv_shortcut=0, hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                                          num_attention_heads=2, num_key_value_heads=2, head_dim=32, rope_theta=10000.0, codebook_size=64,
                                          codebook_dim=16, num_quantizers=8, valid_num_quantizers=8)
    for i, r in enumerate((8, 6, 5, 4)):
        e.upsampling_ratios[i] = r
    table, keep = _ffi.make_tensor_table(W)
    h = C.c_void_p()
    _ffi.check(_ffi.lib().b2a_speech_tokenizer_encoder_create(0, C.byref(e), table, len(W), C.byref(h)))
    z = np.empty((2, T, 64), np.float32)
    c2 = np.empty((2, 8, T), np.int32)
    xa = np.ascontiguousarray(x.reshape(2, -1))
    _ffi.check(_ffi.lib().b2a_speech_tokenizer_encoder_latent_test(h, _ffi.ptr(xa), 2, xa.shape[1], _ffi.ptr(z), _ffi.ptr(c2)))
    _ffi.lib().b2a_speech_tokenizer_encoder_destroy(h)
    assert np.array_equal(codes, c2)
    assert np.array_equal(codes, qer.encode_codes_fp32(cfg, W, z))
    assert np.abs(z - qer.latent(cfg, W, x)).max() < 1e-4 * np.abs(z).max()
    y = m.reconstruct(x)
    assert y.shape == (2, 1, T * 1920) and np.isfinite(y).all()


@pytest.mark.parametrize("chunk", [1, 3, 7])
def test_stream_chunks_equal_one_shot(b2a, chunk):
    cfg, W, m = small(b2a, seed=3)
    codes = codes_for(cfg, 2, 8, 125, seed=chunk)
    one = m.decode(codes)
    m.reset()
    got = np.concatenate([m.decode_step(codes[:, :, t:t + chunk]) for t in range(0, 125, chunk)], 2)
    assert peak_err(got, one) <= 1e-5


def test_decode_frames_and_reset(b2a):
    cfg, W, m = small(b2a, seed=4)
    codes = codes_for(cfg, 1, 8, 125, seed=5)
    one = m.decode(codes)
    sd = b2a.MimiStreamingDecoder(m)
    a = sd.decode_frames(codes[0])               # [K, T] accepted like the reference
    assert a.shape == one.shape and peak_err(a, one) <= 1e-5
    sd.reset()
    assert np.array_equal(sd.decode_frames(codes), a)


def test_long_stream_follows_the_window(b2a):
    cfg, W, m = small(b2a, seed=5)
    codes = codes_for(cfg, 1, 8, 200, seed=6)
    got = b2a.MimiStreamingDecoder(m).decode_frames(codes)
    ref = om.MimiStreamer(cfg, W).decode_frames(codes)
    assert peak_err(got, ref) <= 1e-3
    full = om.decode(cfg, W, codes)
    assert peak_err(got[..., 130 * 1920:], full[..., 130 * 1920:]) > 1e-4     # past the window the stream is not the one-shot decode


def test_batch_rows_bit_exact(b2a):
    cfg, W, m = small(b2a, seed=6, max_batch=3)
    codes = codes_for(cfg, 3, 8, 17, seed=7)
    batch = m.decode(codes)
    for b in range(3):
        assert np.array_equal(batch[b:b + 1], m.decode(codes[b:b + 1]))


def test_errors(b2a):
    from mlx_audio_swift_b200 import _ffi
    cfg, W, m = small(b2a, seed=7, max_batch=2, max_cache_frames=10)
    codes = codes_for(cfg, 1, 8, 4)

    def case(fn, *a):
        with pytest.raises(_ffi.AudioGenerationError) as e:
            fn(*a)
        return e.value.case

    assert case(m.decode, np.zeros((1, 0, 4), np.int32)) == "invalidInput"          # K = 0
    assert case(m.decode, np.zeros((1, 9, 4), np.int32)) == "invalidInput"          # K > nq
    assert case(m.decode, np.full((1, 8, 4), 64, np.int32)) == "invalidInput"       # code >= codebook_size
    assert case(m.decode, np.full((1, 8, 4), -1, np.int32)) == "invalidInput"
    assert case(m.decode, codes_for(cfg, 3, 8, 4)) == "invalidInput"                # batch > max_batch
    m.reset()
    m.decode_step(codes_for(cfg, 1, 8, 8))
    assert case(m.decode_step, codes_for(cfg, 1, 8, 3)) == "invalidInput"           # past max_cache_frames
    assert case(m.decode_step, codes_for(cfg, 2, 8, 1)) == "invalidInput"           # batch changed inside a stream
    m.reset()
    m.decode_step(codes_for(cfg, 2, 8, 10))                                         # exactly max_cache_frames is fine
    assert case(m.encode, np.zeros((1, 1, 0), np.float32)) == "audioEncodingFailed"
    for bad in (dict(norm_rms=1), dict(gating=1), dict(n_residual_layers=2), dict(causal=0), dict(true_skip=0)):
        assert case(lambda: b2a.Mimi(W, 8, **{**SMALL, **bad})) == "invalidInput", bad
    W2 = dict(W)
    del W2["decoder.layers.2.upsample.convtr.convtr.bias"]
    assert case(lambda: b2a.Mimi(W2, 8, **SMALL)) == "modelNotInitialized"
    W3 = {k: v for k, v in W.items() if not k.startswith("encoder.")}
    assert case(lambda: b2a.Mimi(W3, 8, **SMALL)) == "modelNotInitialized"


def test_from_file(b2a, tmp_path):
    from safetensors.numpy import save_file
    cfg = om.mimi_202407(32)
    W = om.init_weights(cfg, 8)
    save_file({k: np.ascontiguousarray(v, np.float32) for k, v in om.unsanitize(W).items()}, str(tmp_path / "tokenizer.safetensors"))
    m = b2a.Mimi.from_file(tmp_path / "tokenizer.safetensors", 32, max_batch=1, max_cache_frames=16)
    assert (m.num_codebooks, m.samples_per_frame, m.codec_sample_rate, m.frame_rate) == (32, 1920, 24000.0, 12.5)
    codes = codes_for(cfg, 1, 32, 6, seed=3)
    assert peak_err(m.decode(codes), om.decode(cfg, W, codes)) <= 1e-3
