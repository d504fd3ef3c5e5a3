"""max_batch is 1..32 for the Llama, Qwen3 LM (VyvoTTS), Soprano and Qwen3-TTS talker handles: 0 and 33 are rejected with invalidInput
before any device work, so no GPU is needed."""
import ctypes as C

import pytest


@pytest.fixture(scope="module")
def ffi():
    import mlx_audio_swift_b200 as m
    return m._ffi


def _llama(ffi, mb):
    c = ffi.LlamaConfig(256, 2, 512, 2, 1, 128, 2048, 1e-5, 500000.0, 32.0, 1.0, 4.0, 8192.0, 1, mb, 64)
    return ffi.lib().b2a_tts_create_random(0, C.byref(c), 0.02, 1, None, C.byref(C.c_void_p()))


def _qwen3_lm(ffi, mb):
    c = ffi.Qwen3LMConfig(256, 2, 512, 2, 1, 128, 2048, 1e-6, 1e6, 1.0, 1, 4096, 24000, 0, mb, 64)
    return ffi.lib().b2a_qwen3_lm_create_random(0, C.byref(c), 0.02, 1, None, C.byref(C.c_void_p()))


def _soprano(ffi, mb):
    from mlx_audio_swift_b200.soprano_tts import SopranoModel
    c = SopranoModel._c_config(dict(hidden_size=256, num_hidden_layers=2, intermediate_size=512, num_attention_heads=2, num_key_value_heads=1,
                                    head_dim=128, vocab_size=512), mb, 64)
    dummy = (ffi.Tensor * 1)()
    return ffi.lib().b2a_soprano_create_random(0, C.byref(c), 0.02, 1, dummy, 1, C.byref(C.c_void_p()))


def _talker(ffi, mb):
    import mlx_audio_swift_b200 as m
    c = m.Qwen3TalkerConfig()._c(mb, 64)
    return ffi.lib().b2a_qwen3_talker_create_random(0, C.byref(c), 0.02, 1, C.byref(C.c_void_p()))


@pytest.mark.parametrize("create", [_llama, _qwen3_lm, _soprano, _talker])
@pytest.mark.parametrize("max_batch", [0, 33])
def test_max_batch_outside_1_to_32_is_invalid_input(ffi, create, max_batch):
    assert create(ffi, max_batch) == ffi.ERR_INVALID_INPUT
    assert b"max_batch must be in 1..32" in ffi.lib().b2a_last_error()
