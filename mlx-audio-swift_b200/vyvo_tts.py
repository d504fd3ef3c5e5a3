"""Host-side mirror of VyvoTTS's `Qwen3Model` (Sources/MLXAudioTTS/Models/Qwen3/Qwen3.swift:305-931) behind SpeechGenerationModel, over
the C ABI.  The handle is a b2a_tts one (b2a_qwen3_lm_create*): generate, streaming, logits and cancel are LlamaTTSModel's, run with
VyvoTTS's token layout -- stop on 151671 (not kept), the Qwen3 parse rule (:333-358) and 50-frame chunked SNAC decoding (:47-83).
Tokenisation stays with the host: prompts are token ids."""
from __future__ import annotations

from . import _ffi
from .llama_tts import GenerateParameters, LlamaTTSModel

START_OF_SPEECH, END_OF_SPEECH, START_OF_AI, PAD_TOKEN, AUDIO_TOKENS_START = 151670, 151671, 151674, 151676, 151679


class Qwen3Model(LlamaTTSModel):
    """VyvoTTS: a Qwen3 language model (per-head q/k RMSNorm, rotate-half RoPE) whose vocabulary speaks SNAC-24 kHz codes.  `config` is
    the checkpoint's config.json as a dict (Qwen3Configuration, Config.swift:15-73; head_dim must be 128)."""
    default_generation_parameters = GenerateParameters(max_tokens=1200, temperature=0.6, top_p=0.8, repetition_penalty=1.3,
                                                       repetition_context_size=20)      # Qwen3.swift:510-518
    _abi = "b2a_qwen3_lm"
    _pad_token = PAD_TOKEN

    @staticmethod
    def _c_config(config: dict, max_batch: int, max_context: int) -> _ffi.Qwen3LMConfig:
        rs = config.get("rope_scaling") or {}
        factor = float(rs["factor"]) if rs.get("type") == "linear" and "factor" in rs else 1.0     # Qwen3.swift:177-188
        return _ffi.Qwen3LMConfig(
            config["hidden_size"], config["num_hidden_layers"], config["intermediate_size"], config["num_attention_heads"],
            config["num_key_value_heads"], config["head_dim"], config["vocab_size"], config["rms_norm_eps"],
            float(config.get("rope_theta") or 1_000_000.0), factor, int(config.get("tie_word_embeddings", False)),
            int(config.get("max_position_embeddings", 32768)), int(config.get("sample_rate", 24000)),
            int(config.get("eos_token_id", 151645)), max_batch, max_context)

    @classmethod
    def config_from_json(cls, path, max_batch: int = 8, max_context: int = 2048):
        """b2a_qwen3_lm_config_from_json: (the C struct with the reference's defaults, quantisation group size, bits)."""
        import ctypes as C
        c, gs, bits = _ffi.Qwen3LMConfig(), C.c_int32(0), C.c_int32(0)
        _ffi.check(_ffi.lib().b2a_qwen3_lm_config_from_json(str(path).encode(), max_batch, max_context, C.byref(c), C.byref(gs),
                                                            C.byref(bits)))
        return c, gs.value, bits.value
