"""Host-side mirror of Qwen3-TTS's autoregressive half (SURVEY.md section 8f row N1) over the C ABI:
`Qwen3TTSTalkerForConditionalGeneration` + `Qwen3TTSCodePredictor` + the frame loop / `sampleToken` of `Qwen3TTSModel.generate`
(Sources/MLXAudioTTS/Models/Qwen3TTS/{Qwen3TTSTalker,Qwen3TTSCodePredictor,Qwen3TTS}.swift).  Every number comes from the library
(`b2a_qwen3_talker_*`); this file only composes the prompt rows the way `prepareGenerationInputs` does (Qwen3TTS.swift:883-999) and
chains the speech-tokenizer decoder for audio; `prepare_icl_generation_inputs` composes the voice-cloning (ICL) prompt from
reference codes (Qwen3TTS.swift:694-837), and `Qwen3TTSModel.prepare_reference_conditioning` builds it from reference audio with the
speech tokenizer's encoder and the speaker encoder (`Qwen3TTSSpeakerEncoder`, the x-vector of a Base checkpoint).  Tokenisation
stays with the host tokenizer: the entry points take token ids."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Callable, Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np

from . import _ffi
from .llama_tts import AudioGenerationInfo


@dataclass
class Qwen3CodePredictorConfig:
    """Qwen3TTSConfig.swift:45-63."""
    vocab_size: int = 2048
    hidden_size: int = 1024
    intermediate_size: int = 3072
    num_hidden_layers: int = 5
    num_attention_heads: int = 16
    num_key_value_heads: int = 8
    head_dim: int = 128
    rms_norm_eps: float = 1e-6
    rope_theta: float = 1_000_000.0
    num_code_groups: int = 16


@dataclass
class Qwen3TalkerConfig:
    """Qwen3TTSConfig.swift:268-292."""
    vocab_size: int = 3072
    hidden_size: int = 1024
    intermediate_size: int = 3072
    num_hidden_layers: int = 28
    num_attention_heads: int = 16
    num_key_value_heads: int = 8
    head_dim: int = 128
    rms_norm_eps: float = 1e-6
    rope_theta: float = 1_000_000.0
    num_code_groups: int = 16
    text_hidden_size: int = 2048
    text_vocab_size: int = 151936
    codec_eos_token_id: int = 2150
    code_predictor: Qwen3CodePredictorConfig = field(default_factory=Qwen3CodePredictorConfig)
    # special ids of the codec prefix (Qwen3TTSConfig.swift:294-300)
    codec_think_id: int = 2154
    codec_nothink_id: int = 2155
    codec_think_bos_id: int = 2156
    codec_think_eos_id: int = 2157
    codec_pad_id: int = 2148
    codec_bos_id: int = 2149
    # config.json's top-level "tts_model_type" ("base" checkpoints clone voices from an x-vector, Qwen3TTS.swift:709-750)
    tts_model_type: str = ""

    def _c(self, max_batch: int, max_context: int) -> _ffi.Qwen3TalkerConfig:
        cp = self.code_predictor
        return _ffi.Qwen3TalkerConfig(self.vocab_size, self.hidden_size, self.intermediate_size, self.num_hidden_layers,
                                      self.num_attention_heads, self.num_key_value_heads, self.head_dim, self.rms_norm_eps, self.rope_theta,
                                      self.num_code_groups, self.text_hidden_size, self.text_vocab_size, self.codec_eos_token_id,
                                      cp.vocab_size, cp.hidden_size, cp.intermediate_size, cp.num_hidden_layers, cp.num_attention_heads,
                                      cp.num_key_value_heads, cp.head_dim, cp.rms_norm_eps, cp.rope_theta, max_batch, max_context)


@dataclass
class Qwen3GenerateParameters:
    """Qwen3TTSModel.defaultGenerationParameters + sampleToken's arguments (Qwen3TTS.swift:360-385, 1003-1118)."""
    max_tokens: int = 4096
    temperature: float = 0.9
    top_p: float = 1.0
    top_k: int = 50
    min_p: float = 0.0
    repetition_penalty: float = 1.05
    seed: int = 0
    mask_eos: bool = False          # benchmark only (b2a_qwen3_talker_set_bench_flags, include/b200audio_internal.h)

    def _c(self) -> _ffi.Qwen3GenParams:
        return _ffi.Qwen3GenParams(self.max_tokens, self.temperature, self.top_p, self.top_k, self.min_p, self.repetition_penalty, self.seed)


@dataclass
class Qwen3SpeakerEncoderConfig:
    """Qwen3TTSSpeakerEncoderConfig (Qwen3TTSConfig.swift:92-103: same keys, same defaults)."""
    mel_dim: int = 128
    enc_dim: int = 1024
    enc_channels: List[int] = field(default_factory=lambda: [512, 512, 512, 512, 1536])
    enc_kernel_sizes: List[int] = field(default_factory=lambda: [5, 3, 3, 3, 1])
    enc_dilations: List[int] = field(default_factory=lambda: [1, 2, 3, 4, 1])
    enc_attention_channels: int = 128
    enc_res2net_scale: int = 8
    enc_se_channels: int = 128
    sample_rate: int = 24000

    def to_ffi(self) -> _ffi.Qwen3SpeakerEncoderConfig:
        n = len(self.enc_channels)
        if len(self.enc_kernel_sizes) != n or len(self.enc_dilations) != n:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "enc_channels, enc_kernel_sizes and enc_dilations must have the same length")
        if n > 8:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "at most 8 speaker-encoder layers")
        c = _ffi.Qwen3SpeakerEncoderConfig()
        for name in ("mel_dim", "enc_dim", "enc_attention_channels", "enc_res2net_scale", "enc_se_channels", "sample_rate"):
            setattr(c, name, int(getattr(self, name)))
        c.num_enc_layers = n
        for name in ("enc_channels", "enc_kernel_sizes", "enc_dilations"):
            for i, v in enumerate(getattr(self, name)):
                getattr(c, name)[i] = int(v)
        return c

    @classmethod
    def from_ffi(cls, c: _ffi.Qwen3SpeakerEncoderConfig) -> "Qwen3SpeakerEncoderConfig":
        n = c.num_enc_layers
        return cls(mel_dim=c.mel_dim, enc_dim=c.enc_dim, enc_channels=list(c.enc_channels)[:n], enc_kernel_sizes=list(c.enc_kernel_sizes)[:n],
                   enc_dilations=list(c.enc_dilations)[:n], enc_attention_channels=c.enc_attention_channels,
                   enc_res2net_scale=c.enc_res2net_scale, enc_se_channels=c.enc_se_channels, sample_rate=c.sample_rate)


def random_init_speaker_encoder_weights(cfg: Qwen3SpeakerEncoderConfig, seed: int = 2468) -> Dict[str, np.ndarray]:
    """Random-init speaker-encoder weights with the reference's module keys (blocks.*, mfa.*, asp.*, fc.*; a checkpoint prefixes
    them with "speaker_encoder.") in torch layout [out, in, k]: weights N(0, 1 / fan_in), biases N(0, 0.05^2)."""
    rng = np.random.default_rng(seed)
    W: Dict[str, np.ndarray] = {}

    def conv(prefix, cout, cin, k):
        W[prefix + ".weight"] = (rng.standard_normal((cout, cin, k)) / np.sqrt(cin * k)).astype(np.float32)
        W[prefix + ".bias"] = (rng.standard_normal(cout) * 0.05).astype(np.float32)

    ch, ks, ds = cfg.enc_channels, cfg.enc_kernel_sizes, cfg.enc_dilations
    conv("blocks.0.conv", ch[0], cfg.mel_dim, ks[0])
    for i in range(1, len(ch) - 1):
        p, w = f"blocks.{i}.", ch[i] // cfg.enc_res2net_scale
        conv(p + "tdnn1.conv", ch[i], ch[i - 1], 1)
        for j in range(cfg.enc_res2net_scale - 1):
            conv(p + f"res2net_block.blocks.{j}.conv", w, w, ks[i])
        conv(p + "tdnn2.conv", ch[i], ch[i], 1)
        conv(p + "se_block.conv1", cfg.enc_se_channels, ch[i], 1)
        conv(p + "se_block.conv2", ch[i], cfg.enc_se_channels, 1)
    conv("mfa.conv", ch[-1], ch[-1], ks[-1])
    conv("asp.tdnn.conv", cfg.enc_attention_channels, 3 * ch[-1], 1)
    conv("asp.conv", ch[-1], cfg.enc_attention_channels, 1)
    conv("fc", cfg.enc_dim, 2 * ch[-1], 1)
    return W


def check_array_shape(shape) -> bool:
    """checkArrayShapeQwen3 (Qwen3TTSSpeechTokenizer.swift:1445-1455): True when a 3-D conv weight already looks like MLX [out, k, in]."""
    if len(shape) != 3:
        return False
    _, d2, d3 = shape
    if d2 == 1:
        return d3 > 64
    if d3 == 1:
        return d2 <= 64
    return d2 < d3


class Qwen3TTSSpeakerEncoder:
    """Qwen3TTSSpeakerEncoder (Qwen3TTSSpeakerEncoder.swift) on the device: audio at sample_rate -> the x-vector [enc_dim].
    ``weights``: the module's keys (blocks.*, mfa.*, asp.*, fc.*; anything up to a "speaker_encoder." component is stripped) in
    torch or MLX layout -- 3-D weights go through the reference's layout rule (check_array_shape), as sanitize does."""

    def __init__(self, config: Optional[Qwen3SpeakerEncoderConfig] = None, weights: Optional[Dict] = None, device: int = 0):
        self.config = config or Qwen3SpeakerEncoderConfig()
        c = self.config.to_ffi()
        w = {}
        for k, v in (weights or {}).items():
            parts = [p for p in k.split(".") if p]
            if "speaker_encoder" in parts:
                parts = parts[parts.index("speaker_encoder") + 1:]
            v = np.asarray(v, dtype=np.float32)
            if k.endswith(".weight") and v.ndim == 3 and not check_array_shape(v.shape):
                v = v.transpose(0, 2, 1)
            if parts:
                w[".".join(parts)] = np.ascontiguousarray(v)
        self._h = C.c_void_p()
        if not w:
            raise _ffi.AudioGenerationError(_ffi.ERR_MODEL_NOT_INITIALIZED, "speaker encoder: no weights")
        table, keep = _ffi.make_tensor_table(w)
        _ffi.check(_ffi.lib().b2a_qwen3_speaker_encoder_create(device, C.byref(c), table, len(w), C.byref(self._h)))
        del keep

    @classmethod
    def from_model_directory(cls, model_dir, device: int = 0) -> "Qwen3TTSSpeakerEncoder":
        """The speaker-encoder half of Qwen3TTSModel.fromModelDirectory (Qwen3TTS.swift:46-48, 1224-1237): config.json's
        speaker_encoder_config + every *.safetensors -> sanitize -> weights on the device.  Only a Base checkpoint has one."""
        self = cls.__new__(cls)
        self._h = C.c_void_p()
        c = _ffi.Qwen3SpeakerEncoderConfig()
        _ffi.check(_ffi.lib().b2a_qwen3_speaker_encoder_config_from_json(str(model_dir).encode() + b"/config.json", C.byref(c)))
        self.config = Qwen3SpeakerEncoderConfig.from_ffi(c)
        _ffi.check(_ffi.lib().b2a_qwen3_speaker_encoder_create_from_directory(str(model_dir).encode(), device, C.byref(self._h)))
        return self

    @property
    def stream(self) -> int:
        return int(_ffi.lib().b2a_qwen3_speaker_encoder_stream(self._h) or 0)

    def frames(self, n_samples: int) -> int:
        return int(_ffi.lib().b2a_qwen3_speaker_encoder_frames(self._h, int(n_samples)))

    def embed(self, audio) -> np.ndarray:
        """audio [B, n] (or [n]) -> x-vectors [B, enc_dim]: the 1024-point log-mel and the network, both on the device."""
        a = np.ascontiguousarray(audio, dtype=np.float32)
        a = a[None] if a.ndim == 1 else a
        if a.ndim != 2:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "audio must be [batch, samples]")
        out = np.empty((a.shape[0], self.config.enc_dim), dtype=np.float32)
        _ffi.check(_ffi.lib().b2a_qwen3_speaker_encoder_embed(self._h, _ffi.ptr(a), a.shape[0], a.shape[1], _ffi.ptr(out)))
        return out

    def embed_dev(self, audio, out, stream: int = 0) -> None:
        """Device tensors (torch, contiguous float32): audio [B, n] -> out [B, enc_dim], enqueued on `stream` (0: the handle's)
        without a host synchronisation."""
        import torch
        if not (isinstance(audio, torch.Tensor) and isinstance(out, torch.Tensor) and audio.is_cuda and out.is_cuda and audio.dim() == 2
                and audio.dtype == torch.float32 and out.dtype == torch.float32 and audio.is_contiguous() and out.is_contiguous()
                and tuple(out.shape) == (audio.shape[0], self.config.enc_dim)):
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "embed_dev: audio must be float32 [B, n] and out float32 [B, enc_dim] on the device")
        _ffi.check(_ffi.lib().b2a_qwen3_speaker_encoder_embed_dev(self._h, _ffi.ptr(audio), int(audio.shape[0]), int(audio.shape[1]),
                                                                  _ffi.ptr(out), C.c_void_p(stream or None)))

    def embed_mel(self, mels) -> np.ndarray:
        """The module's own input (callAsFunction, :299-322): log-mel [B, T, mel_dim] -> [B, enc_dim]."""
        m = np.ascontiguousarray(mels, dtype=np.float32)
        m = m[None] if m.ndim == 2 else m
        if m.ndim != 3 or m.shape[2] != self.config.mel_dim:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "mels must be [batch, frames, mel_dim]")
        out = np.empty((m.shape[0], self.config.enc_dim), dtype=np.float32)
        _ffi.check(_ffi.lib().b2a_qwen3_speaker_encoder_embed_mel(self._h, _ffi.ptr(m), m.shape[0], m.shape[1], _ffi.ptr(out)))
        return out

    def __call__(self, ref_audio) -> np.ndarray:
        """extractSpeakerEmbedding (Qwen3TTS.swift:839-881): [n], [1, n], [B, n] (row 0) or [B, 1, n] (row 0) -> [enc_dim]."""
        a = np.asarray(ref_audio, dtype=np.float32)
        if a.ndim == 3 and a.shape[1] == 1:
            a = a[:, 0]
        if a.ndim == 1:
            a = a[None]
        elif a.ndim != 2:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "reference audio must be [n], [B, n] or [B, 1, n]")
        return self.embed(a[:1])[0]

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                _ffi.lib().b2a_qwen3_speaker_encoder_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:   # interpreter shutdown
            pass


FRAME_CB = C.CFUNCTYPE(None, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_int32))


class Qwen3TTSTalker:
    """Talker + code predictor behind one handle.  `weights`: the reference's keys after sanitize strips "talker."."""

    def __init__(self, config: Qwen3TalkerConfig, weights: Dict, device: int = 0, max_batch: int = 8, max_context: int = 2048):
        self.config = config
        c = config._c(max_batch, max_context)
        table, keep = _ffi.make_tensor_table(weights)
        self._h = C.c_void_p()
        _ffi.check(_ffi.lib().b2a_qwen3_talker_create(device, C.byref(c), table, len(weights), C.byref(self._h)))
        del keep

    @classmethod
    def random_init(cls, config: Qwen3TalkerConfig, device: int = 0, max_batch: int = 8, max_context: int = 2048, std: float = 0.02,
                    seed: int = 1234) -> "Qwen3TTSTalker":
        self = cls.__new__(cls)
        self.config = config
        c = config._c(max_batch, max_context)
        self._h = C.c_void_p()
        _ffi.check(_ffi.lib().b2a_qwen3_talker_create_random(device, C.byref(c), std, seed, C.byref(self._h)))
        return self

    @classmethod
    def from_model_directory(cls, model_dir, device: int = 0, max_batch: int = 8, max_context: int = 2048) -> "Qwen3TTSTalker":
        """The talker half of Qwen3TTSModel.fromModelDirectory (Qwen3TTS.swift:1136-1175): config.json + every *.safetensors ->
        sanitize ("talker." prefix) -> MLX affine de-quantisation as config.json's "quantization" says -> weights on the device, all
        inside the library.  The tokenizer and <dir>/speech_tokenizer (Qwen3TTSSpeechTokenizerDecoder.from_model_directory) stay with
        the caller."""
        self = cls.__new__(cls)
        c = _ffi.Qwen3TalkerConfig()
        _ffi.check(_ffi.lib().b2a_qwen3_talker_config_from_json(str(model_dir).encode() + b"/config.json", max_batch, max_context, C.byref(c)))
        cp = Qwen3CodePredictorConfig(vocab_size=c.cp_vocab_size, hidden_size=c.cp_hidden_size, intermediate_size=c.cp_intermediate_size,
                                      num_hidden_layers=c.cp_num_hidden_layers, num_attention_heads=c.cp_num_attention_heads,
                                      num_key_value_heads=c.cp_num_key_value_heads, head_dim=c.cp_head_dim, rms_norm_eps=c.cp_rms_norm_eps,
                                      rope_theta=c.cp_rope_theta, num_code_groups=c.num_code_groups)
        self.config = Qwen3TalkerConfig(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                                        num_hidden_layers=c.num_hidden_layers, num_attention_heads=c.num_attention_heads,
                                        num_key_value_heads=c.num_key_value_heads, head_dim=c.head_dim, rms_norm_eps=c.rms_norm_eps,
                                        rope_theta=c.rope_theta, num_code_groups=c.num_code_groups, text_hidden_size=c.text_hidden_size,
                                        text_vocab_size=c.text_vocab_size, codec_eos_token_id=c.codec_eos_token_id, code_predictor=cp)
        import json
        from pathlib import Path
        cj = Path(model_dir) / "config.json"
        self.config.tts_model_type = str(json.loads(cj.read_text()).get("tts_model_type", "")) if cj.exists() else ""
        self._h = C.c_void_p()
        _ffi.check(_ffi.lib().b2a_qwen3_talker_create_from_directory(str(model_dir).encode(), device, max_batch, max_context, C.byref(self._h)))
        return self

    @property
    def stream(self) -> int:
        return int(_ffi.lib().b2a_qwen3_talker_stream(self._h) or 0)

    # -- embeddings ------------------------------------------------------------------------------
    def embed_text(self, ids: Sequence[int]) -> np.ndarray:
        """text_projection(text_embedding(ids)) (Qwen3TTS.swift:898) -> [n, hidden]."""
        a = np.ascontiguousarray(ids, dtype=np.int32)
        out = np.empty((len(a), self.config.hidden_size), dtype=np.float32)
        _ffi.check(_ffi.lib().b2a_qwen3_talker_embed_text(self._h, _ffi.ptr(a), len(a), _ffi.ptr(out)))
        return out

    def embed_codec(self, ids: Sequence[int]) -> np.ndarray:
        a = np.ascontiguousarray(ids, dtype=np.int32)
        out = np.empty((len(a), self.config.hidden_size), dtype=np.float32)
        _ffi.check(_ffi.lib().b2a_qwen3_talker_embed_codec(self._h, _ffi.ptr(a), len(a), _ffi.ptr(out)))
        return out

    def embed_code_frames(self, codes) -> np.ndarray:
        """codecEmbedIcl's frame rows (Qwen3TTS.swift:249-265): codes [n, groups] -> [n, hidden], codec_embedding(c0) plus the code
        predictor's embeddings of c1 .. c_{groups-1} (groups < num_code_groups is the reference's `break`)."""
        a = np.ascontiguousarray(codes, dtype=np.int32)
        if a.ndim != 2 or a.shape[0] < 1:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "codes must be [frames, groups]")
        out = np.empty((a.shape[0], self.config.hidden_size), dtype=np.float32)
        _ffi.check(_ffi.lib().b2a_qwen3_talker_embed_code_frames(self._h, _ffi.ptr(a), a.shape[0], a.shape[1], _ffi.ptr(out)))
        return out

    def prepare_icl_generation_inputs(self, ref_codes, ref_chat_ids: Sequence[int], target_chat_ids: Sequence[int], tts_bos: int,
                                      tts_eos: int, tts_pad: int, language_id: Optional[int] = None,
                                      speaker_embedding=None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """prepareReferenceConditioning's id slicing + prepareICLGenerationInputs (Qwen3TTS.swift:709-837) from token ids, the
        voice-cloning prompt.  ref_codes [groups, T] or [1, groups, T] (the speech tokenizer's encode of the reference clip);
        ref_chat_ids = tokens of "<|im_start|>assistant\n{ref_text}<|im_end|>\n"; target_chat_ids = tokens of
        "<|im_start|>assistant\n{text}<|im_end|>\n<|im_start|>assistant\n"; speaker_embedding [hidden] (the x-vector;
        Qwen3TTSModel.prepare_reference_conditioning computes it from the reference audio).  Returns (input_embeds [L, H],
        trailing_text_hidden [1, H] = tts_pad, tts_pad_embed [H])."""
        c = self.config
        if speaker_embedding is None and c.tts_model_type == "base":
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "a Base checkpoint clones from a speaker embedding (x-vector): pass "
                                            "speaker_embedding, or build the prompt from audio with Qwen3TTSModel.prepare_reference_conditioning "
                                            "and a Qwen3TTSSpeakerEncoder")
        rc = np.asarray(ref_codes)
        rc = rc[0] if rc.ndim == 3 else rc
        if rc.ndim != 2 or rc.shape[1] < 1:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "ref_codes must be [groups, frames]")
        rid, tid = list(ref_chat_ids), list(target_chat_ids)
        r0 = min(3, len(rid)); ref_text = rid[r0:max(r0, len(rid) - 2)]                   # :731-735
        t0 = min(3, len(tid)); target_text = tid[t0:max(t0, len(tid) - 5)]                # :762-766
        tts = self.embed_text([tts_bos, tts_eos, tts_pad])
        bos_e, eos_e, pad_e = tts[0:1], tts[1:2], tts[2:3]
        text_ids = ref_text + target_text
        text = np.concatenate(([self.embed_text(text_ids)] if text_ids else []) + [eos_e], axis=0)            # :775-778
        codec_pad = self.embed_codec([c.codec_pad_id])
        icl_codec = np.concatenate([self.embed_codec([c.codec_bos_id]), self.embed_code_frames(rc.T[:, :min(rc.shape[0], c.num_code_groups)])], axis=0)
        icl = np.concatenate([text + codec_pad, icl_codec + pad_e], axis=0)                                   # :786-797
        prefill = ([c.codec_think_id, c.codec_think_bos_id, language_id, c.codec_think_eos_id] if language_id is not None
                   else [c.codec_nothink_id, c.codec_think_bos_id, c.codec_think_eos_id])                    # :800-812
        pieces = [self.embed_codec(prefill)]
        if speaker_embedding is not None:
            se = np.asarray(speaker_embedding, dtype=np.float32).reshape(-1)
            if se.shape[0] != c.hidden_size:
                raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "speaker_embedding must have hidden_size values")
            pieces.append(se[None])
        codec_prefix = np.concatenate(pieces + [self.embed_codec([c.codec_pad_id, c.codec_bos_id])], axis=0)   # :814-823
        role = self.embed_text(tid[0:3])                                                                       # :825
        pad_count = codec_prefix.shape[0] - 2
        combined = np.concatenate([np.repeat(pad_e, pad_count, axis=0), bos_e], axis=0) + codec_prefix[:-1]   # :827-830
        inputs = np.concatenate([role, combined, icl], axis=0)                                                 # :832
        return inputs.astype(np.float32), pad_e.astype(np.float32), pad_e[0].astype(np.float32)

    def prepare_generation_inputs(self, chat_ids: Sequence[int], tts_bos: int, tts_eos: int, tts_pad: int,
                                  language_id: Optional[int] = None, speaker_id: Optional[int] = None,
                                  instruct_ids: Optional[Sequence[int]] = None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """prepareGenerationInputs (Qwen3TTS.swift:883-999) from token ids: chat_ids = tokens of
        "<|im_start|>assistant\\n{text}<|im_end|>\\n<|im_start|>assistant\\n", instruct_ids = tokens of the VoiceDesign instruct turn.
        Returns (input_embeds [L, H], trailing_text_hidden [n, H], tts_pad_embed [H]).  Row selection / concatenation / the two
        adds are host bookkeeping; every embedding row comes from the device."""
        c = self.config
        text = self.embed_text(list(chat_ids))
        tts = self.embed_text([tts_bos, tts_eos, tts_pad])
        bos_e, eos_e, pad_e = tts[0:1], tts[1:2], tts[2:3]
        prefill = ([c.codec_think_id, c.codec_think_bos_id, language_id, c.codec_think_eos_id] if language_id is not None
                   else [c.codec_nothink_id, c.codec_think_bos_id, c.codec_think_eos_id])                          # :938-951
        ids = prefill + ([speaker_id] if speaker_id is not None else []) + [c.codec_pad_id, c.codec_bos_id]          # :957-962
        codec = self.embed_codec(ids)
        pad_count = codec.shape[0] - 2
        combined = np.concatenate([np.repeat(pad_e, pad_count, axis=0), bos_e], axis=0) + codec[:-1]               # :976-979
        pieces = ([self.embed_text(list(instruct_ids))] if instruct_ids else []) + [text[:3], combined]
        first_text = text[3:4] + codec[-1:]                                                                          # :989
        inputs = np.concatenate(pieces + [first_text], axis=0)
        trailing = np.concatenate([text[4:text.shape[0] - 5], eos_e], axis=0)                                        # :993-996
        return inputs.astype(np.float32), trailing.astype(np.float32), pad_e[0].astype(np.float32)

    # -- model -----------------------------------------------------------------------------------
    def __call__(self, input_embeds: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
        """Talker forward from an empty cache: input_embeds [B, L, H] -> (codec logits of the last position [B, V], hidden [B, H])."""
        x = np.ascontiguousarray(input_embeds, dtype=np.float32)
        if x.ndim == 2:
            x = x[None]
        B, L, H = x.shape
        logits = np.empty((B, self.config.vocab_size), dtype=np.float32)
        hidden = np.empty((B, H), dtype=np.float32)
        _ffi.check(_ffi.lib().b2a_qwen3_talker_forward(self._h, _ffi.ptr(x), B, L, _ffi.ptr(logits), _ffi.ptr(hidden)))
        return logits, hidden

    def generate_codes(self, input_embeds, trailing_text_hidden, tts_pad_embed, parameters: Optional[Qwen3GenerateParameters] = None,
                       on_frame: Optional[Callable[[int, int, np.ndarray], None]] = None):
        """The frame loop (Qwen3TTS.swift:380-495) for B utterances with the same prompt length: input_embeds [B, L, H],
        trailing_text_hidden a list of [n_b, H] arrays (or one [B, n, H] array), tts_pad_embed [H].
        Returns ([codes_b [frames_b, num_code_groups]], AudioGenerationInfo)."""
        p = parameters or Qwen3GenerateParameters()
        x = np.ascontiguousarray(input_embeds, dtype=np.float32)
        if x.ndim == 2:
            x = x[None]
        B, L, H = x.shape
        tr = [np.asarray(t, dtype=np.float32).reshape(-1, H) for t in (trailing_text_hidden if not isinstance(trailing_text_hidden, np.ndarray)
                                                                      or trailing_text_hidden.ndim == 3 else [trailing_text_hidden])]
        if len(tr) != B:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "one trailing-text block per utterance")
        nmax = max((t.shape[0] for t in tr), default=0)
        trail = np.zeros((B, max(nmax, 1), H), dtype=np.float32)
        nt = np.zeros(B, dtype=np.int32)
        for b, t in enumerate(tr):
            trail[b, :t.shape[0]] = t
            nt[b] = t.shape[0]
        pad = np.ascontiguousarray(tts_pad_embed, dtype=np.float32).reshape(H)
        G = self.config.num_code_groups
        codes = np.zeros((B, p.max_tokens, G), dtype=np.int32)
        nfr = np.zeros(B, dtype=np.int32)
        info = _ffi.GenInfo()
        gp = p._c()
        _ffi.check(_ffi.lib().b2a_qwen3_talker_set_bench_flags(self._h, int(p.mask_eos)))
        cb = (FRAME_CB(lambda user, b, f, c: on_frame(b, f, np.ctypeslib.as_array(c, shape=(G,)).copy())) if on_frame else FRAME_CB())
        _ffi.check(_ffi.lib().b2a_qwen3_talker_generate(self._h, _ffi.ptr(x), B, L, _ffi.ptr(trail), _ffi.ptr(nt), nmax, _ffi.ptr(pad), C.byref(gp),
                                                        _ffi.ptr(codes), _ffi.ptr(nfr), C.byref(info), cb, None))
        gi = AudioGenerationInfo(info.prompt_token_count, info.generation_token_count, info.prefill_time, info.generate_time,
                                 info.tokens_per_second, info.peak_memory_gb, info.codec_time)
        return [codes[b, :nfr[b]].copy() for b in range(B)], gi

    def cancel(self) -> None:
        _ffi.check(_ffi.lib().b2a_qwen3_talker_cancel(self._h))

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                _ffi.lib().b2a_qwen3_talker_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:   # interpreter shutdown
            pass


class Qwen3TTSModel:
    """SpeechGenerationModel face of Qwen3-TTS (Qwen3TTS.swift:306-569): talker + code predictor -> codes -> speech-tokenizer
    decoder.  `speech_tokenizer` is a qwen3_tts_codec.Qwen3TTSSpeechTokenizer (borrowed; its encoder, when present, turns reference
    audio into codes); `speaker_encoder` a Qwen3TTSSpeakerEncoder (borrowed; a Base checkpoint's x-vector)."""
    sample_rate = 24000

    def __init__(self, talker: Qwen3TTSTalker, speech_tokenizer=None, speaker_encoder: Optional[Qwen3TTSSpeakerEncoder] = None):
        self.talker, self.speech_tokenizer, self.speaker_encoder = talker, speech_tokenizer, speaker_encoder

    def prepare_reference_conditioning(self, ref_audio, ref_chat_ids: Sequence[int], target_chat_ids: Sequence[int], tts_bos: int,
                                       tts_eos: int, tts_pad: int, language_id: Optional[int] = None):
        """The voice-cloning prompt from reference audio: referenceAudioContext + prepareReferenceConditioning +
        prepareICLGenerationInputs (Qwen3TTS.swift:267-300, 709-837).  ref_audio [n], [B, n] or [B, 1, n] at 24 kHz is encoded to
        codes by the speech tokenizer's encoder and, with a speaker encoder, to the x-vector (extractSpeakerEmbedding: row 0).
        The token ids are prepare_icl_generation_inputs'.  Returns (input_embeds, trailing_text_hidden, tts_pad_embed, ref_codes),
        ready for generate(..., ref_codes=ref_codes)."""
        if self.speech_tokenizer is None or not self.speech_tokenizer.has_encoder:
            raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "Qwen3TTS reference conditioning requires a speech tokenizer encoder")
        a = np.asarray(ref_audio, dtype=np.float32)
        codes = self.speech_tokenizer.encode(a)                               # referenceAudioForEncoder's shapes (:239-247)
        xvec = self.speaker_encoder(a) if self.speaker_encoder is not None else None
        ref_codes = codes[0]
        inputs, trailing, pad = self.talker.prepare_icl_generation_inputs(ref_codes, ref_chat_ids, target_chat_ids, tts_bos, tts_eos, tts_pad,
                                                                          language_id=language_id, speaker_embedding=xvec)
        return inputs, trailing, pad, ref_codes

    def generate(self, input_embeds, trailing_text_hidden, tts_pad_embed, parameters: Optional[Qwen3GenerateParameters] = None,
                 ref_codes=None) -> np.ndarray:
        """generate (:412-510) after prepare_generation_inputs / prepare_icl_generation_inputs: one utterance -> 1-D waveform (chunked
        decode, :1059-1068).  With ref_codes [groups, T] (or [1, groups, T]; a voice-cloning prompt), the reference codes are decoded in
        front of the generated ones and the first int(T / total_frames * samples) samples are cut off (:550-565)."""
        if self.speech_tokenizer is None:
            raise _ffi.AudioGenerationError(_ffi.ERR_MODEL_NOT_INITIALIZED, "speech tokenizer not loaded")
        codes, _ = self.talker.generate_codes(np.asarray(input_embeds)[None], [trailing_text_hidden], tts_pad_embed, parameters)
        if codes[0].shape[0] == 0:
            raise _ffi.AudioGenerationError(_ffi.ERR_GENERATION_FAILED, "No audio codes generated")
        frames = codes[0]
        if ref_codes is not None:
            rc = np.asarray(ref_codes, dtype=np.int32)
            rc = rc[0] if rc.ndim == 3 else rc
            if rc.ndim != 2 or rc.shape[0] != frames.shape[1]:
                raise _ffi.AudioGenerationError(_ffi.ERR_INVALID_INPUT, "ref_codes must be [num_code_groups, frames]")
            frames = np.concatenate([rc.T, frames], axis=0)
        wav, lengths = self.speech_tokenizer.decode(frames[None])
        audio = wav[0, :int(lengths[0])] if 0 < int(lengths[0]) < wav.shape[1] else wav[0]
        if ref_codes is not None:
            cut = int(rc.shape[1] / max(frames.shape[0], 1) * audio.shape[0])
            if 0 < cut < audio.shape[0]:
                audio = audio[cut:]
        return audio

    def generate_stream(self, input_embeds, trailing_text_hidden, tts_pad_embed, parameters: Optional[Qwen3GenerateParameters] = None,
                        streaming_interval: float = 2.0, ref_codes=None) -> Iterator:
        """generateStream (:512-569): audio chunks DURING generation -- every int(streaming_interval * 12.5) frames the new codes go
        through the speech tokenizer's streaming step (decodeChunk -> streamingDecode, Qwen3TTS.swift:214-231) and are yielded as
        ('audio', samples); ('token', c0) per frame, ('info', ...) at the end.  A voice-cloning prompt streams only the generated
        codes: like the reference's streaming path (:532-545), ref_codes are not decoded in front, so there is nothing to cut."""
        if self.speech_tokenizer is None:
            raise _ffi.AudioGenerationError(_ffi.ERR_MODEL_NOT_INITIALIZED, "speech tokenizer not loaded")
        chunk = max(1, int(streaming_interval * 12.5))
        dec = self.speech_tokenizer.decoder
        dec.reset_streaming_state()
        events: List = []
        pending: List[np.ndarray] = []

        def flush():
            if pending:
                c = np.stack(pending)[None].transpose(0, 2, 1)                # [1, G, n]
                events.append(("audio", dec.streaming_step(np.ascontiguousarray(c))[0, 0]))
                pending.clear()

        def on_frame(b, f, c):
            events.append(("token", int(c[0])))
            pending.append(c)
            if len(pending) >= chunk:
                flush()

        _, info = self.talker.generate_codes(np.asarray(input_embeds)[None], [trailing_text_hidden], tts_pad_embed, parameters, on_frame=on_frame)
        flush()
        yield from events
        yield ("info", info)
