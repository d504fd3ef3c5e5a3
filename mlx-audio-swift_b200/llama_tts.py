"""Host-side mirror of `LlamaTTSModel` (Sources/MLXAudioTTS/Models/Llama/LlamaTTS.swift:354-977) behind
SpeechGenerationModel (Sources/MLXAudioTTS/Generation.swift:8-39), over the C ABI.  Tokenisation stays
with the host (SURVEY.md section 8b): `generate` takes token ids."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Callable, Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np

from . import _ffi
from .snac import SNAC

START_OF_HUMAN, END_OF_HUMAN, END_OF_TEXT = 128259, 128260, 128009
START_OF_SPEECH, END_OF_SPEECH, PAD_TOKEN = 128257, 128258, 128263
AUDIO_TOKEN_OFFSET = 128266


@dataclass
class GenerateParameters:
    """defaultGenerationParameters, LlamaTTS.swift:573-581."""
    max_tokens: int = 1200
    temperature: float = 0.6
    top_p: float = 0.8
    repetition_penalty: float = 1.3
    repetition_context_size: int = 20
    seed: int = 0
    mask_eos: bool = False      # benchmark only
    wrap_codes: bool = False    # benchmark only

    def _c(self) -> _ffi.GenParams:
        return _ffi.GenParams(self.max_tokens, self.temperature, self.top_p, self.repetition_penalty,
                              self.repetition_context_size, self.seed)


@dataclass
class AudioGenerationInfo:
    """GenerationTypes.swift:14-45."""
    prompt_token_count: int
    generation_token_count: int
    prefill_time: float
    generate_time: float
    tokens_per_second: float
    peak_memory_usage: float
    codec_time: float = 0.0


class LlamaTTSModel:
    sample_rate = 24000
    default_generation_parameters = GenerateParameters()
    _abi = "b2a_tts"            # prefix of the constructors, prompt framing and parse entry points of this model's token layout
    _pad_token = PAD_TOKEN

    @staticmethod
    def _c_config(config: dict, max_batch: int, max_context: int) -> _ffi.LlamaConfig:
        rs = config.get("rope_scaling") or {}
        nh = config["num_attention_heads"]
        return _ffi.LlamaConfig(
            config["hidden_size"], config["num_hidden_layers"], config["intermediate_size"], nh,
            config.get("num_key_value_heads", nh), config.get("head_dim") or config["hidden_size"] // nh,
            config["vocab_size"], config["rms_norm_eps"], config.get("rope_theta", 10000.0),
            float(rs.get("factor", 32.0)), float(rs.get("low_freq_factor", 1.0)), float(rs.get("high_freq_factor", 4.0)),
            float(rs.get("original_max_position_embeddings", 8192.0)), int(config.get("tie_word_embeddings", True)),
            max_batch, max_context)

    @classmethod
    def random_init(cls, config: dict, snac: Optional[SNAC] = None, device: int = 0, max_batch: int = 8,
                    max_context: int = 2048, std: float = 0.02, seed: int = 1234) -> "LlamaTTSModel":
        """Random-init weights drawn on the device (benchmarks / full-size property tests)."""
        self = cls.__new__(cls)
        c = cls._c_config(config, max_batch, max_context)
        self.config, self.vocab_size, self._snac_model = config, config["vocab_size"], snac
        self._h = C.c_void_p()
        _ffi.check(getattr(_ffi.lib(), cls._abi + "_create_random")(device, C.byref(c), std, seed, snac._h if snac else None,
                                                                    C.byref(self._h)))
        return self

    @property
    def stream(self) -> int:
        return int(_ffi.lib().b2a_tts_stream(self._h) or 0)

    def debug_trace(self, enable: bool, batch: int = 0, read: bool = False):
        """Parity hook: residual stream at every RMSNorm input for the last traced forward position."""
        out = None
        if read:
            out = np.empty((2 * self.config["num_hidden_layers"] + 1, batch, self.config["hidden_size"]), dtype=np.float32)
        _ffi.check(_ffi.lib().b2a_tts_debug_trace(self._h, int(enable), batch, _ffi.ptr(out)))
        return out

    def time_steps(self, batch: int, ctx: int, iters: int) -> float:
        """Average device milliseconds of one captured decode step (CUDA events on the handle's stream)."""
        ms = C.c_float(0)
        _ffi.check(_ffi.lib().b2a_tts_time_steps(self._h, batch, ctx, iters, C.byref(ms)))
        return float(ms.value)

    def __init__(self, config: dict, weights: Dict, snac: Optional[SNAC] = None, device: int = 0,
                 max_batch: int = 8, max_context: int = 2048):
        c = self._c_config(config, max_batch, max_context)
        self.config, self.vocab_size, self._snac_model = config, config["vocab_size"], snac
        weights = {k: v for k, v in weights.items() if "rotary_emb.inv_freq" not in k}      # sanitize (:583-593)
        if c.tie_word_embeddings:
            weights.pop("lm_head.weight", None)
        table, keep = _ffi.make_tensor_table(weights)
        self._h = C.c_void_p()
        _ffi.check(getattr(_ffi.lib(), self._abi + "_create")(device, C.byref(c), table, len(weights), snac._h if snac else None,
                                                              C.byref(self._h)))
        del keep

    @classmethod
    def from_model_directory(cls, model_dir, snac: Optional[SNAC] = None, device: int = 0, max_batch: int = 8,
                             max_context: int = 2048) -> "LlamaTTSModel":
        """fromModelDirectory (LlamaTTS.swift:942-977): config.json + every *.safetensors -> sanitize -> MLX affine de-quantisation ->
        weights on the device, all inside the library (b2a_tts_create_from_directory).  The tokenizer and the SNAC download of
        post_load_hook (:595-602) stay with the host: pass `snac`."""
        import json
        from pathlib import Path
        self = cls.__new__(cls)
        self.config = json.loads((Path(model_dir) / "config.json").read_text())
        self.vocab_size, self._snac_model = self.config.get("vocab_size", 0), snac      # a bad config.json is the library's error to raise
        self._h = C.c_void_p()
        _ffi.check(getattr(_ffi.lib(), cls._abi + "_create_from_directory")(str(model_dir).encode(), device, max_batch, max_context,
                                                                            snac._h if snac else None, C.byref(self._h)))
        return self

    # -- token plumbing -------------------------------------------------------------------------
    @classmethod
    def prepare_input_ids(cls, prompt_token_ids: Sequence[Sequence[int]], ref_code_list: Optional[Sequence[int]] = None,
                          ref_text_ids: Optional[Sequence[int]] = None) -> Tuple[np.ndarray, np.ndarray]:
        """prepareInputIds (:446-553) on already-tokenised prompts.  With both `ref_code_list` (the 7-token interleaved codes
        of a reference clip, `encode_audio_to_code_list`) and `ref_text_ids` (its tokenised transcript) every row gets the
        voice-cloning reference block between its padding and its prompt; with either missing the prompts are framed alone."""
        B = len(prompt_token_ids)
        rows = [np.ascontiguousarray(p, dtype=np.int32) for p in prompt_token_ids]
        lens = np.asarray([len(r) for r in rows], dtype=np.int32)
        pp = (C.c_void_p * B)(*[r.ctypes.data for r in rows])
        n = C.c_int32(0)
        if ref_code_list is None or ref_text_ids is None:
            fn, extra = getattr(_ffi.lib(), cls._abi + "_prepare_input_ids"), ()
        else:
            rc = np.ascontiguousarray(ref_code_list, dtype=np.int32).reshape(-1)
            rt = np.ascontiguousarray(ref_text_ids, dtype=np.int32).reshape(-1)
            fn, extra = getattr(_ffi.lib(), cls._abi + "_prepare_input_ids_ref"), (_ffi.ptr(rt), len(rt), _ffi.ptr(rc), len(rc))
        _ffi.check(fn(pp, _ffi.ptr(lens), B, *extra, None, C.byref(n)))
        out = np.empty((B, n.value), dtype=np.int32)
        _ffi.check(fn(pp, _ffi.ptr(lens), B, *extra, _ffi.ptr(out), C.byref(n)))
        return out, out != cls._pad_token

    def encode_audio_to_code_list(self, audio) -> List[int]:
        """llamaEncodeAudioToCodes (:72-98): a 1-D reference clip at 24 kHz -> SNAC codes on the device -> 7-token interleave."""
        if self._snac_model is None:
            raise _ffi.AudioGenerationError(_ffi.ERR_MODEL_NOT_INITIALIZED, "SNAC model not loaded")
        codes = self._snac_model.encode(np.asarray(audio, dtype=np.float32).reshape(1, 1, -1))
        return self.code_list_from_codes(codes)

    def _prompt_ids(self, prompt_token_ids, ref_audio, ref_text_ids):
        # cloning applies only when both the reference audio and its transcript are given (:456)
        if ref_audio is not None and ref_text_ids is not None:
            return self.prepare_input_ids([list(prompt_token_ids)], self.encode_audio_to_code_list(ref_audio), ref_text_ids)[0]
        return self.prepare_input_ids([list(prompt_token_ids)])[0]

    @classmethod
    def parse_output(cls, input_ids) -> List[List[int]]:
        """parseOutput (:383-434)."""
        ids = np.ascontiguousarray(input_ids, dtype=np.int32)
        B, n = ids.shape
        out = np.empty((B, max(n, 1)), dtype=np.int32)
        lens = np.empty(B, dtype=np.int32)
        _ffi.check(getattr(_ffi.lib(), cls._abi + "_parse_output")(_ffi.ptr(ids), B, n, _ffi.ptr(out), _ffi.ptr(lens)))
        return [out[b, :lens[b]].tolist() for b in range(B)]

    @staticmethod
    def codes_from_code_list(code_list: Sequence[int]) -> List[np.ndarray]:
        """llamaDecodeAudioFromCodes' de-interleave (:41-63) -> 3 layers [1, T_i]."""
        cl = np.ascontiguousarray(code_list, dtype=np.int32)
        g = (len(cl) + 1) // 7
        c0, c1, c2 = (np.empty(k * g, dtype=np.int32) for k in (1, 2, 4))
        nf = C.c_int32(0)
        _ffi.check(_ffi.lib().b2a_tts_deinterleave(_ffi.ptr(cl), len(cl), _ffi.ptr(c0), _ffi.ptr(c1), _ffi.ptr(c2), C.byref(nf)))
        return [c0[None], c1[None], c2[None]]

    @staticmethod
    def code_list_from_codes(codes: Sequence[np.ndarray]) -> List[int]:
        """llamaEncodeAudioToCodes' interleave (:72-98)."""
        c0, c1, c2 = (np.ascontiguousarray(np.asarray(c).reshape(-1), dtype=np.int32) for c in codes)
        out = np.empty(7 * len(c0), dtype=np.int32)
        _ffi.check(_ffi.lib().b2a_tts_interleave(_ffi.ptr(c0), _ffi.ptr(c1), _ffi.ptr(c2), len(c0), _ffi.ptr(out)))
        return out.tolist()

    # -- forward / generate ----------------------------------------------------------------------
    def __call__(self, input_ids, reset_cache: bool = True) -> np.ndarray:
        """callAsFunction(_:cache:) (:557-567): ids [B, L] -> logits [B, L, V]."""
        ids = np.ascontiguousarray(input_ids, dtype=np.int32)
        B, L = ids.shape
        out = np.empty((B, L, self.vocab_size), dtype=np.float32)
        _ffi.check(_ffi.lib().b2a_tts_forward_logits(self._h, _ffi.ptr(ids), B, L, int(reset_cache), _ffi.ptr(out)))
        return out

    def _params(self, p: GenerateParameters) -> _ffi.GenParams:
        # mask_eos / wrap_codes are benchmark switches on the handle (include/b200audio_internal.h), not part of GenerateParameters' ABI struct
        _ffi.check(_ffi.lib().b2a_tts_set_bench_flags(self._h, int(p.mask_eos), int(p.wrap_codes)))
        return p._c()

    def generate_batch(self, input_ids, parameters: Optional[GenerateParameters] = None, decode_audio: bool = True,
                       on_token: Optional[Callable[[int, int, int], None]] = None):
        """B independent utterances through generate (:658-765).  Returns (tokens [list per row],
        waveforms [list of 1-D float32 or None], AudioGenerationInfo)."""
        p = parameters or self.default_generation_parameters
        ids = np.ascontiguousarray(input_ids, dtype=np.int32)
        B, L = ids.shape
        toks = np.zeros((B, p.max_tokens), dtype=np.int32)
        ntok = np.zeros(B, dtype=np.int32)
        hop = self._snac_model.hop_length if self._snac_model else 0
        cap = 4 * ((L + p.max_tokens) // 7 + 1) * hop if decode_audio else 0
        wave = np.empty((B, cap), dtype=np.float32) if decode_audio else None
        wlen = np.zeros(B, dtype=np.int64)
        info = _ffi.GenInfo()
        gp = self._params(p)
        cb = _ffi.TOKEN_CB(lambda user, b, step, tok: on_token(b, step, tok)) if on_token else _ffi.TOKEN_CB()
        _ffi.check(_ffi.lib().b2a_tts_generate(self._h, _ffi.ptr(ids), B, L, C.byref(gp), _ffi.ptr(toks), _ffi.ptr(ntok),
                                               _ffi.ptr(wave), cap, _ffi.ptr(wlen), C.byref(info), cb, None))
        tokens = [toks[b, :ntok[b]].tolist() for b in range(B)]
        waves = [wave[b, :wlen[b]].copy() if decode_audio and wlen[b] > 0 else None for b in range(B)]
        gi = AudioGenerationInfo(info.prompt_token_count, info.generation_token_count, info.prefill_time,
                                 info.generate_time, info.tokens_per_second, info.peak_memory_gb, info.codec_time)
        return tokens, waves, gi

    def generate_into(self, ids, parameters: GenerateParameters, tokens, n_tokens, wave, wave_len):
        """Zero-allocation form of generate_batch for callers that own (pinned) host buffers: `ids` [B, L]
        int32, `tokens` [B, max_tokens] int32, `n_tokens` [B] int32, `wave` [B, cap] float32, `wave_len` [B]
        int64 -- numpy arrays or torch CPU tensors.  Returns AudioGenerationInfo."""
        B, L = ids.shape
        info = _ffi.GenInfo()
        gp = self._params(parameters)
        cap = wave.shape[1] if wave is not None else 0
        _ffi.check(_ffi.lib().b2a_tts_generate(self._h, _ffi.ptr(ids), B, L, C.byref(gp), _ffi.ptr(tokens), _ffi.ptr(n_tokens),
                                               _ffi.ptr(wave), cap, _ffi.ptr(wave_len), C.byref(info), _ffi.TOKEN_CB(), None))
        return AudioGenerationInfo(info.prompt_token_count, info.generation_token_count, info.prefill_time,
                                   info.generate_time, info.tokens_per_second, info.peak_memory_gb, info.codec_time)

    def generate(self, prompt_token_ids: Sequence[int], parameters: Optional[GenerateParameters] = None, ref_audio=None,
                 ref_text_ids: Optional[Sequence[int]] = None) -> np.ndarray:
        """generate(text:voice:refAudio:refText:...) (:658-765) for ONE utterance, after tokenisation: returns the 1-D waveform.
        `ref_audio` (1-D, 24 kHz) with `ref_text_ids` clones the reference voice (prepareInputIds, :446-553)."""
        if self._snac_model is None:
            raise _ffi.AudioGenerationError(_ffi.ERR_MODEL_NOT_INITIALIZED, "SNAC model not loaded")
        ids = self._prompt_ids(prompt_token_ids, ref_audio, ref_text_ids)
        _, waves, _ = self.generate_batch(ids, parameters)
        return waves[0]

    def generate_audio_chunks(self, input_ids, parameters: Optional[GenerateParameters] = None, frames_per_chunk: int = 4,
                              left_context_frames: int = 8, on_audio: Optional[Callable[[int, np.ndarray, bool], None]] = None,
                              on_token: Optional[Callable[[int, int, int], None]] = None):
        """Row N2: audio DURING generation (b2a_tts_generate_stream).  Every `frames_per_chunk` new 7-token frames of a row are
        decoded by SNAC with `left_context_frames` already-emitted frames in front and passed to on_audio(row, samples, is_final)
        from inside the call.  Returns (tokens, [chunk list per row], AudioGenerationInfo)."""
        p = parameters or self.default_generation_parameters
        ids = np.ascontiguousarray(input_ids, dtype=np.int32)
        B, L = ids.shape
        toks = np.zeros((B, p.max_tokens), dtype=np.int32)
        ntok = np.zeros(B, dtype=np.int32)
        info = _ffi.GenInfo()
        gp = self._params(p)
        chunks: List[List[np.ndarray]] = [[] for _ in range(B)]

        def audio(user, b, ptr, n, final):
            a = np.ctypeslib.as_array(ptr, shape=(n,)).copy()
            chunks[b].append(a)
            if on_audio:
                on_audio(b, a, bool(final))

        acb = _ffi.AUDIO_CB(audio)
        tcb = _ffi.TOKEN_CB(lambda user, b, step, tok: on_token(b, step, tok)) if on_token else _ffi.TOKEN_CB()
        _ffi.check(_ffi.lib().b2a_tts_generate_stream(self._h, _ffi.ptr(ids), B, L, C.byref(gp), frames_per_chunk, left_context_frames,
                                                      _ffi.ptr(toks), _ffi.ptr(ntok), C.byref(info), tcb, acb, None))
        gi = AudioGenerationInfo(info.prompt_token_count, info.generation_token_count, info.prefill_time, info.generate_time,
                                 info.tokens_per_second, info.peak_memory_gb, info.codec_time)
        return [toks[b, :ntok[b]].tolist() for b in range(B)], chunks, gi

    def generate_stream(self, prompt_token_ids: Sequence[int], parameters: Optional[GenerateParameters] = None,
                        streaming_interval: Optional[float] = None, ref_audio=None,
                        ref_text_ids: Optional[Sequence[int]] = None) -> Iterator:
        """generateStream (:777-913): yields ('token', id)..., ('info', AudioGenerationInfo), ('audio', waveform).  With
        streaming_interval = None the audio comes once, at the end, as the reference's Orpheus does (the protocol's default overload
        ignores the interval for such models, Generation.swift:119-137); with a float (seconds) ('audio', chunk) events are produced
        every round(interval * 24000 / 2048) frames while tokens are still being generated (row N2).  `ref_audio` with
        `ref_text_ids` clones the reference voice, as in generate."""
        if self._snac_model is None:
            raise _ffi.AudioGenerationError(_ffi.ERR_MODEL_NOT_INITIALIZED, "SNAC model not loaded")
        ids = self._prompt_ids(prompt_token_ids, ref_audio, ref_text_ids)
        if streaming_interval is not None:
            events = []
            fpc = max(1, int(round(streaming_interval * 24000.0 / 2048.0)))
            _, _, info = self.generate_audio_chunks(ids, parameters, frames_per_chunk=fpc,
                                                    on_audio=lambda b, a, fin: events.append(("audio", a)),
                                                    on_token=lambda b, s, t: events.append(("token", t)))
            yield from events
            yield ("info", info)
            return
        events = []
        _, waves, info = self.generate_batch(ids, parameters, on_token=lambda b, s, t: events.append(("token", t)))
        yield from events
        yield ("info", info)
        yield ("audio", waves[0])

    def generate_samples_stream(self, prompt_token_ids: Sequence[int], parameters: Optional[GenerateParameters] = None,
                                streaming_interval: Optional[float] = None, ref_audio=None,
                                ref_text_ids: Optional[Sequence[int]] = None) -> Iterator[np.ndarray]:
        """generateSamplesStream (Generation.swift:52-74): only the .audio events of generateStream, as sample arrays."""
        for kind, value in self.generate_stream(prompt_token_ids, parameters, streaming_interval, ref_audio, ref_text_ids):
            if kind == "audio" and value is not None:
                yield value

    def generate_dev(self, d_input_ids, parameters: GenerateParameters, d_wave, wave_cap: int):
        """Device-resident variant (bench `value`): torch CUDA int32 ids [B, L]; waveform stays in HBM."""
        B, L = d_input_ids.shape
        wlen = np.zeros(B, dtype=np.int64)
        info = _ffi.GenInfo()
        gp = self._params(parameters)
        _ffi.check(_ffi.lib().b2a_tts_generate_dev(self._h, _ffi.ptr(d_input_ids), B, L, C.byref(gp), _ffi.ptr(d_wave),
                                                   wave_cap, _ffi.ptr(wlen), C.byref(info)))
        return wlen, AudioGenerationInfo(info.prompt_token_count, info.generation_token_count, info.prefill_time,
                                         info.generate_time, info.tokens_per_second, info.peak_memory_gb, info.codec_time)

    def cancel(self) -> None:
        _ffi.check(_ffi.lib().b2a_tts_cancel(self._h))

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                _ffi.lib().b2a_tts_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:   # interpreter shutdown: ctypes globals may already be gone
            pass
