"""Host-side mirror of `SopranoModel` (Sources/MLXAudioTTS/Models/Soprano/Soprano.swift:184-977) behind SpeechGenerationModel, over the
C ABI.  The handle is a b2a_tts one (b2a_soprano_create*) that owns a Vocos decoder: the decode step captures every row's final-norm hidden
state on the device and the decoder turns them into audio (SopranoDecoder.swift:222-285).  Text cleaning, sentence splitting and
tokenisation stay with the caller: prompts are token ids, one prompt per `[STOP][TEXT]...[START]` sentence."""
from __future__ import annotations

import ctypes as C
from typing import Callable, Dict, Iterator, List, Optional, Sequence, Union

import numpy as np

from . import _ffi
from .llama_tts import AudioGenerationInfo, GenerateParameters

Prompt = Sequence[int]


def _info(info: _ffi.GenInfo) -> AudioGenerationInfo:
    return AudioGenerationInfo(info.prompt_token_count, info.generation_token_count, info.prefill_time, info.generate_time,
                               info.tokens_per_second, info.peak_memory_gb, info.codec_time)


class SopranoModel:
    """Soprano: a Qwen3 language model whose final-norm hidden states a Vocos decoder turns into 32 kHz audio.  `config` is the
    checkpoint's config.json as a dict (SopranoConfiguration, SopranoConfig.swift:65-176; head_dim must be 128)."""
    default_generation_parameters = GenerateParameters(max_tokens=1200, temperature=0.7, top_p=0.95, repetition_penalty=1.5,
                                                       repetition_context_size=30)    # Soprano.swift:577-587
    default_stream_parameters = GenerateParameters(max_tokens=512, temperature=0.3, top_p=0.95, repetition_penalty=1.5,
                                                   repetition_context_size=30)        # Soprano.swift:693-702

    @staticmethod
    def _c_config(config: dict, max_batch: int, max_context: int, repo: Optional[str] = None, stop_token_id: int = 3) -> _ffi.SopranoConfig:
        """SopranoConfiguration's defaults, then fromModelDirectory's decoder rule (:934-941) when `repo` is given."""
        g = config.get
        c = _ffi.SopranoConfig(
            config["hidden_size"], config["num_hidden_layers"], config["intermediate_size"], config["num_attention_heads"],
            config["num_key_value_heads"], config["head_dim"], config["vocab_size"], float(g("rms_norm_eps", 1e-6)),
            float(g("rope_theta", 10000.0)), int(g("tie_word_embeddings", False)), int(g("max_position_embeddings", 512)),
            int(g("bos_token_id", 1)), int(g("eos_token_id", 2)), int(g("pad_token_id", 0)), stop_token_id, int(g("sample_rate", 32000)),
            int(g("decoder_num_layers", 8)), int(g("decoder_dim", 768)), int(g("decoder_intermediate_dim", 2304)), int(g("hop_length", 512)),
            int(g("n_fft", 2048)), int(g("upscale", 4)), int(g("input_kernel", 1)), int(g("dw_kernel", 3)), int(g("token_size", 2048)),
            int(g("receptive_field", 4)), max_batch, max_context)
        if repo is not None and "soprano-1.1" not in repo.lower():
            c.decoder_dim, c.decoder_intermediate_dim, c.input_kernel = 512, 1536, 3
        return c

    def _init(self, config: dict, c: _ffi.SopranoConfig):
        self.config, self.vocab_size, self.hidden_size = config, c.vocab_size, c.hidden_size
        self.sample_rate, self.max_batch = c.sample_rate, c.max_batch

    def __init__(self, config: dict, weights: Dict, device: int = 0, max_batch: int = 8, max_context: int = 2048,
                 repo: Optional[str] = None, stop_token_id: int = 3):
        """`weights` in SopranoModel.sanitize's layout (model.*, lm_head.weight, decoder.decoder.*, decoder.head.out.*); `repo` (a repo
        name) applies the decoder rule of fromModelDirectory, None takes config's decoder geometry as it is."""
        c = self._c_config(config, max_batch, max_context, repo, stop_token_id)
        self._init(config, c)
        table, keep = _ffi.make_tensor_table(weights)
        self._h = C.c_void_p()
        _ffi.check(_ffi.lib().b2a_soprano_create(device, C.byref(c), table, len(weights), C.byref(self._h)))
        del keep

    @classmethod
    def random_init(cls, config: dict, decoder_weights: Dict, device: int = 0, max_batch: int = 8, max_context: int = 2048,
                    std: float = 0.02, seed: int = 1234, stop_token_id: int = 3) -> "SopranoModel":
        """Language model drawn on the device (benchmarks), decoder from `decoder_weights` (decoder.decoder.* / decoder.head.*)."""
        self = cls.__new__(cls)
        c = cls._c_config(config, max_batch, max_context, None, stop_token_id)
        self._init(config, c)
        table, keep = _ffi.make_tensor_table(decoder_weights)
        self._h = C.c_void_p()
        _ffi.check(_ffi.lib().b2a_soprano_create_random(device, C.byref(c), std, seed, table, len(decoder_weights), C.byref(self._h)))
        del keep
        return self

    @classmethod
    def from_model_directory(cls, model_dir, repo: Optional[str] = None, device: int = 0, max_batch: int = 8,
                             max_context: int = 2048) -> "SopranoModel":
        """fromModelDirectory (:928-976) inside the library (b2a_soprano_create_from_directory): config.json, the decoder rule on `repo`
        (default: the directory's name), every *.safetensors, sanitize, de-quantisation; the stop token is the tokenizer's EOS."""
        import json
        from pathlib import Path
        self = cls.__new__(cls)
        config = json.loads((Path(model_dir) / "config.json").read_text())
        if repo is None:           # the directory name as given (trailing slashes dropped, not resolved), for both calls below
            d = str(model_dir).rstrip("/") or "/"
            repo = d[d.rfind("/") + 1:] or "/"
        self._h = C.c_void_p()
        _ffi.check(_ffi.lib().b2a_soprano_create_from_directory(str(model_dir).encode(), repo.encode(), device, max_batch, max_context,
                                                                 C.byref(self._h)))
        c = _ffi.SopranoConfig()
        _ffi.check(_ffi.lib().b2a_soprano_config_from_json(str(Path(model_dir) / "config.json").encode(), repo.encode(), max_batch,
                                                           max_context, C.byref(c), None, None))
        self._init(config, c)
        return self

    @property
    def stream(self) -> int:
        return int(_ffi.lib().b2a_tts_stream(self._h) or 0)

    def wave_length(self, n_states: int) -> int:
        """Samples of the waveform of n hidden states (after the cut, Soprano.swift:664-671)."""
        return int(_ffi.lib().b2a_soprano_wave_length(self._h, n_states))

    # -- forward / generate ----------------------------------------------------------------------
    def __call__(self, input_ids, reset_cache: bool = True) -> np.ndarray:
        """callAsFunction (:241-251): ids [B, L] -> logits [B, L, V]."""
        ids = np.ascontiguousarray(input_ids, dtype=np.int32)
        B, L = ids.shape
        out = np.empty((B, L, self.vocab_size), dtype=np.float32)
        _ffi.check(_ffi.lib().b2a_tts_forward_logits(self._h, _ffi.ptr(ids), B, L, int(reset_cache), _ffi.ptr(out)))
        return out

    def generate_batch(self, input_ids, parameters: Optional[GenerateParameters] = None, decode_audio: bool = True,
                       on_token: Optional[Callable[[int, int, int], None]] = None):
        """B independent sentences, one streamGenerate (:801-885) + decode (:656-673) each, as the rows of one call.  Returns (tokens
        [list per row], waveforms [list of 1-D float32, or None without decode_audio], AudioGenerationInfo)."""
        p = parameters or self.default_generation_parameters
        ids = np.ascontiguousarray(input_ids, dtype=np.int32)
        B, L = ids.shape
        toks = np.zeros((B, p.max_tokens), dtype=np.int32)
        ntok = np.zeros(B, dtype=np.int32)
        self._slots = p.max_tokens + 1
        cap = self.wave_length(p.max_tokens + 1) if decode_audio else 0
        wave = np.empty((B, cap), dtype=np.float32) if decode_audio else None
        wlen = np.zeros(B, dtype=np.int64)
        info = _ffi.GenInfo()
        _ffi.check(_ffi.lib().b2a_tts_set_bench_flags(self._h, int(p.mask_eos), 0))
        gp = p._c()
        cb = _ffi.TOKEN_CB(lambda user, b, step, tok: on_token(b, step, tok)) if on_token else _ffi.TOKEN_CB()
        _ffi.check(_ffi.lib().b2a_tts_generate(self._h, _ffi.ptr(ids), B, L, C.byref(gp), _ffi.ptr(toks), _ffi.ptr(ntok),
                                               _ffi.ptr(wave), cap, _ffi.ptr(wlen), C.byref(info), cb, None))
        tokens = [toks[b, :ntok[b]].tolist() for b in range(B)]
        waves = [wave[b, :wlen[b]].copy() for b in range(B)] if decode_audio else [None] * B
        return tokens, waves, _info(info)

    def hidden_states(self, batch: int) -> List[np.ndarray]:
        """The hidden states the last generate_batch call captured: per row [1 + generated tokens, hidden_size]."""
        n = np.zeros(batch, dtype=np.int32)
        out = np.empty((batch, self._slots, self.hidden_size), dtype=np.float32)      # max_tokens + 1 slots per row
        _ffi.check(_ffi.lib().b2a_soprano_hidden_states(self._h, batch, _ffi.ptr(out), _ffi.ptr(n)))
        return [out[b, :n[b]].copy() for b in range(batch)]

    def _groups(self, prompts: Sequence[Prompt]) -> List[List[int]]:
        """Sentence indices grouped by prompt length (at most max_batch per group), in order of first appearance."""
        groups: Dict[int, List[List[int]]] = {}
        order: List[List[int]] = []
        for i, pr in enumerate(prompts):
            g = groups.setdefault(len(pr), [])
            if not g or len(g[-1]) == self.max_batch:
                g.append([])
                order.append(g[-1])
            g[-1].append(i)
        return order

    def _run(self, prompts: Sequence[Prompt], p: GenerateParameters, on_token=None):
        waves: List[Optional[np.ndarray]] = [None] * len(prompts)
        infos = []
        for grp in self._groups(prompts):
            ids = np.asarray([list(prompts[i]) for i in grp], dtype=np.int32)
            cb = (lambda b, s, t, grp=grp: on_token(grp[b], s, t)) if on_token else None
            _, w, info = self.generate_batch(ids, p, on_token=cb)
            infos.append(info)
            for k, i in enumerate(grp):
                waves[i] = w[k]
        return waves, infos

    @staticmethod
    def _prompts(prompt_ids: Union[Prompt, Sequence[Prompt]]) -> List[Prompt]:
        if len(prompt_ids) and isinstance(prompt_ids[0], (int, np.integer)):
            return [prompt_ids]
        return list(prompt_ids)

    def generate(self, prompt_ids: Union[Prompt, Sequence[Prompt]], parameters: Optional[GenerateParameters] = None) -> np.ndarray:
        """generate(text:...) (:577-690) after tokenisation: one token-id prompt, or one per sentence.  Sentences whose prompts have
        equal length run as the rows of one call; the waveforms are concatenated in sentence order."""
        prompts = self._prompts(prompt_ids)
        if not prompts:
            raise _ffi.AudioGenerationError(_ffi.ERR_GENERATION_FAILED, "No audio generated")      # :686
        waves, _ = self._run(prompts, parameters or self.default_generation_parameters)
        return np.concatenate(waves)

    def generate_stream(self, prompt_ids: Union[Prompt, Sequence[Prompt]], parameters: Optional[GenerateParameters] = None) -> Iterator:
        """generateStream (:693-798): ('token', id) for every kept token in sentence order, then ('info', AudioGenerationInfo), then one
        ('audio', waveform) of all sentences."""
        prompts = self._prompts(prompt_ids)
        p = parameters or self.default_stream_parameters
        toks: List[List[int]] = [[] for _ in prompts]
        waves, infos = self._run(prompts, p, on_token=lambda i, s, t: toks[i].append(t))
        for t in toks:
            for x in t:
                yield ("token", x)
        n = sum(i.generation_token_count for i in infos)
        el = sum(i.prefill_time + i.generate_time + i.codec_time for i in infos)
        yield ("info", AudioGenerationInfo(0, n, 0.0, el, n / max(el, 1e-9), max((i.peak_memory_usage for i in infos), default=0.0),
                                           sum(i.codec_time for i in infos)))
        yield ("audio", np.concatenate(waves))

    def decode(self, hidden) -> List[np.ndarray]:
        """SopranoDecoder.callAsFunction (SopranoDecoder.swift:263-284) + the cut (:664-671): hidden [B, n, H] (or [n, H]) -> B waveforms."""
        h = np.ascontiguousarray(hidden, dtype=np.float32)
        if h.ndim == 2:
            h = h[None]
        B, n, _ = h.shape
        cap = self.wave_length(n)
        out = np.empty((B, cap), dtype=np.float32)
        wl = np.zeros(B, dtype=np.int64)
        _ffi.check(_ffi.lib().b2a_soprano_decode_hidden(self._h, _ffi.ptr(h), B, n, _ffi.ptr(out), cap, _ffi.ptr(wl)))
        return [out[b, :wl[b]].copy() for b in range(B)]

    def cancel(self) -> None:
        _ffi.check(_ffi.lib().b2a_tts_cancel(self._h))

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                _ffi.lib().b2a_tts_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:   # interpreter shutdown: ctypes globals may already be gone
            pass
