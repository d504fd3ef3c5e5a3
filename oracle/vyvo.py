"""Oracle for VyvoTTS: a Qwen3 language model whose vocabulary speaks SNAC-24 kHz codes.  Test infrastructure only.

Follows (paths relative to the reference checkout):
  Sources/MLXAudioTTS/Models/Qwen3/Qwen3.swift:18-29     special token ids
  Sources/MLXAudioTTS/Models/Qwen3/Qwen3.swift:47-114    decodeAudioFromCodes: whole row up to 50 frames, else independent 50-frame chunks
  Sources/MLXAudioTTS/Models/Qwen3/Qwen3.swift:145-303   Qwen3Attention (per-head q/k RMSNorm BEFORE RoPE; RoPE(base, scale = 1 / factor)
                                                         for rope_scaling type "linear"), MLP, block, inner model
  Sources/MLXAudioTTS/Models/Qwen3/Qwen3.swift:333-358   parseOutputRow
  Sources/MLXAudioTTS/Models/Qwen3/Qwen3.swift:377-474   prepareInputIds (token-id level)
  Sources/MLXAudioTTS/Models/Qwen3/Qwen3.swift:476-486   tied (embedTokens.asLinear) or untied lm head
  Sources/MLXAudioTTS/Models/Qwen3/Qwen3.swift:643-681   generate loop (stop on 151671, not kept)
  Sources/MLXAudioTTS/Models/Qwen3/Config.swift:15-73    Qwen3Configuration and its defaults
Numerics as oracle/llama.py: bf16 weights, activations in ``dtype`` (float32 for the device parity tests, float64 to pin the oracle
against ``transformers.Qwen3ForCausalLM`` in tests/test_oracle_vyvo.py).  The sampler helpers are oracle/llama.py's.
"""
from __future__ import annotations

import json
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .llama import repetition_penalty

TOKENIZER_LENGTH = 151669
START_OF_TEXT, END_OF_TEXT = 151643, 151645
START_OF_SPEECH, END_OF_SPEECH = TOKENIZER_LENGTH + 1, TOKENIZER_LENGTH + 2
START_OF_HUMAN, END_OF_HUMAN = TOKENIZER_LENGTH + 3, TOKENIZER_LENGTH + 4
START_OF_AI, END_OF_AI = TOKENIZER_LENGTH + 5, TOKENIZER_LENGTH + 6
PAD_TOKEN = TOKENIZER_LENGTH + 7
AUDIO_TOKENS_START = TOKENIZER_LENGTH + 10
DECODE_CHUNK = 50


@dataclass
class Qwen3Config:
    """Qwen3Configuration (Config.swift:15-73).  Defaults of the required keys = Qwen3-0.6B's layer shapes with VyvoTTS's vocabulary
    (an assumption: the published checkpoint's config.json is not at hand)."""
    hidden_size: int = 1024
    num_hidden_layers: int = 28
    intermediate_size: int = 3072
    num_attention_heads: int = 16
    num_key_value_heads: int = 8
    head_dim: int = 128
    vocab_size: int = 180352
    rms_norm_eps: float = 1e-6
    rope_theta: float = 1_000_000.0
    rope_scaling: Optional[dict] = None
    tie_word_embeddings: bool = False
    max_position_embeddings: int = 32768
    sample_rate: int = 24000
    eos_token_id: int = 151645

    @property
    def rope_linear_factor(self) -> float:
        """Qwen3.swift:177-188: only {"type": "linear", "factor": f} changes RoPE; anything else is ignored."""
        rs = self.rope_scaling or {}
        return float(rs["factor"]) if rs.get("type") == "linear" and "factor" in rs else 1.0

    def to_json(self) -> dict:
        return {k: getattr(self, k) for k in self.__dataclass_fields__}


REQUIRED = ("hidden_size", "num_hidden_layers", "intermediate_size", "num_attention_heads", "rms_norm_eps", "vocab_size",
            "num_key_value_heads", "head_dim")


def config_from_json(d: dict) -> Qwen3Config:
    """Qwen3Configuration.init(from:) (Config.swift:50-73): the eight decode()d keys are required, the rest default."""
    missing = [k for k in REQUIRED if d.get(k) is None]
    if missing:
        raise KeyError(f"config.json: missing {missing[0]}")
    c = Qwen3Config(**{k: d[k] for k in REQUIRED})
    c.rope_theta = float(d.get("rope_theta") or 1_000_000.0)
    c.rope_scaling = d.get("rope_scaling")
    c.tie_word_embeddings = bool(d.get("tie_word_embeddings", False))
    c.max_position_embeddings = int(d.get("max_position_embeddings", 32768))
    c.sample_rate = int(d.get("sample_rate", 24000))
    c.eos_token_id = int(d.get("eos_token_id", 151645))
    return c


def init_weights(cfg: Qwen3Config, seed: int = 1234, std: float = 0.02) -> Dict[str, torch.Tensor]:
    """Random init N(0, std^2) in bf16, norm gains (q/k norms included) 1 +- 0.1; the reference's keys."""
    g = torch.Generator().manual_seed(seed)
    H, I, hd, nq, nkv = cfg.hidden_size, cfg.intermediate_size, cfg.head_dim, cfg.num_attention_heads, cfg.num_key_value_heads

    def lin(o, i):
        return (torch.randn(o, i, generator=g) * std).to(torch.bfloat16)

    def gain(n):
        return (1.0 + 0.1 * torch.randn(n, generator=g)).to(torch.bfloat16)

    w = {"model.embed_tokens.weight": lin(cfg.vocab_size, H)}
    for l in range(cfg.num_hidden_layers):
        p = f"model.layers.{l}."
        w[p + "self_attn.q_proj.weight"] = lin(nq * hd, H)
        w[p + "self_attn.k_proj.weight"] = lin(nkv * hd, H)
        w[p + "self_attn.v_proj.weight"] = lin(nkv * hd, H)
        w[p + "self_attn.o_proj.weight"] = lin(H, nq * hd)
        w[p + "self_attn.q_norm.weight"] = gain(hd)
        w[p + "self_attn.k_norm.weight"] = gain(hd)
        w[p + "mlp.gate_proj.weight"] = lin(I, H)
        w[p + "mlp.up_proj.weight"] = lin(I, H)
        w[p + "mlp.down_proj.weight"] = lin(H, I)
        w[p + "input_layernorm.weight"] = gain(H)
        w[p + "post_attention_layernorm.weight"] = gain(H)
    w["model.norm.weight"] = gain(H)
    if not cfg.tie_word_embeddings:
        w["lm_head.weight"] = lin(cfg.vocab_size, H)
    return w


def sanitize(cfg: Qwen3Config, weights: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Qwen3Model.sanitize (Qwen3.swift:520-526): lm_head.weight goes when the head is tied."""
    return {k: v for k, v in weights.items() if not (cfg.tie_word_embeddings and k == "lm_head.weight")}


def rope_freqs(cfg: Qwen3Config) -> torch.Tensor:
    """MLXFast.RoPE(base: theta, scale: 1 / factor), traditional = false: angle = pos / (theta^(2i/d) * factor)."""
    i = torch.arange(0, cfg.head_dim, 2, dtype=torch.float64)
    return cfg.rope_theta ** (i / cfg.head_dim) * cfg.rope_linear_factor


def rope(x: torch.Tensor, positions: torch.Tensor, freqs: torch.Tensor) -> torch.Tensor:
    d2 = x.shape[-1] // 2
    ang = positions[:, None].to(torch.float64) / freqs[None, :]
    cos, sin = torch.cos(ang).to(x.dtype), torch.sin(ang).to(x.dtype)
    x1, x2 = x[..., :d2], x[..., d2:]
    return torch.cat([x1 * cos - x2 * sin, x2 * cos + x1 * sin], dim=-1)


def rms_norm(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    return x * torch.rsqrt((x * x).mean(-1, keepdim=True) + eps) * w.to(x.dtype)


class VyvoOracle:
    """Qwen3Model.callAsFunction (Qwen3.swift:476-486) with a contiguous KV cache (KVCacheSimple)."""

    def __init__(self, cfg: Qwen3Config, weights: Dict[str, torch.Tensor], dtype: torch.dtype = torch.float32):
        self.cfg, self.dtype = cfg, dtype
        self.w = {k: v.to(dtype) for k, v in weights.items()}
        self.freqs = rope_freqs(cfg)
        self.reset()

    def reset(self):
        self.k = [None] * self.cfg.num_hidden_layers
        self.v = [None] * self.cfg.num_hidden_layers
        self.offset = 0

    @torch.no_grad()
    def forward(self, ids, head_positions: Optional[Sequence[int]] = None) -> torch.Tensor:
        """ids [B, L] -> logits [B, L, V] (or [B, len(head_positions), V])."""
        cfg, W = self.cfg, self.w
        ids = torch.as_tensor(np.asarray(ids), dtype=torch.long)
        B, L = ids.shape
        nq, nkv, hd, eps = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim, cfg.rms_norm_eps
        h = W["model.embed_tokens.weight"][ids]
        pos = torch.arange(self.offset, self.offset + L)
        for l in range(cfg.num_hidden_layers):
            p = f"model.layers.{l}."
            xn = rms_norm(h, W[p + "input_layernorm.weight"], eps)
            q = (xn @ W[p + "self_attn.q_proj.weight"].T).view(B, L, nq, hd)
            k = (xn @ W[p + "self_attn.k_proj.weight"].T).view(B, L, nkv, hd)
            v = (xn @ W[p + "self_attn.v_proj.weight"].T).view(B, L, nkv, hd).transpose(1, 2)
            q = rope(rms_norm(q, W[p + "self_attn.q_norm.weight"], eps).transpose(1, 2), pos, self.freqs)
            k = rope(rms_norm(k, W[p + "self_attn.k_norm.weight"], eps).transpose(1, 2), pos, self.freqs)
            self.k[l] = k if self.k[l] is None else torch.cat([self.k[l], k], dim=2)
            self.v[l] = v if self.v[l] is None else torch.cat([self.v[l], v], dim=2)
            kk = self.k[l].repeat_interleave(nq // nkv, dim=1)
            vv = self.v[l].repeat_interleave(nq // nkv, dim=1)
            s = (q @ kk.transpose(-1, -2)) * (hd ** -0.5)
            if L > 1:
                s = s.masked_fill(torch.arange(kk.shape[2])[None, :] > pos[:, None], float("-inf"))
            a = (torch.softmax(s, dim=-1) @ vv).transpose(1, 2).reshape(B, L, nq * hd)
            h = h + a @ W[p + "self_attn.o_proj.weight"].T
            xn = rms_norm(h, W[p + "post_attention_layernorm.weight"], eps)
            g, u = xn @ W[p + "mlp.gate_proj.weight"].T, xn @ W[p + "mlp.up_proj.weight"].T
            h = h + (torch.nn.functional.silu(g) * u) @ W[p + "mlp.down_proj.weight"].T
        self.offset += L
        if head_positions is not None:
            h = h[:, list(head_positions)]
        hn = rms_norm(h, W["model.norm.weight"], eps)
        head = W["model.embed_tokens.weight"] if cfg.tie_word_embeddings else W["lm_head.weight"]
        return hn @ head.T


@torch.no_grad()
def generate_tokens(model: VyvoOracle, input_ids: np.ndarray, max_tokens: int, rep_penalty: float = 1.0, rep_context: int = 20,
                    mask_eos: bool = False) -> List[List[int]]:
    """Greedy generate (Qwen3.swift:643-681) per row, rows independent: repetition penalty over the last rep_context tokens, stop on
    151671 (not kept)."""
    B = input_ids.shape[0]
    model.reset()
    logits = model.forward(input_ids)[:, -1].float().numpy()
    ctx = [list(map(int, row[-rep_context:])) if rep_context > 0 else [] for row in input_ids]
    done, gen = [False] * B, [[] for _ in range(B)]
    for _ in range(max_tokens):
        nxt = np.zeros(B, dtype=np.int64)
        for b in range(B):
            lg = repetition_penalty(logits[b], ctx[b], rep_penalty)
            if mask_eos:
                lg[END_OF_SPEECH] = -np.inf
            nxt[b] = int(np.argmax(lg))
        for b in range(B):
            if done[b]:
                continue
            if nxt[b] == END_OF_SPEECH:
                done[b] = True
            else:
                gen[b].append(int(nxt[b]))
                if rep_context > 0:
                    ctx[b] = (ctx[b] + [int(nxt[b])])[-rep_context:]
        if all(done):
            break
        logits = model.forward(nxt[:, None])[:, -1].float().numpy()
    return gen


# --------------------------------------------------------------------------- token plumbing

def prepare_input_ids(prompts: Sequence[Sequence[int]], ref_text_ids: Optional[Sequence[int]] = None,
                      ref_code_list: Optional[Sequence[int]] = None) -> Tuple[np.ndarray, np.ndarray]:
    """prepareInputIds (Qwen3.swift:377-474) after tokenisation: left-pad with 151676 to the longest prompt, then (with a reference clip's
    7-token interleaved codes and its transcript) [SOH] transcript [EOT, EOH] [SOAI, SOS] codes + 151679 [EOS, EOAI], then
    [SOH] prompt [EOT, EOH]."""
    max_len = max((len(p) for p in prompts), default=0)
    rows = []
    for p in prompts:
        seq = [PAD_TOKEN] * (max_len - len(p))
        if ref_text_ids is not None and ref_code_list is not None:
            seq += [START_OF_HUMAN] + list(ref_text_ids) + [END_OF_TEXT, END_OF_HUMAN]
            seq += [START_OF_AI, START_OF_SPEECH] + [c + AUDIO_TOKENS_START for c in ref_code_list] + [END_OF_SPEECH, END_OF_AI]
        seq += [START_OF_HUMAN] + list(p) + [END_OF_TEXT, END_OF_HUMAN]
        rows.append(seq)
    ids = np.asarray(rows, dtype=np.int32)
    return ids, ids != PAD_TOKEN


def parse_output_row(tokens: Sequence[int]) -> List[int]:
    """parseOutputRow (Qwen3.swift:333-358)."""
    t = [int(x) for x in tokens]
    start = max((i for i, x in enumerate(t) if x == START_OF_SPEECH), default=None)
    if start is None:
        soa = max((i for i, x in enumerate(t) if x == START_OF_AI), default=None)
        if soa is not None:
            first = next((i for i in range(soa + 1, len(t)) if t[i] >= AUDIO_TOKENS_START), None)
            if first is not None:
                start = first - 1
    sl = t[start + 1:] if start is not None else t
    f = [x for x in sl if x != END_OF_SPEECH]
    n = (len(f) // 7) * 7
    return [x - AUDIO_TOKENS_START for x in f[:n]]


def decode_chunks(n_codes: int, chunk: int = DECODE_CHUNK) -> List[Tuple[int, int]]:
    """decodeAudioFromCodes (Qwen3.swift:47-83): the (first frame, frames) pieces a code list of n_codes is decoded in."""
    groups = (n_codes + 1) // 7
    if groups <= chunk:
        return [(0, groups)]
    return [(g0, min(chunk, groups - g0)) for g0 in range(0, groups, chunk)]


def load_config(path) -> Qwen3Config:
    with open(path) as f:
        return config_from_json(json.load(f))
