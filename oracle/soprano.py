"""Oracle for Soprano: a Qwen3 language model whose final-norm hidden states a Vocos decoder turns into audio.  Test infrastructure only.

Follows (paths relative to the reference checkout):
  Sources/MLXAudioTTS/Models/Soprano/SopranoConfig.swift:65-176  SopranoConfiguration and its defaults
  Sources/MLXAudioTTS/Models/Soprano/Soprano.swift:24-180        the Qwen3 stack (oracle/vyvo.py's forward, RoPE without scaling)
  Sources/MLXAudioTTS/Models/Soprano/Soprano.swift:254-275       forwardWithHiddenStates
  Sources/MLXAudioTTS/Models/Soprano/Soprano.swift:314-361       sanitize
  Sources/MLXAudioTTS/Models/Soprano/Soprano.swift:656-673       the cut: the last n * token_size - token_size samples
  Sources/MLXAudioTTS/Models/Soprano/Soprano.swift:801-901       streamGenerate and applyRepetitionPenalty
  Sources/MLXAudioTTS/Models/Soprano/Soprano.swift:928-941       fromModelDirectory's decoder rule
  Sources/MLXAudioTTS/Models/Soprano/Soprano.swift:996-1059      TopPSampler (top-p on exp of the raw logits, temperature afterwards)
  Sources/MLXAudioTTS/Models/Soprano/SopranoDecoder.swift:22-80  interpolate1d (align corners)
  Sources/MLXAudioTTS/Models/Soprano/SopranoDecoder.swift:263-284 SopranoDecoder: upsample, Vocos backbone, ISTFT head (oracle/vocos.py)
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import vocos as ovocos
from . import vyvo


@dataclass
class SopranoConfig:
    """SopranoConfiguration.  Defaults of the required keys: an ASSUMED Soprano-80M geometry (hidden 512 = the decoder's input
    channels, head_dim 128, vocab 8192, 8 layers, MLP 2048); the published config.json is not at hand."""
    hidden_size: int = 512
    num_hidden_layers: int = 8
    intermediate_size: int = 2048
    num_attention_heads: int = 4
    num_key_value_heads: int = 1
    head_dim: int = 128
    vocab_size: int = 8192
    max_position_embeddings: int = 512
    rms_norm_eps: float = 1e-6
    rope_theta: float = 10000.0
    tie_word_embeddings: bool = False
    bos_token_id: int = 1
    eos_token_id: int = 2
    pad_token_id: int = 0
    sample_rate: int = 32000
    decoder_num_layers: int = 8
    decoder_dim: int = 768
    decoder_intermediate_dim: int = 2304
    hop_length: int = 512
    n_fft: int = 2048
    upscale: int = 4
    input_kernel: int = 1
    dw_kernel: int = 3
    token_size: int = 2048
    receptive_field: int = 4

    def to_json(self) -> dict:
        return {k: getattr(self, k) for k in self.__dataclass_fields__}

    def qwen3(self) -> vyvo.Qwen3Config:
        return vyvo.Qwen3Config(hidden_size=self.hidden_size, num_hidden_layers=self.num_hidden_layers, intermediate_size=self.intermediate_size,
                                num_attention_heads=self.num_attention_heads, num_key_value_heads=self.num_key_value_heads,
                                head_dim=self.head_dim, vocab_size=self.vocab_size, rms_norm_eps=self.rms_norm_eps, rope_theta=self.rope_theta,
                                tie_word_embeddings=self.tie_word_embeddings)

    def vocos(self) -> ovocos.VocosConfig:
        return ovocos.VocosConfig(input_channels=self.hidden_size, dim=self.decoder_dim, intermediate_dim=self.decoder_intermediate_dim,
                                  num_layers=self.decoder_num_layers, n_fft=self.n_fft, hop_length=self.hop_length,
                                  input_kernel_size=self.input_kernel, dw_kernel_size=self.dw_kernel)


def apply_repo_rule(cfg: SopranoConfig, repo: str) -> SopranoConfig:
    """fromModelDirectory (Soprano.swift:934-941): only a repo named like soprano-1.1 keeps config's decoder; any other gets 512 / 1536 / 3."""
    if "soprano-1.1" not in repo.lower():
        cfg.decoder_dim, cfg.decoder_intermediate_dim, cfg.input_kernel = 512, 1536, 3
    return cfg


def init_weights(cfg: SopranoConfig, seed: int = 1234, std: float = 0.02) -> Dict[str, object]:
    """The sanitized key layout: model.* / lm_head.weight (bf16, oracle/vyvo.py's init) and decoder.decoder.* / decoder.head.* (fp32)."""
    w: Dict[str, object] = dict(vyvo.init_weights(cfg.qwen3(), seed, std))
    w.update(decoder_weights_only(cfg, seed))
    return w


def decoder_weights_only(cfg: SopranoConfig, seed: int = 1234) -> Dict[str, np.ndarray]:
    """init_weights' decoder.decoder.* / decoder.head.* entries alone (a device-drawn language model needs no host copy)."""
    return {("decoder.decoder." + k[len("backbone."):]) if k.startswith("backbone.") else "decoder." + k: v
            for k, v in ovocos.init_weights(cfg.vocos(), seed + 1).items()}


def decoder_weights(w: Dict) -> Dict[str, np.ndarray]:
    """decoder.* -> the keys oracle/vocos.py reads."""
    out = {}
    for k, v in w.items():
        if k.startswith("decoder.decoder."):
            out["backbone." + k[len("decoder.decoder."):]] = v
        elif k.startswith("decoder.head."):
            out["head." + k[len("decoder.head."):]] = v
    return out


def sanitize(cfg: SopranoConfig, weights: Dict) -> Dict:
    """SopranoModel.sanitize (Soprano.swift:314-361) on key names (the dtype changes are the loader's)."""
    out = {}
    for key, v in weights.items():
        k = key[len("model."):] if key.startswith("model.") else key
        if k.startswith("decoder."):
            pass
        elif k.startswith("language_model.lm_head"):
            k = k.replace("language_model.", "")
        elif k.startswith("language_model."):
            k = k.replace("language_model.", "model.")
        elif not k.startswith("lm_head"):
            k = "model." + k
        out[k] = v
    if cfg.tie_word_embeddings:
        out.pop("lm_head.weight", None)
    return out


# --------------------------------------------------------------------------- language model with hidden states

class SopranoLM(vyvo.VyvoOracle):
    """forwardWithHiddenStates (Soprano.swift:254-275): logits and the final-RMSNorm hidden states of every position, with a contiguous
    KV cache; the layers are oracle/vyvo.py's Qwen3 forward."""

    def __init__(self, cfg: SopranoConfig, weights: Dict, dtype: torch.dtype = torch.float32):
        super().__init__(cfg.qwen3(), {k: v for k, v in weights.items() if not k.startswith("decoder.")}, dtype)

    @torch.no_grad()
    def forward_hidden(self, ids) -> Tuple[torch.Tensor, torch.Tensor]:
        """ids [B, L] -> (logits [B, L, V], hidden [B, L, H])."""
        cfg, W = self.cfg, self.w
        ids = torch.as_tensor(np.asarray(ids), dtype=torch.long)
        B, L = ids.shape
        nq, nkv, hd, eps = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim, cfg.rms_norm_eps
        h = W["model.embed_tokens.weight"][ids]
        pos = torch.arange(self.offset, self.offset + L)
        for l in range(cfg.num_hidden_layers):
            p = f"model.layers.{l}."
            xn = vyvo.rms_norm(h, W[p + "input_layernorm.weight"], eps)
            q = (xn @ W[p + "self_attn.q_proj.weight"].T).view(B, L, nq, hd)
            k = (xn @ W[p + "self_attn.k_proj.weight"].T).view(B, L, nkv, hd)
            v = (xn @ W[p + "self_attn.v_proj.weight"].T).view(B, L, nkv, hd).transpose(1, 2)
            q = vyvo.rope(vyvo.rms_norm(q, W[p + "self_attn.q_norm.weight"], eps).transpose(1, 2), pos, self.freqs)
            k = vyvo.rope(vyvo.rms_norm(k, W[p + "self_attn.k_norm.weight"], eps).transpose(1, 2), pos, self.freqs)
            self.k[l] = k if self.k[l] is None else torch.cat([self.k[l], k], dim=2)
            self.v[l] = v if self.v[l] is None else torch.cat([self.v[l], v], dim=2)
            kk = self.k[l].repeat_interleave(nq // nkv, dim=1)
            vv = self.v[l].repeat_interleave(nq // nkv, dim=1)
            s = (q @ kk.transpose(-1, -2)) * (hd ** -0.5)
            if L > 1:
                s = s.masked_fill(torch.arange(kk.shape[2])[None, :] > pos[:, None], float("-inf"))
            a = (torch.softmax(s, dim=-1) @ vv).transpose(1, 2).reshape(B, L, nq * hd)
            h = h + a @ W[p + "self_attn.o_proj.weight"].T
            xn = vyvo.rms_norm(h, W[p + "post_attention_layernorm.weight"], eps)
            g, u = xn @ W[p + "mlp.gate_proj.weight"].T, xn @ W[p + "mlp.up_proj.weight"].T
            h = h + (torch.nn.functional.silu(g) * u) @ W[p + "mlp.down_proj.weight"].T
        self.offset += L
        hn = vyvo.rms_norm(h, W["model.norm.weight"], eps)
        head = W["model.embed_tokens.weight"] if cfg.tie_word_embeddings else W["lm_head.weight"]
        return hn @ head.T, hn


# --------------------------------------------------------------------------- sampler

def repetition_penalty(logits: np.ndarray, generated: Sequence[int], penalty: float, context: int) -> np.ndarray:
    """applyRepetitionPenalty (Soprano.swift:888-901) as streamGenerate calls it (:843-850): nothing while no token has been generated,
    else over the last `context` GENERATED tokens (never the prompt), once per OCCURRENCE, in sequence, in fp32."""
    out = np.asarray(logits, dtype=np.float32).copy()
    if penalty == 1.0 or not generated:
        return out
    p = np.float32(penalty)
    for t in list(generated)[-context:]:
        if 0 <= t < len(out):
            out[t] = out[t] / p if out[t] > 0 else out[t] * p
    return out


def top_p_keep(logits: np.ndarray, top_p: float) -> np.ndarray:
    """applyTopP(logprobs:) (Soprano.swift:1002-1037) on UNNORMALISED logits: keep token i iff the ascending cumulative sum of exp(l_j)
    through i exceeds 1 - top_p (float64 here; ties count as one block, i.e. strictly-larger mass)."""
    l = np.asarray(logits, dtype=np.float64)
    e = np.exp(l)
    larger = np.array([e[l > x].sum() for x in l])      # the cumulative sum through i = total - mass of strictly larger logits
    return e.sum() - larger > 1.0 - top_p


def sample_probs(logits: np.ndarray, temperature: float, top_p: float) -> np.ndarray:
    """The distribution TopPSampler.sample draws from (:1039-1059): categorical(filtered / T) over the kept set; the argmax alone when no
    token is kept (the reference would sample an all -inf row; the library's deliberate difference)."""
    l = np.asarray(logits, dtype=np.float64)
    keep = top_p_keep(l, top_p)
    if not keep.any():
        out = np.zeros_like(l)
        out[int(np.argmax(l))] = 1.0
        return out
    z = np.where(keep, l / temperature, -np.inf)
    z = np.exp(z - z.max())
    return z / z.sum()


def penalty_variant(logits: np.ndarray, prompt: Sequence[int], generated: Sequence[int], penalty: float, context: int,
                    variant: str) -> np.ndarray:
    """The penalty streamGenerate applies ("soprano": repetition_penalty above), or one of two rules it must NOT be mistaken for, so that
    tests can show they tell them apart: "unique" penalises each token of the window once (mlx-swift-lm's RepetitionContext), "prompt"
    lets the prompt's tokens into the window."""
    if variant == "soprano":
        return repetition_penalty(logits, generated, penalty, context)
    if variant == "unique":
        return repetition_penalty(logits, list(dict.fromkeys(list(generated)[-context:])), penalty, context)
    if variant == "prompt":
        return repetition_penalty(logits, (list(prompt) + list(generated))[-context:], penalty, context)
    raise ValueError(variant)


@torch.no_grad()
def generate(model: SopranoLM, input_ids: np.ndarray, max_tokens: int, stop_token: int = 3, rep_penalty: float = 1.5,
             rep_context: int = 30, variant: str = "soprano") -> Tuple[List[List[int]], List[np.ndarray]]:
    """streamGenerate (Soprano.swift:801-885) at temperature 0, rows independent: (tokens per row, hidden states per row [1 + n, H]).
    The state of the last prompt position, then one per kept token fed back; the stop token is neither kept nor fed.  `variant`: see
    penalty_variant (only "soprano" is the reference's)."""
    B = input_ids.shape[0]
    model.reset()
    logits, hid = model.forward_hidden(input_ids)
    states = [[hid[b, -1].float().numpy()] for b in range(B)]
    logits = logits[:, -1].float().numpy()
    done, gen = [False] * B, [[] for _ in range(B)]
    for _ in range(max_tokens):
        nxt = np.zeros(B, dtype=np.int64)
        fed = [False] * B
        for b in range(B):
            nxt[b] = int(np.argmax(penalty_variant(logits[b], input_ids[b], gen[b], rep_penalty, rep_context, variant)))
            if done[b]:
                continue
            if nxt[b] == stop_token:
                done[b] = True
            else:
                gen[b].append(int(nxt[b]))
                fed[b] = True
        if all(done):
            break
        lg, hid = model.forward_hidden(nxt[:, None])
        logits = lg[:, -1].float().numpy()
        for b in range(B):
            if fed[b]:
                states[b].append(hid[b, -1].float().numpy())
    return gen, [np.stack(s) for s in states]


# --------------------------------------------------------------------------- decoder

def interpolate1d(x: torch.Tensor, size: int) -> torch.Tensor:
    """interpolate1d(alignCorners: true) (SopranoDecoder.swift:22-80) on x [B, C, n]: x_t = t * ((n-1)/(size-1)) in fp32 in that order."""
    n = x.shape[-1]
    if size < 1 or n < 1 or size == n:
        return x
    if n == 1:
        return x.expand(*x.shape[:-1], size)
    pos = torch.arange(size, dtype=torch.float32) * np.float32(np.float32(n - 1) / np.float32(size - 1))
    lo = torch.floor(pos).to(torch.long)
    hi = torch.clamp(lo + 1, max=n - 1)
    f = (pos - lo.to(torch.float32)).to(x.dtype)
    return x[..., lo] * (1 - f) + x[..., hi] * f


def wave_cut(n: int, token_size: int, audio: np.ndarray) -> np.ndarray:
    """Soprano.swift:664-671: keep the last n * token_size - token_size samples when that is positive."""
    keep = n * token_size - token_size
    return audio[-keep:] if keep > 0 else audio


def decode(cfg: SopranoConfig, weights: Dict, hidden: np.ndarray) -> List[np.ndarray]:
    """SopranoDecoder (SopranoDecoder.swift:263-284) + the cut on hidden [B, n, H] (float64)."""
    h = torch.as_tensor(np.asarray(hidden), dtype=torch.float64)
    n = h.shape[1]
    up = interpolate1d(h.transpose(1, 2), cfg.upscale * (n - 1) + 1).transpose(1, 2)
    audio = ovocos.decode(cfg.vocos(), decoder_weights(weights), up.numpy())
    return [wave_cut(n, cfg.token_size, a) for a in audio]
