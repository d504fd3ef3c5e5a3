"""CPU study: what operand precision does a tensor-core causal PROMPT attention (the Orpheus prefill) need?

The fp32 oracle (oracle/llama.py) is re-run with the causal attention of the prompt pass (every forward call with more than one
position) emulated as a tensor-core kernel would compute it: q, k, v and the probabilities p rounded to fp16 or bf16, optionally as
hi + lo pairs (x = hi + lo, lo = round(x - hi)), the products accumulated in fp32.  The decode steps stay exact.

    python tools/prompt_attention_precision_study.py

For a tiny model with Orpheus's head geometry (3 query heads per kv head, head_dim 128) and prompts of 129, 330 and 913 tokens it
prints, against the exact run: the relative L2 error of the logits of the last prompt position, the same for one more position fed
after 8 greedy tokens (what tests/test_gpu_long_prefill.py bounds: 4e-5 against the per-position replay), and whether the greedy
tokens change."""
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import llama as ol  # noqa: E402

# (name, fp type, q/k as hi/lo pairs, v as hi/lo pairs, p as hi/lo pairs)
MODES = [
    ("fp16", "fp16", False, False, False),
    ("bf16", "bf16", False, False, False),
    ("fp16 qk-hilo", "fp16", True, False, False),
    ("fp16 qk,v-hilo", "fp16", True, True, False),
    ("fp16 qk,p-hilo", "fp16", True, False, True),
    ("fp16 qk,v,p-hilo", "fp16", True, True, True),
    ("bf16 qk,v,p-hilo", "bf16", True, True, True),
]


def rnd(x, kind):
    return x.to(torch.bfloat16 if kind == "bf16" else torch.float16).to(torch.float32)


def pair(x, kind, split):
    hi = rnd(x, kind)
    return (hi, rnd(x - hi, kind)) if split else (hi, torch.zeros_like(x))


def emulated_forward(mode):
    _, kind, qk_s, v_s, p_s = mode
    exact = ol.LlamaOracle.forward

    def softmax_at_v(q, kk, vv, mask, hd):
        qh, ql = pair(q, kind, qk_s)
        kh, kl = pair(kk, kind, qk_s)
        s = (qh @ kh.transpose(-1, -2) + qh @ kl.transpose(-1, -2) + ql @ kh.transpose(-1, -2)) * hd ** -0.5
        s = s.masked_fill(mask, float("-inf"))
        m = s.amax(-1, keepdim=True)
        e = torch.exp(s - m)
        ph, pl = pair(e, kind, p_s)
        vh, vl = pair(vv, kind, v_s)
        # the sum of what the tensor core multiplies: the normaliser is taken over the rounded probabilities
        return (ph @ vh + ph @ vl + pl @ vh) / (ph + pl).sum(-1, keepdim=True)

    def forward(self, ids, trace=None, head_positions=None):
        if ids.shape[1] == 1:
            return exact(self, ids, trace, head_positions)
        cfg = self.cfg
        B, L = ids.shape
        nq, nkv, hd = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        assert self.offset == 0 and not self.round
        h = self.w["model.embed_tokens.weight"][ids].to(torch.float32)
        pos = torch.arange(L)
        mask = torch.arange(L)[None, :] > pos[:, None]
        for l in range(cfg.num_hidden_layers):
            p = f"model.layers.{l}."
            xn = ol.rms_norm(h, self.w[p + "input_layernorm.weight"], cfg.rms_norm_eps)
            q = self._lin(xn, p + "self_attn.q_proj.weight").view(B, L, nq, hd).transpose(1, 2)
            k = self._lin(xn, p + "self_attn.k_proj.weight").view(B, L, nkv, hd).transpose(1, 2)
            v = self._lin(xn, p + "self_attn.v_proj.weight").view(B, L, nkv, hd).transpose(1, 2)
            q, k = ol.rope(q, pos, self.freqs), ol.rope(k, pos, self.freqs)
            self.k[l], self.v[l] = k, v
            kk = k.repeat_interleave(nq // nkv, dim=1)
            vv = v.repeat_interleave(nq // nkv, dim=1)
            a = softmax_at_v(q, kk, vv, mask, hd).transpose(1, 2).reshape(B, L, nq * hd)
            h = h + self._lin(a, p + "self_attn.o_proj.weight")
            xn = ol.rms_norm(h, self.w[p + "post_attention_layernorm.weight"], cfg.rms_norm_eps)
            g = self._lin(xn, p + "mlp.gate_proj.weight")
            u = self._lin(xn, p + "mlp.up_proj.weight")
            h = h + self._lin(torch.nn.functional.silu(g) * u, p + "mlp.down_proj.weight")
        self.offset += L
        hn = ol.rms_norm(h, self.w["model.norm.weight"], cfg.rms_norm_eps)
        head = self.w["model.embed_tokens.weight"]
        return hn @ head.to(torch.float32).T
    return forward


def rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def run(cfg, W, ids, n_gen):
    m = ol.LlamaOracle(cfg, W, False)
    first = m.forward(torch.as_tensor(ids))[:, -1].numpy()
    toks = ol.generate_tokens(ol.LlamaOracle(cfg, W, False), ids, n_gen, temperature=0.0, rep_penalty=1.0, rep_context=0)
    m = ol.LlamaOracle(cfg, W, False)
    m.forward(torch.as_tensor(ids))
    for j in range(n_gen):
        nxt = m.forward(torch.as_tensor(np.asarray([[t[j]] for t in toks], dtype=np.int64)))
    return first, toks, nxt[:, -1].numpy()


def main():
    cfg = ol.LlamaConfig(hidden_size=256, num_hidden_layers=2, intermediate_size=512, num_attention_heads=3,
                         num_key_value_heads=1, head_dim=128, vocab_size=2048)
    W = ol.init_weights(cfg, 1234, std=0.08)
    exact = ol.LlamaOracle.forward
    for L in (129, 330, 913):
        ids = np.random.default_rng(100 + L).integers(0, 2048, size=(1, L)).astype(np.int64)
        f0, t0, n0 = run(cfg, W, ids, 8)
        for mode in MODES:
            ol.LlamaOracle.forward = emulated_forward(mode)
            try:
                f, t, n = run(cfg, W, ids, 8)
            finally:
                ol.LlamaOracle.forward = exact
            print(f"L {L:4d}  {mode[0]:18s} last-prompt logits {rel(f, f0):.2e}   next-step logits {rel(n, n0):.2e}   "
                  f"greedy tokens {'same' if t == t0 else 'CHANGED'}", flush=True)


if __name__ == "__main__":
    main()
