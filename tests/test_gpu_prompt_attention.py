"""The Orpheus long-prompt attention (csrc/prompt_attn_tc.cuh: pack_prompt_kernel + prompt_attn_kernel, through b2a_prompt_attn_test)
against float64 causal GQA attention with RoPE, at lengths on both sides of every tile edge (64-key tiles, 128-query tiles) and
every query-per-kv-head ratio the engine accepts.

The operand arithmetic comes from tools/prompt_attention_precision_study.py, which re-runs the oracle with the prompt attention
emulated in each candidate arithmetic (tiny model, 3 query heads per kv head, relative L2 of the logits against the exact run):

    L  913  fp16               last-prompt logits 5.61e-04   next-step logits 1.71e-04   greedy tokens same
    L  913  bf16               last-prompt logits 5.39e-03   next-step logits 1.70e-03   greedy tokens same
    L  913  fp16 qk-hilo       last-prompt logits 3.29e-04   next-step logits 1.11e-04   greedy tokens same
    L  913  fp16 qk,v-hilo     last-prompt logits 1.43e-04   next-step logits 4.87e-05   greedy tokens same
    L  913  fp16 qk,p-hilo     last-prompt logits 3.01e-04   next-step logits 1.23e-04   greedy tokens same
    L  913  fp16 qk,v,p-hilo   last-prompt logits 1.78e-06   next-step logits 6.82e-07   greedy tokens same
    L  913  bf16 qk,v,p-hilo   last-prompt logits 8.37e-06   next-step logits 3.33e-06   greedy tokens same

(L = 129 and 330 read the same.)  Only hi/lo pairs on q/k, v and p stay inside the 4e-5 the per-position replay is held to, so the
kernel computes S = qh kh + qh kl + ql kh and O = ph vh + ph vl + pl vh in fp16 with fp32 accumulation.

Two float64 references on the same fp32 q | k | v:
  * the kernel's arithmetic: q, k after RoPE (the keys read back from the cache the kernel wrote) and v as the fp16 hi + lo pairs the
    kernel multiplies; softmax exact.  The pairs carry 22 significand bits, so the rest is fp32 accumulation, the hi/lo rounding of
    P and the bf16 hi/lo output pair.
  * exact attention from the fp32 projections, RoPE with the oracle's angles (float32 position / float32 frequency).
Also checked: the cache rows 0..L-1 hold the RoPE'd keys and the raw values, rows >= L and the output rows of padding tokens are
untouched (NaN sentinels), and each output lo is the remainder of its hi."""
import math

import pytest
import torch

from gemm_reference import assert_lo_within_half_ulp, errors, hilo_rows
from oracle import llama as ol

pytestmark = pytest.mark.gpu

HD = 128
FREQS = torch.from_numpy(ol.llama3_rope_freqs(ol.LlamaConfig()))


def _rope64(x, L):
    """[.., L, 128] float64 RoPE with the oracle's fp32 angles."""
    ang = (torch.arange(L, dtype=torch.float32)[:, None] / FREQS[None, :]).double().to(x.device)
    c, s = torch.cos(ang), torch.sin(ang)
    x1, x2 = x[..., :HD // 2], x[..., HD // 2:]
    return torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1)


def _pair(x):
    """float -> float64 value of its fp16 hi + lo pair."""
    x = x.float()
    hi = x.half()
    return hi.double() + (x - hi.float()).half().double()


def _attn(q, k, v, G):
    """causal GQA attention, float64: q [B, nq, L, 128], k / v [B, nkv, L, 128]."""
    L = q.shape[2]
    k, v = k.repeat_interleave(G, 1), v.repeat_interleave(G, 1)
    s = (q @ k.transpose(-1, -2)) / math.sqrt(HD)
    s = s.masked_fill(torch.ones(L, L, dtype=torch.bool, device=q.device).triu(1), float("-inf"))
    return torch.softmax(s, -1) @ v


# (B, L, nkv, G): a covering subset of L x G x B
CASES = [(1, 2, 1, 3), (3, 64, 2, 1), (1, 129, 2, 3), (8, 130, 1, 2), (3, 191, 1, 4), (1, 192, 1, 6), (3, 193, 1, 8),
         (8, 330, 1, 3), (1, 913, 8, 3), (1, 2048, 1, 8), (8, 129, 1, 8), (1, 913, 1, 6)]


@pytest.mark.parametrize("B,L,nkv,G", CASES)
def test_prompt_attention_matches_float64(b2a, B, L, nkv, G):
    """Measured on an H100 80GB HBM3 (700 W power limit): worst case over all cases (relative L2 / max over peak) 4.6e-6 / 7.2e-6
    against the kernel's arithmetic and against exact attention alike (the hi/lo operands leave nothing the emulation can see; what is
    left is fp32 accumulation and the bf16 hi/lo output), RoPE'd keys 3.8e-8 / 1.2e-7 from float64.  Bounds: 2-4x the worst case for
    the output, about 20x for the keys (sincosf against float64 cos / sin of the same fp32 angle)."""
    nq = nkv * G
    max_ctx = L + 37
    g = torch.Generator(device="cuda").manual_seed(1000 * B + L + G)
    T, dq, dk = B * L, nq * HD, nkv * HD
    qkv = torch.randn(T, dq + 2 * dk, device="cuda", generator=g)
    qkv[:, :dq] *= 2.0                                                 # scores with a standard deviation of about 2
    kc = torch.full((B, nkv, max_ctx, HD), float("nan"), device="cuda")
    vc = torch.full_like(kc, float("nan"))
    rows = 2 * 64 * (-(-T // 64))
    out = torch.full((rows, dq), float("nan"), device="cuda", dtype=torch.bfloat16)
    freqs = FREQS.float().cuda()
    f = b2a._ffi
    st = f.lib().b2a_prompt_attn_test(f.ptr(qkv), f.ptr(freqs), f.ptr(kc), f.ptr(vc), f.ptr(out), B, L, nq, nkv, max_ctx, None)
    torch.cuda.synchronize()
    assert st == 0, f.lib().b2a_last_error()

    def heads(x, n):
        return x.view(B, L, n, HD).transpose(1, 2)
    q, k, v = heads(qkv[:, :dq], nq), heads(qkv[:, dq:dq + dk], nkv), heads(qkv[:, dq + dk:], nkv)
    # the cache: RoPE'd keys and the values bit for bit at rows < L, sentinels above
    assert kc[:, :, L:].isnan().all() and vc[:, :, L:].isnan().all()
    assert torch.equal(vc[:, :, :L], v)
    k_exact = _rope64(k.double(), L)
    e_k = errors(kc[:, :, :L], k_exact)
    assert e_k[0] < 1e-6 and e_k[1] < 2e-6, e_k

    hr, lr = hilo_rows(T, 128)
    hi, lo = out[hr], out[lr]
    assert_lo_within_half_ulp(hi, lo)
    written = torch.zeros(rows, dtype=torch.bool, device="cuda")
    written[hr] = True
    written[lr] = True
    assert out[~written].isnan().all()
    got = heads(hi.double() + lo.double(), nq)

    q_rope = _rope64(q.double(), L)
    emulated = _attn(_pair(q_rope), _pair(kc[:, :, :L]), _pair(v), G)
    exact = _attn(q_rope, k_exact, v.double(), G)
    e_emu, e_exact = errors(got, emulated), errors(got, exact)
    print(f"B={B} L={L} nkv={nkv} G={G}: emulated {e_emu[0]:.2e} / {e_emu[1]:.2e}, exact {e_exact[0]:.2e} / {e_exact[1]:.2e}, "
          f"keys {e_k[0]:.2e} / {e_k[1]:.2e}")
    assert e_emu[0] < 1e-5 and e_emu[1] < 3e-5, e_emu
    assert e_exact[0] < 1e-5 and e_exact[1] < 3e-5, e_exact
