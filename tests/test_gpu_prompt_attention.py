"""The prompt attention of the batched prefill (through b2a_prompt_attn_test) against float64 causal GQA attention with RoPE, with and
without Qwen3's per-head q/k RMSNorm, at every query-per-kv-head ratio the engine accepts:
  * path 2, the long-prompt wgmma attention (csrc/prompt_attn_tc.cuh: pack_prompt_kernel + prompt_attn_kernel), at lengths on both
    sides of every tile edge (64-key tiles, 128-query tiles);
  * path 1, the SIMT prefill_attn_kernel<G> (csrc/llama.cu) that every prompt of up to 128 positions takes, at lengths around its
    32-query tiles up to the largest the engine gives it (128 at G <= 4, 124 at G = 6, 92 at G = 8: the shared-memory edge).

The wgmma path's operand arithmetic comes from tools/prompt_attention_precision_study.py, which re-runs the oracle with the prompt
attention emulated in each candidate arithmetic (tiny model, 3 query heads per kv head, relative L2 of the logits against the exact run):

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
  * the wgmma kernel's arithmetic: q, k after RoPE (the keys read back from the cache the kernel wrote) and v as the fp16 hi + lo pairs
    the kernel multiplies; softmax exact.  The pairs carry 22 significand bits, so the rest is fp32 accumulation, the hi/lo rounding of
    P and the bf16 hi/lo output pair.
  * exact attention from the fp32 projections: q/k RMSNorm with the gains, RoPE with the oracle's angles (float32 position / float32
    frequency).  The SIMT kernel has no reduced-precision operand, so it is held to this one alone.
Also checked: the cache rows 0..L-1 hold the (normalised) RoPE'd keys and the raw values, rows >= L and the output rows of padding
tokens are untouched (NaN sentinels), and each output lo is the remainder of its hi.

Then the cache the three Llama / Qwen3 attention kernels share: the SIMT prefill, the wgmma pack and the decode step
(test_gpu_decode_attention.py) must write the same rows for the same q|k|v at the same position, and decode steps after either prefill
must match float64 attention over the whole sequence."""
import math

import pytest
import torch

from attention_reference import FREQS, decode_attn, qk_gains, rmsnorm64, rope64
from gemm_reference import assert_lo_within_half_ulp, errors, hilo_rows

pytestmark = pytest.mark.gpu

HD, EPS = 128, 1e-6


def _rope64(x, L):
    """[.., L, 128] float64 RoPE at positions 0..L-1 with the oracle's fp32 angles."""
    return rope64(x, torch.arange(L))


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


def _simt_max_len(G):
    """The largest L the engine gives the SIMT prefill_attn_kernel<G>: L <= 128 and 2 L + 32 G rows of 128 fp32 in 220 KB."""
    return max(L for L in range(1, 129) if (2 * L + 32 * G) * HD * 4 <= 220 * 1024)


def _case(B, L, nkv, G, path, norm, id=None):
    return pytest.param(B, L, nkv, G, path, norm, id=id or f"{'simt' if path == 1 else 'wgmma'}-B{B}-L{L}-nkv{nkv}-G{G}"
                                                         f"{'-qk_norm' if norm else ''}")


# (B, L, nkv, G): a covering subset of L x G x B for the wgmma path (ids as they were before the other cases joined)
CASES = [(1, 2, 1, 3), (3, 64, 2, 1), (1, 129, 2, 3), (8, 130, 1, 2), (3, 191, 1, 4), (1, 192, 1, 6), (3, 193, 1, 8),
         (8, 330, 1, 3), (1, 913, 8, 3), (1, 2048, 1, 8), (8, 129, 1, 8), (1, 913, 1, 6)]
WGMMA_NORM_CASES = [(1, 129, 2, 3), (3, 193, 1, 8), (8, 330, 1, 3)]
SIMT_LENGTHS = [2, 31, 32, 33, 64, 100]


def _simt_cases():
    """Every G, every length up to the largest admitted (and that one), B cycling through 1, 3, 8, q/k norm on and off."""
    out, i = [], 0
    for G in (1, 2, 3, 4, 6, 8):
        for L in [L for L in SIMT_LENGTHS if L < _simt_max_len(G)] + [_simt_max_len(G)]:
            for norm in (False, True):
                out.append(_case((1, 3, 8)[i % 3], L, 2 if G <= 4 else 1, G, 1, norm))
                i += 1
    return out


ALL_CASES = ([_case(*c, 2, False, id="-".join(map(str, c))) for c in CASES] + [_case(*c, 2, True) for c in WGMMA_NORM_CASES]
             + _simt_cases())


def _prompt(b2a, qkv, kc, vc, B, L, nq, nkv, path, qn=None, kn=None):
    """One b2a_prompt_attn_test launch into a fresh NaN-filled output; returns (status, output)."""
    rows = 2 * 64 * (-(-B * L // 64))
    out = torch.full((rows, nq * HD), float("nan"), device="cuda", dtype=torch.bfloat16)
    f = b2a._ffi
    st = f.lib().b2a_prompt_attn_test(f.ptr(qkv), f.ptr(FREQS.cuda()), f.ptr(qn), f.ptr(kn), EPS, f.ptr(kc), f.ptr(vc), f.ptr(out),
                                      B, L, nq, nkv, kc.shape[2], path, None)
    torch.cuda.synchronize()
    return st, out


@pytest.mark.parametrize("B,L,nkv,G,path,norm", ALL_CASES)
def test_prompt_attention_matches_float64(b2a, B, L, nkv, G, path, norm):
    """Measured on an H100 80GB HBM3 (700 W power limit), path 2 without q/k norm: worst case over all cases (relative L2 / max over
    peak) 4.6e-6 / 7.2e-6 against the kernel's arithmetic and against exact attention alike (the hi/lo operands leave nothing the
    emulation can see; what is left is fp32 accumulation and the bf16 hi/lo output), RoPE'd keys 3.8e-8 / 1.2e-7 from float64.  Bounds:
    2-4x the worst case for the output, about 20x for the keys (sincosf against float64 cos / sin of the same fp32 angle).
    The other cases, same card: path 2 with q/k norm (gains 1 + 0.3 N(0, 1), q's times 2 for the score spread, eps 1e-6, the second
    token's k scaled to about 1e-4 so that eps outweighs mean(k^2)) 2.8e-6 / 5.3e-6 against either reference; path 1 (fp32 throughout,
    so exact attention only) 2.7e-6 / 6.2e-6 with or without the norm; keys 7.0e-8 / 2.3e-7.  Bounds: 3-4x, the keys' too."""
    nq = nkv * G
    max_ctx = L + 37
    g = torch.Generator(device="cuda").manual_seed(1000 * B + L + G + (7 if path == 1 else 0) + 3 * norm)
    T, dq, dk = B * L, nq * HD, nkv * HD
    qkv = torch.randn(T, dq + 2 * dk, device="cuda", generator=g)
    qn, kn = qk_gains(L + G, 2.0) if norm else (None, None)
    if norm and T > 1:
        qkv[1, dq:dq + dk] *= 1e-4
    else:
        qkv[:, :dq] *= 2.0                                             # scores with a standard deviation of about 2
    kc = torch.full((B, nkv, max_ctx, HD), float("nan"), device="cuda")
    vc = torch.full_like(kc, float("nan"))
    st, out = _prompt(b2a, qkv, kc, vc, B, L, nq, nkv, path, qn, kn)
    assert st == 0, b2a._ffi.lib().b2a_last_error()
    rows = out.shape[0]

    def heads(x, n):
        return x.view(B, L, n, HD).transpose(1, 2)
    q, k, v = heads(qkv[:, :dq], nq), heads(qkv[:, dq:dq + dk], nkv), heads(qkv[:, dq + dk:], nkv)
    # the cache: (normalised) RoPE'd keys and the values bit for bit at rows < L, sentinels above
    assert kc[:, :, L:].isnan().all() and vc[:, :, L:].isnan().all()
    assert torch.equal(vc[:, :, :L], v)
    k_exact = _rope64(rmsnorm64(k, kn, EPS), L)
    e_k = errors(kc[:, :, :L], k_exact)
    original = path == 2 and not norm                                  # the cases and bounds from before the SIMT path and the norm
    k_tol, tol = ((1e-6, 2e-6), (1e-5, 3e-5)) if original else ((2.5e-7, 8e-7), (8e-6, 2e-5))
    assert e_k[0] < k_tol[0] and e_k[1] < k_tol[1], e_k

    hr, lr = hilo_rows(T, 128)
    hi, lo = out[hr], out[lr]
    assert_lo_within_half_ulp(hi, lo)
    written = torch.zeros(rows, dtype=torch.bool, device="cuda")
    written[hr] = True
    written[lr] = True
    assert out[~written].isnan().all()
    got = heads(hi.double() + lo.double(), nq)

    q_rope = _rope64(rmsnorm64(q, qn, EPS), L)
    exact = _attn(q_rope, k_exact, v.double(), G)
    e_exact = errors(got, exact)
    if path == 1:
        print(f"simt B={B} L={L} nkv={nkv} G={G} norm={norm}: exact {e_exact[0]:.2e} / {e_exact[1]:.2e}, "
              f"keys {e_k[0]:.2e} / {e_k[1]:.2e}")
    else:
        emulated = _attn(_pair(q_rope), _pair(kc[:, :, :L]), _pair(v), G)
        e_emu = errors(got, emulated)
        print(f"wgmma B={B} L={L} nkv={nkv} G={G} norm={norm}: emulated {e_emu[0]:.2e} / {e_emu[1]:.2e}, "
              f"exact {e_exact[0]:.2e} / {e_exact[1]:.2e}, keys {e_k[0]:.2e} / {e_k[1]:.2e}")
        assert e_emu[0] < tol[0] and e_emu[1] < tol[1], e_emu
    assert e_exact[0] < tol[0] and e_exact[1] < tol[1], e_exact


@pytest.mark.parametrize("G", [1, 2, 3, 4, 6, 8])
def test_simt_prompt_attention_refuses_longer_prompts(b2a, G):
    """Path 1 takes exactly the lengths the engine gives the SIMT kernel: one position more is refused before anything runs."""
    nkv, L = 1, _simt_max_len(G) + 1
    qkv = torch.zeros(L, (G + 2) * HD, device="cuda")
    kc = torch.zeros(1, nkv, L, HD, device="cuda")
    vc = torch.zeros_like(kc)
    st, out = _prompt(b2a, qkv, kc, vc, 1, L, G, nkv, 1)
    assert st == b2a._ffi.ERR_INVALID_INPUT, b2a._ffi.lib().b2a_last_error()
    assert out.isnan().all() and not kc.any()


@pytest.mark.parametrize("norm", [False, True], ids=["plain", "qk_norm"])
def test_three_kernels_write_one_cache(b2a, norm):
    """The SIMT prefill, the wgmma pack and the decode step, fed the same q|k|v row at the same position, write the same cache row:
    the prompt's 128 positions through both prefill paths, and 8 of them (around the 32-query and 64-key tile edges) as the 8 rows of
    one decode step.  Values are bit-equal, and so are keys, with and without q/k norm, on an H100 80GB HBM3 (sm_90a build, nvcc -O3
    without fast math): the three kernels compute the norm's warp reduction, x * rstd * gain and x1 * cos - x2 * sin the same way,
    from the same sincosf angle, and the compiler contracts them alike."""
    nq, nkv, L = 16, 8, 128
    ld = (nq + 2 * nkv) * HD
    g = torch.Generator(device="cuda").manual_seed(31 + norm)
    qkv = torch.randn(L, ld, device="cuda", generator=g)
    qkv[1, nq * HD:(nq + nkv) * HD] *= 1e-4
    qn, kn = qk_gains(5, 2.0) if norm else (None, None)
    caches = []
    for path in (1, 2):
        kc = torch.full((1, nkv, L, HD), float("nan"), device="cuda")
        vc = torch.full_like(kc, float("nan"))
        st, _ = _prompt(b2a, qkv, kc, vc, 1, L, nq, nkv, path, qn, kn)
        assert st == 0, b2a._ffi.lib().b2a_last_error()
        caches.append((kc[0], vc[0]))
    (k1, v1), (k2, v2) = caches
    P = [0, 1, 31, 32, 63, 64, 100, 127]
    kd = torch.full((8, nkv, L, HD), float("nan"), device="cuda")
    vd = torch.full_like(kd, float("nan"))
    for b, p in enumerate(P):                                          # the rows before p as the prefill left them
        kd[b, :, :p], vd[b, :, :p] = k1[:, :p], v1[:, :p]
    st, out = decode_attn(b2a, qkv[P].contiguous(), torch.tensor(P, dtype=torch.int32, device="cuda"), kd, vd, nq, nkv, qn, kn, EPS)
    assert st == 0, b2a._ffi.lib().b2a_last_error()
    assert torch.isfinite(out[:8].float()).all()
    k3 = torch.stack([kd[b, :, p] for b, p in enumerate(P)], 1)       # [nkv, 8, 128]
    v3 = torch.stack([vd[b, :, p] for b, p in enumerate(P)], 1)
    assert torch.equal(v1, v2) and torch.equal(v3, v1[:, P])
    print(f"norm={norm}: keys that differ: SIMT vs wgmma pack {int((k1 != k2).sum())} of {k1.numel()}, "
          f"decode vs SIMT {int((k3 != k1[:, P]).sum())} of {k3.numel()}")
    assert torch.equal(k1, k2) and torch.equal(k3, k1[:, P])


@pytest.mark.parametrize("L,path", [(100, 1), (300, 2)], ids=["simt_100", "wgmma_300"])
def test_decode_steps_after_prefill(b2a, L, path):
    """Qwen3 geometry (16 q / 8 kv heads, q/k norm): prefill L positions on one path, then 4 decode steps at L .. L + 3 on the same
    cache, each against float64 attention over the whole sequence (every key normalised and rotated from its fp32 projection).
    Measured on an H100 80GB HBM3 (700 W power limit): worst step 2.5e-6 / 4.2e-6 after the SIMT prefill, 2.7e-6 / 4.6e-6 after the
    wgmma one (the cache is fp32 either way).  Bounds 3x."""
    nq, nkv, G, B, n_dec = 16, 8, 2, 2, 4
    ld, dq, dk = (nq + 2 * nkv) * HD, nq * HD, nkv * HD
    max_ctx = L + n_dec + 5
    g = torch.Generator(device="cuda").manual_seed(L)
    qkv = torch.randn(B, L + n_dec, ld, device="cuda", generator=g)
    qn, kn = qk_gains(L, 2.0)
    kc = torch.full((B, nkv, max_ctx, HD), float("nan"), device="cuda")
    vc = torch.full_like(kc, float("nan"))
    st, _ = _prompt(b2a, qkv[:, :L].reshape(B * L, ld).contiguous(), kc, vc, B, L, nq, nkv, path, qn, kn)
    assert st == 0, b2a._ffi.lib().b2a_last_error()
    n = L + n_dec
    k_all = rope64(rmsnorm64(qkv[:, :, dq:dq + dk].view(B, n, nkv, HD).transpose(1, 2), kn, EPS), torch.arange(n))
    v_all = qkv[:, :, dq + dk:].view(B, n, nkv, HD).transpose(1, 2).double()
    q_all = rope64(rmsnorm64(qkv[:, :, :dq].view(B, n, nq, HD).transpose(1, 2), qn, EPS), torch.arange(n))
    worst = (0.0, 0.0)
    for i in range(n_dec):
        p = L + i
        pos = torch.full((B,), p, dtype=torch.int32, device="cuda")
        st, out = decode_attn(b2a, qkv[:, p].contiguous(), pos, kc, vc, nq, nkv, qn, kn, EPS)
        assert st == 0, b2a._ffi.lib().b2a_last_error()
        got = out[:B].double() + out[8:8 + B].double()
        s = q_all[:, :, p:p + 1] @ k_all[:, :, :p + 1].repeat_interleave(G, 1).transpose(-1, -2) / math.sqrt(HD)
        ref = (torch.softmax(s, -1) @ v_all[:, :, :p + 1].repeat_interleave(G, 1))[:, :, 0].reshape(B, dq)
        e = errors(got, ref)
        worst = max(worst[0], e[0]), max(worst[1], e[1])
    print(f"prefill L={L} path {path} + {n_dec} decode steps: worst {worst[0]:.2e} / {worst[1]:.2e}")
    assert worst[0] < 8e-6 and worst[1] < 1.4e-5, worst
