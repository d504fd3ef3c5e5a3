"""The Whisper encoder attention (csrc/attn_tc.cuh: pack_qkv_f16_kernel + mha_tc_kernel, through b2a_mha_tc_test) at the only length
the encoder launches, T = 1500: 11 full 128-query / 128-key tiles and a tail tile of 92 valid queries and keys.

Two float64 references on the same fp32 q | k | v:
  * the kernel's stated arithmetic: q * 64^-1/2, k and v rounded to fp16; S exact; P = fp16(exp(S - rowmax)); l = sum of the rounded
    P; O = (P V) / l.  What is left is fp32 accumulation and the bf16 hi/lo output pair, so the bound is tight.
  * exact softmax attention, which bounds what the fp16 operands cost.
The output is written as the out-projection's B operand: hi/lo bf16 tiles of 64 tokens, token t = b * T + i at hi row
(t // 64) * 128 + t % 64 and lo row hi + 64.  Rows of tokens >= B * T must not be written."""
import math

import pytest
import torch

from gemm_reference import assert_lo_within_half_ulp, errors, hilo_rows

pytestmark = pytest.mark.gpu

T, HD = 1500, 64


def _mha(b2a, qkv, out, B, nh):
    f = b2a._ffi
    st = f.lib().b2a_mha_tc_test(f.ptr(qkv), f.ptr(out), B, T, nh, None)
    torch.cuda.synchronize()
    assert st == 0, f.lib().b2a_last_error()


def _heads(x, B, nh):
    """[B * T, nh * 64] -> [B, nh, T, 64] float64."""
    return x.double().view(B, T, nh, HD).transpose(1, 2)


@pytest.mark.parametrize("B,nh", [(1, 2), (1, 8), (3, 8), (1, 12), (3, 12), (3, 2)])
def test_encoder_attention_matches_float64(b2a, B, nh):
    """Measured on an H100 80GB HBM3, worst case over all cases (relative L2 / max over peak): against the emulated arithmetic
    1.1e-5 / 9.2e-5 (tail tile alone 1.4e-5 / 6.4e-5), rms of the per-query output scale 3.2e-6; against exact attention
    6.4e-4 / 9.2e-4.  The emulation cannot round P exactly as the kernel does (its S and exp differ in the last fp32 bits, which
    moves a few P across an fp16 rounding boundary), hence the max/peak of order 1e-4.  Summing l from the unrounded P instead
    moves the per-query scale by 2e-5.  Bounds: about 2-3x the worst case."""
    d = nh * HD
    g = torch.Generator(device="cuda").manual_seed(B * 100 + nh)
    qkv = torch.randn(B * T, 3 * d, device="cuda", generator=g)
    qkv[:, :d] *= 2.0                                                  # scores with a standard deviation of about 2
    q, k, v = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
    n_tok = B * T
    rows = 2 * 64 * (-(-n_tok // 64))
    out = torch.full((rows, d), float("nan"), device="cuda", dtype=torch.bfloat16)
    _mha(b2a, qkv, out, B, nh)

    hr, lr = hilo_rows(n_tok, 128)
    hi, lo = out[hr], out[lr]
    got = (hi.double() + lo.double()).view(B, T, nh, HD).transpose(1, 2)
    assert_lo_within_half_ulp(hi, lo)
    written = torch.zeros(rows, dtype=torch.bool, device="cuda")
    written[hr] = True
    written[lr] = True
    assert out[~written].isnan().all()

    qh = _heads((q * (1.0 / math.sqrt(HD))).half(), B, nh)
    kh, vh = _heads(k.half(), B, nh), _heads(v.half(), B, nh)
    s = qh @ kh.transpose(-1, -2)
    p = torch.exp(s - s.amax(-1, keepdim=True)).half().double()
    emulated = (p @ vh) / p.sum(-1, keepdim=True)
    s = _heads(q, B, nh) @ _heads(k, B, nh).transpose(-1, -2) / math.sqrt(HD)
    exact = torch.softmax(s, -1) @ _heads(v, B, nh)
    # per-query scale of the output against the emulation: 1 / l is the only factor common to a whole output row
    scale = (got * emulated).sum(-1) / (emulated * emulated).sum(-1)
    scale_rms = float((scale - 1).pow(2).mean().sqrt())
    e_emu, e_tail, e_exact = errors(got, emulated), errors(got[..., 1408:, :], emulated[..., 1408:, :]), errors(got, exact)
    print(f"B={B} nh={nh}: emulated {e_emu[0]:.2e} / {e_emu[1]:.2e}, tail {e_tail[0]:.2e} / {e_tail[1]:.2e}, "
          f"exact {e_exact[0]:.2e} / {e_exact[1]:.2e}, row scale rms {scale_rms:.2e}")
    assert e_emu[0] < 3e-5 and e_emu[1] < 2e-4, e_emu
    assert e_tail[0] < 3e-5 and e_tail[1] < 2e-4, e_tail       # the tail tile: queries and keys 1408..1499
    assert scale_rms < 1e-5, scale_rms
    assert e_exact[0] < 2e-3 and e_exact[1] < 3e-3, e_exact
