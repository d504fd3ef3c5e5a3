"""The fused SNAC kernels of the 128- and 64-channel decoder stages (csrc/snac_fused.cuh) in isolation, against float64:

- rf::ru_fused_kernel through b2a_snac_unit_test: one ResidualUnit (dilation 1, 3, 9) or NoiseBlock per launch, with the optional
  Snake'd hi/lo copy in the next transposed conv's 2-tap im2col layout;
- rf::convt_fused_kernel through b2a_snac_convt_test: the last block's Snake + transposed conv.

The sequence lengths reach the kernels' edges: T < 27 (the dilation-9 halo spans the whole utterance), T <= 64 (the second
64-token sub-tile of a C = 64 tile is empty), 64 < T < 128 (it is partly valid), odd tile counts (one team of the last CTA idles),
several utterances (the halo must not read the neighbour) and one CTA (both teams loop over tiles, which runs the register
prefetch chain and the one-time weight wait).

Tolerances: measured on an H100 80GB HBM3 at a 400 W power limit, the worst unit case was relative L2 5.0e-6 (the hi/lo copy,
dilation 1, C = 64) and max/peak 1.1e-5 (the hi/lo copy, dilation 9, C = 128); y alone stays below 3.8e-6 and 6.3e-6.  Bounds:
1.5e-5 and 3e-5, about 3x the worst case.  The transposed conv (worst 4.6e-6 and 6.4e-6) takes the same bounds."""
import math

import numpy as np
import pytest
import torch

from codec_reference import check_hilo_output, conv_transpose, dual_layout, dwconv7, gauss, nan_hilo_buffer, pointwise, snake
from gemm_reference import assert_close

pytestmark = pytest.mark.gpu

MODE_RU, MODE_NOISE = 0, 1
REL_TOL, PEAK_TOL = 1.5e-5, 3e-5
SHAPES = [(2, 20), (1, 50), (2, 100), (1, 300), (3, 77)]          # (B, T)


def unit(b2a, mode, C, dil, x, y, B, T, pw_w, dw_w=None, dw_b=None, a_in=None, a_mid=None, pw_bias=None, noise=None, seed=0, hl=None,
         a_next=None, ctas=0) -> int:
    f = b2a._ffi
    st = f.lib().b2a_snac_unit_test(mode, C, dil, f.ptr(x), f.ptr(y), B, T, f.ptr(dw_w), f.ptr(dw_b), f.ptr(a_in), f.ptr(a_mid), f.ptr(pw_w),
                                    f.ptr(pw_bias), f.ptr(noise), seed, f.ptr(hl), f.ptr(a_next), ctas, None)
    torch.cuda.synchronize()
    return st


def _unit_case(b2a, kind, C, B, T, ctas, noise_kind="explicit", with_hl=False):
    """Runs one unit and returns (y, reference y, hl, reference hl in the dual layout, untouched x)."""
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(C * 1000 + T * 10 + B + (7 if kind == "noise" else kind))
    x = torch.randn(B * T, C, device=dev, generator=g)
    x_keep = x.clone()
    W = torch.randn(C, C, device=dev, generator=g) / math.sqrt(C)
    y = torch.full((B * T + 5, C), float("nan"), device=dev)
    kw = {}
    if kind == "noise":
        mode, dil = MODE_NOISE, 0
        if noise_kind == "seed":
            seed = 0xC0DEC + 17 * T
            nz = torch.from_numpy(gauss(seed, np.arange(B * T))).to(dev)
            kw["seed"] = seed
        else:
            nz = torch.randn(B * T, device=dev, generator=g).double()
            kw["noise"] = nz.float()
        ref = x.double() + nz[:, None] * pointwise(x, W)
    else:
        mode, dil = MODE_RU, kind
        dw_w = 0.4 * torch.randn(C, 7, device=dev, generator=g)
        dw_b = 0.1 * torch.randn(C, device=dev, generator=g)
        a_in = 0.5 + torch.rand(C, device=dev, generator=g)
        a_mid = 0.5 + torch.rand(C, device=dev, generator=g)
        pw_bias = 0.1 * torch.randn(C, device=dev, generator=g)
        kw.update(dw_w=dw_w, dw_b=dw_b, a_in=a_in, a_mid=a_mid, pw_bias=pw_bias)
        ref = x.double() + pointwise(snake(dwconv7(snake(x, a_in), dw_w, dw_b, dil, B), a_mid), W, pw_bias)
    hl = hl_ref = None
    if with_hl:
        a_next = 0.5 + torch.rand(C, device=dev, generator=g)
        hl_ref = dual_layout(snake(ref, a_next), B, T)
        hl = nan_hilo_buffer(B * (T + 1) + 1, 2 * C)
        kw.update(hl=hl, a_next=a_next)
    st = unit(b2a, mode, C, dil, x, y, B, T, W.cpu().numpy(), ctas=ctas, **kw)
    assert st == 0, b2a._ffi.lib().b2a_last_error()
    assert torch.equal(x, x_keep), "the unit wrote its input"
    assert y[B * T:].isnan().all(), "rows past the last token were written"
    return y[:B * T], ref, hl, hl_ref


@pytest.mark.parametrize("B,T", SHAPES, ids=[f"B{b}-T{t}" for b, t in SHAPES])
@pytest.mark.parametrize("ctas", [0, 1], ids=["engine-ctas", "one-cta"])
@pytest.mark.parametrize("C", [64, 128])
@pytest.mark.parametrize("kind", [1, 3, 9, "noise"], ids=["ru-dil1", "ru-dil3", "ru-dil9", "noise"])
def test_unit_matches_float64(b2a, kind, C, ctas, B, T):
    """y = x + W Snake(dwconv7_dil(Snake(x)) + b) + b_pw (ResidualUnit) or x + n[t] (W x) (NoiseBlock, explicit noise)."""
    y, ref, _, _ = _unit_case(b2a, kind, C, B, T, ctas)
    assert_close(f"{kind} C{C}", y, ref, REL_TOL, PEAK_TOL)


@pytest.mark.parametrize("B,T", [(2, 20), (1, 300)])
@pytest.mark.parametrize("ctas", [0, 1], ids=["engine-ctas", "one-cta"])
@pytest.mark.parametrize("C", [64, 128])
def test_seeded_noise_is_the_draw_of_each_token(b2a, C, ctas, B, T):
    """With no explicit noise the NoiseBlock draws cg::gauss(seed, b*T + t): a wrong token index would pass a statistical check."""
    y, ref, _, _ = _unit_case(b2a, "noise", C, B, T, ctas, noise_kind="seed")
    assert_close(f"seeded noise C{C}", y, ref, REL_TOL, PEAK_TOL)


@pytest.mark.parametrize("B,T", [(2, 20), (2, 100), (1, 300)])
@pytest.mark.parametrize("ctas", [0, 1], ids=["engine-ctas", "one-cta"])
@pytest.mark.parametrize("C", [64, 128])
@pytest.mark.parametrize("dil", [1, 9])
def test_unit_hilo_copy_is_the_next_im2col(b2a, dil, C, ctas, B, T):
    """The last unit of a block can also write Snake(a_next, y) as the next block's 2-tap im2col (hi/lo tiles, ld 2C): token (b, t)
    at row b*(T+1) + t, columns [0, C), and row b*(T+1) + t + 1, columns [C, 2C).  The edge half-rows and everything past the last
    row keep the NaN sentinel."""
    y, ref, hl, hl_ref = _unit_case(b2a, dil, C, B, T, ctas, with_hl=True)
    assert_close(f"dil{dil} C{C} y", y, ref, REL_TOL, PEAK_TOL)
    check_hilo_output(f"dil{dil} C{C}", hl, hl_ref, REL_TOL, PEAK_TOL)


CONVT_SHAPES = [(2, 64), (1, 128)]                                # (stride, cout): 128 input channels -> 128 phase rows


@pytest.mark.parametrize("Tin", [63, 64, 77])
@pytest.mark.parametrize("ctas", [0, 1], ids=["engine-ctas", "one-cta"])
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "no-bias"])
@pytest.mark.parametrize("stride,cout", CONVT_SHAPES)
def test_convt_matches_float64(b2a, stride, cout, bias, ctas, Tin):
    """y = conv_transpose1d(Snake(x), W, b, stride, padding ceil(stride / 2)), Tin*stride outputs per utterance, two utterances.
    Tin = 63 and 64 put q = Tin (the last input position of a tile) on either side of a 64-token tile edge."""
    dev, B = "cuda", 2
    g = torch.Generator(device=dev).manual_seed(stride * 100 + Tin + (1000 if bias else 0))
    x = torch.randn(B * Tin, 128, device=dev, generator=g)
    alpha = 0.5 + torch.rand(128, device=dev, generator=g)
    W = torch.randn(128, cout, 2 * stride, device=dev, generator=g) / math.sqrt(256)
    b = 0.1 * torch.randn(cout, device=dev, generator=g) if bias else None
    Tout = Tin * stride
    y = torch.full((B * Tout + 5, cout), float("nan"), device=dev)
    f = b2a._ffi
    w_host = W.cpu().numpy()                                      # the hook reads it: it must outlive the call
    st = f.lib().b2a_snac_convt_test(f.ptr(x), f.ptr(y), f.ptr(alpha), f.ptr(b), f.ptr(w_host), B, Tin, stride, cout, ctas, None)
    torch.cuda.synchronize()
    assert st == 0, f.lib().b2a_last_error()
    ref = conv_transpose(snake(x, alpha), W, b, stride, B)
    assert_close(f"convt s{stride}", y[:B * Tout], ref, REL_TOL, PEAK_TOL)
    assert y[B * Tout:].isnan().all(), "rows past the last output were written"


def test_unused_shapes_are_rejected(b2a):
    dev = "cuda"
    f = b2a._ffi
    x = torch.zeros(64, 128, device=dev)
    y = torch.zeros(256, 128, device=dev)
    one = torch.ones(128, device=dev)
    w = np.zeros((128, 64, 8), np.float32)
    assert f.lib().b2a_snac_convt_test(f.ptr(x), f.ptr(y), f.ptr(one), None, f.ptr(w), 1, 64, 4, 32, 0, None) == f.ERR_INVALID_INPUT
    pw = np.zeros((64, 64), np.float32)
    assert unit(b2a, MODE_RU, 64, 5, x, y, 1, 64, pw, dw_w=one, a_in=one, a_mid=one) == f.ERR_INVALID_INPUT          # dilation 5
    assert unit(b2a, MODE_RU, 96, 1, x, y, 1, 64, pw, dw_w=one, a_in=one, a_mid=one) == f.ERR_INVALID_INPUT          # 96 channels
    assert unit(b2a, MODE_NOISE, 64, 0, x, y, 1, 64, pw, pw_bias=one) == f.ERR_INVALID_INPUT                          # biased noise
    assert unit(b2a, MODE_RU, 64, 1, x, x, 1, 64, pw, dw_w=one, a_in=one, a_mid=one) == f.ERR_INVALID_INPUT           # y aliases x
    assert not y.any()
