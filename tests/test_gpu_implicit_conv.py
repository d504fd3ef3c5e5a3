"""The implicit-GEMM causal convolution kernel (csrc/conv_gemm.cu) alone, through b2a_implicit_conv_test and the engines' launch
(ic::launch), against its numpy contract (tests/implicit_conv_model.py).  (row N1)."""
import os

import numpy as np
import pytest

from implicit_conv_model import implicit_conv

pytestmark = pytest.mark.gpu


def run(b2a, w, x, T, *, dil=1, shift0=0, up=1, bias=None, gamma=None, gelu=False, add=None, twice=False, sa=None, sb=None, Hout=0, want_xo=True, want_hl=True, fp16=0):
    f = b2a._ffi
    M, taps, cin = w.shape
    B, Ttot, _ = x.shape
    cout = M // up
    c32 = lambda a: None if a is None else np.ascontiguousarray(a, np.float32)
    xo = (np.zeros((B, T * up, cout), np.float32) if add is None else c32(add).copy()) if want_xo else None
    hl = np.zeros((B, Hout + T * up, cout), np.float32) if want_hl else None
    w32, x32, b32, g32, sa32, sb32 = c32(w), c32(x), c32(bias), c32(gamma), c32(sa), c32(sb)
    f.check(f.lib().b2a_implicit_conv_test(f.ptr(w32), M, taps, cin, f.ptr(x32), B, Ttot, T, dil, shift0, up, f.ptr(b32), f.ptr(g32), int(gelu),
                                           int(add is not None), int(twice), f.ptr(sa32), f.ptr(sb32), Hout, fp16, f.ptr(xo), f.ptr(hl)))
    return xo, hl


def model(w, x, T, *, add=None, Hout=0, up=1, want_xo=True, want_hl=True, twice=False, **kw):
    M, _, cin = w.shape
    B = x.shape[0]
    cout = M // up
    xo = (np.zeros((B, T * up, cout)) if add is None else np.asarray(add, np.float64).copy()) if want_xo else None
    hl = np.zeros((B, Hout + T * up, cout)) if want_hl else None
    wp = np.zeros((M, w.shape[1], (cin + 63) // 64 * 64))
    wp[:, :, :cin] = w
    implicit_conv(wp, cin, np.asarray(x, np.float64), T, up=up, add=add is not None, bias_twice_t0=twice, xo=xo, hl=hl, Hout=Hout, **kw)
    return xo, hl


def close(a, b, tol=2e-5):
    return np.abs(a - b).max() <= tol * max(1.0, np.abs(b).max())


@pytest.mark.parametrize("M,taps,cin,B,T,dil", [(128, 1, 64, 1, 64, 1), (96, 7, 96, 2, 150, 1), (200, 7, 72, 2, 70, 3), (136, 3, 128, 3, 37, 9), (384, 2, 256, 1, 5, 1)])
def test_plain_causal_conv(b2a, M, taps, cin, B, T, dil):
    rng = np.random.default_rng(M + T)
    H = (taps - 1) * dil
    w = rng.standard_normal((M, taps, cin)) / np.sqrt(taps * cin)
    x = rng.standard_normal((B, H + T, cin))
    bias = rng.standard_normal(M)
    xo, hl = run(b2a, w, x, T, dil=dil, bias=bias, Hout=5)
    rx, rh = model(w.astype(np.float32), x.astype(np.float32), T, dil=dil, bias=bias.astype(np.float32), Hout=5)
    assert close(xo, rx) and close(hl, rh) and not hl[:, :5].any()


def test_frames_beyond_the_input_are_zero_fill(b2a):
    rng = np.random.default_rng(1)
    w = rng.standard_normal((64, 3, 64)) / 14
    x = rng.standard_normal((1, 10, 64))                            # Ttot = 10 < T + (taps-1)
    xo, _ = run(b2a, w, x, 12, shift0=1, want_hl=False)
    rx, _ = model(w.astype(np.float32), x.astype(np.float32), 12, shift0=1, want_hl=False)
    assert close(xo, rx)


@pytest.mark.parametrize("up,taps", [(2, 1), (8, 2), (3, 2)])
def test_phase_major_transposed_conv_epilogue(b2a, up, taps):
    rng = np.random.default_rng(up)
    cout, cin, B, T = 48, 96, 2, 67
    w = rng.standard_normal((up * cout, taps, cin)) / np.sqrt(taps * cin)
    x = rng.standard_normal((B, taps - 1 + T, cin))
    bias, sa, sb = rng.standard_normal(cout), np.exp(rng.standard_normal(cout) * 0.3), np.exp(rng.standard_normal(cout) * 0.3)
    for twice in (False, True):
        xo, hl = run(b2a, w, x, T, up=up, bias=bias, sa=sa, sb=sb, Hout=6, twice=twice)
        rx, rh = model(w.astype(np.float32), x.astype(np.float32), T, up=up, bias=bias.astype(np.float32), sa=sa.astype(np.float32), sb=sb.astype(np.float32), Hout=6, twice=twice)
        assert close(xo, rx) and close(hl, rh, 5e-5)


def test_gelu_gamma_residual(b2a):
    rng = np.random.default_rng(7)
    M, cin, B, T = 256, 64, 2, 100
    w = rng.standard_normal((M, 1, cin)) / 8
    x = rng.standard_normal((B, T, cin))
    bias, gamma, res = rng.standard_normal(M), rng.standard_normal(M), rng.standard_normal((B, T, M))
    _, hl = run(b2a, w, x, T, bias=bias, gelu=True, want_xo=False)
    _, rh = model(w.astype(np.float32), x.astype(np.float32), T, bias=bias.astype(np.float32), gelu=True, want_xo=False)
    assert close(hl, rh)
    xo, hl = run(b2a, w, x, T, bias=bias, gamma=gamma, add=res)
    rx, rh = model(w.astype(np.float32), x.astype(np.float32), T, bias=bias.astype(np.float32), gamma=gamma.astype(np.float32), add=res.astype(np.float32))
    assert close(xo, rx) and close(hl, rh)


def test_fp16_operand_pairs(b2a):
    """Same contract with fp16 hi/lo operands (Args::f16, the decoder default; B2A_ST_FP16=0 selects bf16 pairs): 22 mantissa bits per operand instead of 16."""
    rng = np.random.default_rng(9)
    w = rng.standard_normal((192, 7, 96)) / np.sqrt(7 * 96)
    x = rng.standard_normal((2, 54 + 130, 96)) * 3.0
    bias = rng.standard_normal(192)
    xo16, hl16 = run(b2a, w, x, 130, dil=9, bias=bias, fp16=1)
    xob, _ = run(b2a, w, x, 130, dil=9, bias=bias, fp16=0)
    rx, rh = model(w.astype(np.float32), x.astype(np.float32), 130, dil=9, bias=bias.astype(np.float32))
    e16, eb = np.abs(xo16 - rx).max(), np.abs(xob - rx).max()
    assert e16 < 4e-6 * max(1.0, np.abs(rx).max()) and close(hl16, rh, 2e-6)
    assert e16 < eb                                               # and it is the more accurate of the two formats
