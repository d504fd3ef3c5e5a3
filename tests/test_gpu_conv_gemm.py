"""The codec conv GEMM (cg::conv_gemm_kernel, csrc/conv_gemm.cu) in isolation through b2a_conv_gemm_test, one case per engine
call site at that call site's shapes, against float64.

The kernel multiplies the fp32 weight, split into bf16 hi + lo, by fp32 activations given as bf16 hi/lo tiles, and drops the
Wl * Xl product; the references use the exact fp32 weight and activations.  Every output is checked: the fp32 x, the hi/lo
copy read back as hi + lo (each lo within ulp(hi)/2), the dual 2-tap im2col layout, and the NaN sentinel in every cell the
epilogue must not write (the im2col edge cells x2_zero_edges_kernel owns, rows past the last token, columns past the output).

Tolerances: measured on an H100 80GB HBM3 at a 400 W power limit, the worst case was relative L2 6.7e-6 and max/peak 8.5e-6
(both the hi/lo copy of SNAC block 0's transposed conv, K = 2048).  Bounds: 2e-5 and 3e-5, about 3x the worst case.  The seeded
NoiseBlock and the same launch given the model's draws agreed to 9.1e-8 relative L2 and 5.0e-7 max/peak (the device's logf and
cospif against float64); bounds 3e-7 and 1.5e-6."""
import math

import numpy as np
import pytest
import torch

from codec_reference import check_hilo_output, dual_layout, gauss, nan_hilo_buffer, snake
from gemm_reference import assert_close, hilo_tiles

pytestmark = pytest.mark.gpu

E_STORE_HILO, E_CONVT, E_NOISE, E_ADD, E_ADD_HILO, E_STORE_F32 = range(6)          # csrc/conv_gemm.cuh
REL_TOL, PEAK_TOL = 2e-5, 3e-5


def conv_gemm(b2a, w, M, K, X, N, epi, bias=None, alpha=None, gamma=None, gelu=0, x=None, ldx=0, hl=None, ldh=0, dual=0, T=0,
              Cout=0, stride=0, pad=0, Tin=0, noise=None, seed=0, ctas=0) -> int:
    f = b2a._ffi
    st = f.lib().b2a_conv_gemm_test(f.ptr(w), M, K, f.ptr(X), N, epi, f.ptr(bias), f.ptr(alpha), f.ptr(gamma), gelu, f.ptr(x), ldx,
                                    f.ptr(hl), ldh, dual, T, Cout, stride, pad, Tin, f.ptr(noise), seed, ctas, None)
    torch.cuda.synchronize()
    return st


# name: (M, K, epilogue and options, B, T (tokens per utterance; Tin for E_CONVT))
SNAC = {   # SNAC 24 kHz: latent 768, decoder 1024, rates 8 8 4 2 (csrc/snac.cu decode_dev_tc)
    "snac-pw0-dual": (1024, 768, dict(epi=E_STORE_HILO, bias=1, alpha=1, dual=1), 2, 13),
    "snac-convt0-hl": (4096, 2048, dict(epi=E_CONVT, bias=1, hl=1, stride=8, cout=512), 2, 13),
    "snac-convt0-hl-looping": (4096, 2048, dict(epi=E_CONVT, bias=1, hl=1, stride=8, cout=512, ctas=5), 1, 64),
    "snac-convt1-hl": (2048, 1024, dict(epi=E_CONVT, bias=1, hl=1, stride=8, cout=256), 2, 20),
    "snac-convt2": (512, 512, dict(epi=E_CONVT, bias=1, stride=4, cout=128), 3, 50),
    "snac-noise512-explicit": (512, 512, dict(epi=E_NOISE, noise="explicit"), 2, 104),
    "snac-noise512-seed": (512, 512, dict(epi=E_NOISE, noise="seed"), 2, 104),
    "snac-noise256-seed": (256, 256, dict(epi=E_NOISE, noise="seed"), 2, 150),
    "snac-add512": (512, 512, dict(epi=E_ADD, bias=1), 2, 104),
    "snac-add256": (256, 256, dict(epi=E_ADD, bias=1), 2, 150),
    "snac-addhilo512-dual": (512, 512, dict(epi=E_ADD_HILO, bias=1, alpha=1, dual=1), 2, 104),
    "snac-addhilo256-dual": (256, 256, dict(epi=E_ADD_HILO, bias=1, alpha=1, dual=1), 2, 150),
    "snac-addhilo256-looping": (256, 256, dict(epi=E_ADD_HILO, bias=1, alpha=1, dual=1, ctas=3), 3, 333),
}
VOCOS = {  # csrc/vocos.cu decode_dev; default geometry (100 -> 512, 1536, n_fft 1024, kernel 7) and Soprano's (512 -> 768, 2304, 2048)
    "vocos-embed-k700": (512, 704, dict(epi=E_STORE_F32, bias=1, k_used=700), 2, 37),
    "vocos-pwconv1-gelu": (1536, 512, dict(epi=E_STORE_HILO, bias=1, gelu=1), 2, 37),
    "vocos-pwconv2-gamma": (512, 1536, dict(epi=E_ADD, bias=1, gamma=1), 2, 37),
    "vocos-head": (1026, 512, dict(epi=E_STORE_F32, bias=1), 2, 37),
    "vocos-head-padded-ldx": (1026, 512, dict(epi=E_STORE_F32, bias=1, ldx=1088), 2, 37),
    "vocos-idft": (1024, 1088, dict(epi=E_STORE_F32), 2, 37),
    "soprano-embed": (768, 512, dict(epi=E_STORE_F32, bias=1), 2, 37),
    "soprano-pwconv1-gelu": (2304, 768, dict(epi=E_STORE_HILO, bias=1, gelu=1), 2, 37),
    "soprano-pwconv2-gamma": (768, 2304, dict(epi=E_ADD, bias=1, gamma=1), 2, 37),
    "soprano-head": (2050, 768, dict(epi=E_STORE_F32, bias=1), 2, 37),
    "soprano-idft": (2048, 2112, dict(epi=E_STORE_F32), 1, 130),
}
CASES = {**SNAC, **VOCOS}


@pytest.mark.parametrize("name", list(CASES))
def test_call_site_matches_float64(b2a, name):
    """The call site's weight shape, epilogue and options on random fp32 data; ctas = 0 is the engine's min(SM count, tiles), and
    the *-looping cases give each CTA several tiles."""
    M, K, c, B, T = CASES[name]
    epi, dev = c["epi"], "cuda"
    g = torch.Generator(device=dev).manual_seed(sum(map(ord, name)))
    convt = epi == E_CONVT
    N = B * (T + 1) if convt else B * T                        # E_CONVT: tokens (b, q), q = 0 .. Tin
    ku = c.get("k_used", K)                                     # the embed conv's K = 700 is zero-padded to 704
    W = torch.zeros(M, K, device=dev)
    W[:, :ku] = torch.randn(M, ku, device=dev, generator=g) / math.sqrt(ku)
    xin = torch.zeros(N, K, device=dev)
    xin[:, :ku] = torch.randn(N, ku, device=dev, generator=g)
    X, _ = hilo_tiles(xin, 128)
    acc = xin.double() @ W.double().T
    bias = 0.2 * torch.randn(c["cout"] if convt else M, device=dev, generator=g) if c.get("bias") else None
    alpha = 0.5 + torch.rand(M, device=dev, generator=g) if c.get("alpha") else None
    gamma = 0.5 + torch.rand(M, device=dev, generator=g) if c.get("gamma") else None
    v = acc
    if convt:
        s, cout = c["stride"], c["cout"]
        pad, Tout = (s + 1) // 2, T * s
        # row m = r*cout + co of token (b, q) -> output token b*Tout + q*s + r - pad, kept inside [0, Tout)
        full = acc.view(B, T + 1, s, cout).reshape(B, (T + 1) * s, cout)
        v = full[:, pad:pad + Tout].reshape(B * Tout, cout)
        if bias is not None:
            v = v + bias.double()
        rows, cols = B * Tout, cout
    else:
        if bias is not None:
            v = v + bias.double()
        if c.get("gelu"):
            v = 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))
        if gamma is not None:
            v = v * gamma.double()
        rows, cols = N, M
    ldx = c.get("ldx", cols)
    x = hl = noise = None
    x_ref = hl_ref = None
    seed = 0
    if epi != E_STORE_HILO:
        x = torch.full((rows + 3, ldx), float("nan"), device=dev)
        if epi in (E_NOISE, E_ADD, E_ADD_HILO):
            x0 = torch.randn(rows, cols, device=dev, generator=g)
            x[:rows, :cols] = x0
            if epi == E_NOISE:
                seed = 0x5EED0000 + M if c["noise"] == "seed" else 0
                nz = torch.from_numpy(gauss(seed, np.arange(N))).to(dev) if seed else torch.randn(N, device=dev, generator=g).double()
                noise = None if seed else nz.float()
                x_ref = x0.double() + nz[:, None] * v
            else:
                x_ref = x0.double() + v
        else:
            x_ref = v
    dual = c.get("dual", 0)
    if epi in (E_STORE_HILO, E_ADD_HILO) or c.get("hl"):
        hv = x_ref if epi == E_ADD_HILO else v
        if alpha is not None:
            hv = snake(hv, alpha)
        if dual:
            hl_ref, ldh = dual_layout(hv, B, T), 2 * M
        else:
            hl_ref, ldh = hv, cols
        hl = nan_hilo_buffer(hl_ref.shape[0] + 1, ldh)
    st = conv_gemm(b2a, W.cpu().numpy(), M, K, X, N, epi, bias=bias, alpha=alpha, gamma=gamma, gelu=c.get("gelu", 0), x=x, ldx=ldx,
                   hl=hl, ldh=hl.shape[1] if hl is not None else 0, dual=dual, T=T * c["stride"] if convt else T,
                   Cout=c.get("cout", 0), stride=c.get("stride", 0), pad=(c["stride"] + 1) // 2 if convt else 0,
                   Tin=T if convt else 0, noise=noise, seed=seed, ctas=c.get("ctas", 0))
    assert st == 0, b2a._ffi.lib().b2a_last_error()
    if x is not None:
        assert_close(name + " x", x[:rows, :cols], x_ref, REL_TOL, PEAK_TOL)
        assert x[rows:].isnan().all() and x[:, cols:].isnan().all(), "x written outside its rows / columns"
    if hl is not None:
        check_hilo_output(name, hl, hl_ref, REL_TOL, PEAK_TOL)
    if epi == E_NOISE and seed:
        # the seeded draw is the one for token b*T + t: the same launch given those draws explicitly agrees to fp32 rounding
        x2 = torch.full_like(x, float("nan"))
        x2[:rows, :cols] = x0
        st = conv_gemm(b2a, W.cpu().numpy(), M, K, X, N, epi, x=x2, ldx=ldx, noise=torch.from_numpy(gauss(seed, np.arange(N))).float().to(dev))
        assert st == 0, b2a._ffi.lib().b2a_last_error()
        assert_close(name + " seeded vs explicit", x[:rows], x2[:rows], 3e-7, 1.5e-6)


@pytest.mark.parametrize("why,kw", [
    ("GELU outside pwconv1", dict(epi=E_ADD, gelu=1)),
    ("gamma outside the ConvNeXt add", dict(epi=E_STORE_F32, gamma=1)),
    ("Snake on an fp32-only output", dict(epi=E_ADD, alpha=1)),
    ("E_ADD_HILO without the 2-tap im2col", dict(epi=E_ADD_HILO, hl=1, alpha=1)),
    ("noise outside E_NOISE", dict(epi=E_ADD, noise=1)),
    ("E_CONVT with M != stride * Cout", dict(epi=E_CONVT, Cout=100, stride=2, Tin=3)),
    ("dual outputs of a partial utterance", dict(epi=E_STORE_HILO, hl=1, dual=1, T=5)),
])
def test_unused_combinations_are_rejected(b2a, why, kw):
    M, K, N = 256, 128, 8
    dev = "cuda"
    X = torch.zeros(2 * 64, K, device=dev, dtype=torch.bfloat16)
    x = torch.zeros(N + 64, 2 * M, device=dev)
    hl = torch.zeros(128, 2 * M, device=dev, dtype=torch.bfloat16) if kw.get("hl") else None
    ones = torch.ones(M, device=dev)
    st = conv_gemm(b2a, np.zeros((M, K), np.float32), M, K, X, N, kw["epi"], alpha=ones if kw.get("alpha") else None,
                   gamma=ones if kw.get("gamma") else None, gelu=kw.get("gelu", 0), x=None if kw["epi"] == E_STORE_HILO else x, ldx=2 * M,
                   hl=hl, ldh=2 * M, dual=kw.get("dual", 0), T=kw.get("T", 0), Cout=kw.get("Cout", 0), stride=kw.get("stride", 0),
                   Tin=kw.get("Tin", 0), noise=torch.ones(N, device=dev) if kw.get("noise") else None)
    assert st == b2a._ffi.ERR_INVALID_INPUT, why
    assert not x.any() and (hl is None or not hl.any())
