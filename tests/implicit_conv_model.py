"""numpy statement of the Args contract of ic::implicit_conv_kernel (csrc/conv_gemm.cuh).  Shared by the CPU data-flow
model (test_speech_tokenizer_design.py) and the gated GPU kernel test (test_gpu_implicit_conv.py).  Test infrastructure."""
import math

import numpy as np


def implicit_conv(Wg, cin, X, T, *, dil=1, shift0=0, up=1, bias=None, gamma=None, gelu=False, add=False, bias_twice_t0=False,
                  xo=None, hl=None, Hout=0, sa=None, sb=None):
    """The Args contract of ic::implicit_conv_kernel.  X: planes as one float64 array [B, Ttot, cin]; xo [B, T*up, Cout] and
    hl [B, Hout + T*up, Cout] are written in place."""
    M, taps, _ = Wg.shape
    B, Ttot, _ = X.shape
    Cout = M // up
    acc = np.zeros((B, T, M))
    for j in range(taps):
        for t in range(T):
            f = t + shift0 + j * dil
            if 0 <= f < Ttot:                                      # out-of-range frames are TMA zero fill
                acc[:, t, :] += X[:, f, :] @ Wg[:, j, :cin].T
    for rho in range(up):
        val = acc[:, :, rho * Cout:(rho + 1) * Cout].copy()
        if bias is not None:
            val += bias
            if bias_twice_t0:
                val[:, 0, :] += bias
        if gelu:
            val = 0.5 * val * (1.0 + np.vectorize(math.erf)(val / math.sqrt(2.0)))
        if gamma is not None:
            val = val * gamma
        fo = np.arange(T) * up + rho
        if add:
            val = val + xo[:, fo, :]
        if xo is not None:
            xo[:, fo, :] = val
        if hl is not None:
            hv = val + sb * np.sin(sa * val) ** 2 if sa is not None else val
            hl[:, Hout + fo, :] = hv


OPERAND = "bf16"          # "fp16": what Args::f16 selects (the decoder default; B2A_ST_FP16=0 = bf16)


def _bf16(x):
    import torch
    kind = torch.bfloat16 if OPERAND == "bf16" else torch.float16
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(kind).to(torch.float32).numpy().astype(np.float64)


def implicit_conv_hilo(Wg, cin, X, T, *, dil=1, shift0=0, up=1, bias=None, gamma=None, gelu=False, add=False, bias_twice_t0=False,
                       xo=None, hl=None, Hout=0, sa=None, sb=None):
    """Same contract with the kernel's ARITHMETIC: weights and activations as bf16 (or, with OPERAND = "fp16", fp16) hi + lo, the three tensor-core products
    Wh*Xh + Wh*Xl + Wl*Xh (Wl*Xl dropped), fp32 accumulator / epilogue values, hi/lo planes on output.  Used to predict the
    numerical error of the CUDA path before it has run."""
    Wh = _bf16(Wg); Wl = _bf16(Wg - Wh)
    Xh = _bf16(X); Xl = _bf16(X - Xh)
    B, M = X.shape[0], Wg.shape[0]
    Cout = M // up
    a1, a2 = np.zeros((B, T * up, Cout)), np.zeros((B, T * up, Cout))
    implicit_conv(Wh + Wl, cin, Xh, T, dil=dil, shift0=shift0, up=up, xo=a1)
    implicit_conv(Wh, cin, Xl, T, dil=dil, shift0=shift0, up=up, xo=a2)
    acc = (a1 + a2).astype(np.float32).astype(np.float64)
    for rho in range(up):
        fo = np.arange(T) * up + rho
        val = acc[:, fo, :].copy()
        if bias is not None:
            val += bias
            if bias_twice_t0:
                val[:, 0, :] += bias
        if gelu:
            val = 0.5 * val * (1.0 + np.vectorize(math.erf)(val / math.sqrt(2.0)))
        if gamma is not None:
            val = val * gamma
        if add:
            val = val + xo[:, fo, :]
        val = val.astype(np.float32).astype(np.float64)
        if xo is not None:
            xo[:, fo, :] = val
        if hl is not None:
            hv = val + sb * np.sin(sa * val) ** 2 if sa is not None else val
            hi = _bf16(hv)
            hl[:, Hout + fo, :] = hi + _bf16(hv - hi)
