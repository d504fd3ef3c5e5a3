"""float64 references and checks shared by the codec kernel tests (test_gpu_conv_gemm.py, test_gpu_snac_fused.py).

Activations are channels-last: [tokens, channels], token b*T + t for utterance b.  The references take the exact fp32 inputs the
kernels are given; what is left is the kernels' bf16 hi/lo splits of weights and activations, the dropped Wl*Xl product, fp32
arithmetic and the kernels' sin (|error| < 5e-7)."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from gemm_reference import assert_close, assert_lo_within_half_ulp, hilo_rows


def snake(x: torch.Tensor, alpha: torch.Tensor) -> torch.Tensor:
    """Snake over the last (channel) axis: x + sin(alpha x)^2 / (alpha + 1e-9)."""
    x, a = x.double(), alpha.double()
    return x + torch.sin(a * x) ** 2 / (a + 1e-9)


def pointwise(x: torch.Tensor, W: torch.Tensor, bias=None) -> torch.Tensor:
    """1x1 conv: [N, Cin] x W [Cout, Cin] (+ bias) -> [N, Cout]."""
    return F.linear(x.double(), W.double(), None if bias is None else bias.double())


def dwconv7(x: torch.Tensor, w: torch.Tensor, b, dil: int, B: int) -> torch.Tensor:
    """Depthwise conv, kernel 7, dilation dil, 'same' zero padding within each utterance: [B*T, C], w [C, 7] -> [B*T, C]."""
    C = x.shape[1]
    xt = x.double().view(B, -1, C).transpose(1, 2)
    y = F.conv1d(xt, w.double().view(C, 1, 7), None if b is None else b.double(), padding=3 * dil, dilation=dil, groups=C)
    return y.transpose(1, 2).reshape(-1, C)


def conv_transpose(x: torch.Tensor, W: torch.Tensor, b, stride: int, B: int) -> torch.Tensor:
    """SNAC's transposed conv (kernel 2*stride, padding ceil(stride / 2)) of [B*Tin, Cin], W [Cin, Cout, 2*stride] in torch layout,
    as Tin*stride outputs per utterance: [B*Tin*stride, Cout].  For even strides this is F.conv_transpose1d(..., padding=ceil(stride/2))
    itself; for odd ones that call returns one output fewer, and the last output here is the next sample of the same convolution."""
    Cin, Cout = W.shape[0], W.shape[1]
    pad = (stride + 1) // 2
    xt = x.double().view(B, -1, Cin).transpose(1, 2)
    Tin = xt.shape[2]
    y = F.conv_transpose1d(xt, W.double(), None if b is None else b.double(), stride=stride)     # full: (Tin + 1) * stride outputs
    return y[:, :, pad:pad + Tin * stride].transpose(1, 2).reshape(-1, Cout)


def gauss(seed: int, idx) -> np.ndarray:
    """The kernels' counter-based N(0, 1) draw (csrc/conv_gemm.cuh cg::gauss): splitmix64 of seed + golden * (idx + 1), two 24-bit
    uniforms as fp32, then Box-Muller in float64.  float64 [len(idx)]."""
    with np.errstate(over="ignore"):
        i = np.asarray(idx, dtype=np.uint64)
        z = np.uint64(seed) + np.uint64(0x9E3779B97F4A7C15) * (i + np.uint64(1))
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    u1 = ((z >> np.uint64(40)).astype(np.float32) + np.float32(1.0)) * np.float32(1.0 / 16777217.0)
    u2 = (z >> np.uint64(8) & np.uint64(0xFFFFFF)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    return np.sqrt(-2.0 * np.log(u1.astype(np.float64))) * np.cos(math.pi * (2.0 * u2.astype(np.float64)))


def dual_layout(v: torch.Tensor, B: int, T: int) -> torch.Tensor:
    """The 2-tap im2col a transposed conv reads ("dual" outputs): token (b, t) of v [B*T, C] goes to row b*(T+1) + t, columns
    [0, C), and to row b*(T+1) + t + 1, columns [C, 2C).  [B*(T+1), 2C] float64, NaN in the two half-rows per utterance no token
    writes (row b*(T+1) columns [C, 2C), row b*(T+1) + T columns [0, C))."""
    C = v.shape[1]
    e = torch.full((B, T + 1, 2 * C), float("nan"), dtype=torch.float64, device=v.device)
    vv = v.double().view(B, T, C)
    e[:, :T, :C] = vv
    e[:, 1:, C:] = vv
    return e.view(B * (T + 1), 2 * C)


def nan_hilo_buffer(rows: int, ld: int, device="cuda") -> torch.Tensor:
    """A bf16 buffer of 64-token hi/lo tiles for `rows` token rows, filled with the NaN sentinel."""
    return torch.full((2 * 64 * (-(-rows // 64)), ld), float("nan"), dtype=torch.bfloat16, device=device)


def check_hilo_output(name: str, hl: torch.Tensor, expect: torch.Tensor, rel_tol: float, peak_tol: float):
    """hl: a NaN-filled bf16 tile buffer after the launch; expect: float64 [R, Cols], the value of token row r, column c, NaN where
    nothing may be written.  hi + lo must match expect, each lo must be within ulp(hi)/2 and every other cell must keep the NaN."""
    R, Cols = expect.shape
    hr, lr = hilo_rows(R, 128, hl.device)
    hi, lo = hl[hr][:, :Cols], hl[lr][:, :Cols]
    w = ~expect.isnan()
    assert_close(name + " hi+lo", hi.double()[w] + lo.double()[w], expect[w], rel_tol, peak_tol)
    assert_lo_within_half_ulp(hi[w], lo[w])
    assert hi[~w].isnan().all() and lo[~w].isnan().all(), f"{name}: hi/lo cells outside the written layout were overwritten"
    rest = torch.ones(hl.shape, dtype=torch.bool, device=hl.device)
    rest[hr, :Cols] = False
    rest[lr, :Cols] = False
    assert hl[rest].isnan().all(), f"{name}: rows or columns past the output were written"
