"""float64 references and checks shared by the GEMM kernel tests (test_gpu_tc_gemm.py, test_gpu_splitk_norm.py).

The kernels read activations as bf16 hi/lo pairs: X tiles of bn rows, rows [0, bn/2) = hi(x) = bf16(x), rows [bn/2, bn) = lo(x) =
bf16(x - hi), token t in tile t // (bn/2).  They write bf16 outputs the same way.  The references use the exact value hi + lo of
the pairs the kernel is given, so what is left is the kernel's own fp32 arithmetic."""
import torch

EPI_STORE, EPI_SWIGLU, EPI_STORE_BF16, EPI_ADD = 0, 2, 3, 4        # csrc/tc_gemm.cuh
ACT_GELU = 1


def run_tc_gemm(b2a, W, X, out, M, N, K, bn, epi, split, hilo, ctas, bias=None, act=0, tile_rows=0, lo_rows=0, rstd_ss=None,
                rstd_parts=0, rstd_eps=0.0, stages=0) -> int:
    """One b2a_tc_gemm_epilogue_test launch (include/b200audio_internal.h) on device tensors; returns the status."""
    f = b2a._ffi
    st = f.lib().b2a_tc_gemm_epilogue_test(f.ptr(W), f.ptr(X), f.ptr(out), M, N, K, bn, epi, split, hilo, ctas, f.ptr(bias), act, tile_rows,
                                           lo_rows, f.ptr(rstd_ss), rstd_parts, rstd_eps, stages, None)
    torch.cuda.synchronize()
    return st


def tc_gemm(b2a, *args, **kw):
    st = run_tc_gemm(b2a, *args, **kw)
    assert st == 0, b2a._ffi.lib().b2a_last_error()


def hilo_tiles(x: torch.Tensor, bn: int):
    """fp32 [N, K] -> (bf16 [cdiv(N, bn/2) * bn, K] in the kernel's tile layout, float64 [N, K] = hi + lo)."""
    half = bn // 2
    N, K = x.shape
    nt = -(-N // half)
    xp = torch.zeros(nt * half, K, device=x.device, dtype=torch.float32)
    xp[:N] = x
    hi = xp.to(torch.bfloat16)
    lo = (xp - hi.float()).to(torch.bfloat16)
    X = torch.stack([hi.view(nt, half, K), lo.view(nt, half, K)], 1).reshape(nt * bn, K).contiguous()
    return X, (hi.double() + lo.double())[:N]


def hilo_rows(N: int, bn: int, device="cuda"):
    """Row indices of the hi and lo rows of tokens 0..N-1 in a hi/lo tile layout of bn rows per tile."""
    half = bn // 2
    t = torch.arange(N, device=device)
    hi = (t // half) * bn + t % half
    return hi, hi + half


def errors(got: torch.Tensor, ref: torch.Tensor):
    """(relative L2 error, max |error| / max |ref|) in float64."""
    g, r = got.double(), ref.double()
    d = g - r
    return float(d.norm() / r.norm()), float(d.abs().max() / r.abs().max())


def assert_close(name: str, got, ref, rel_tol: float, peak_tol: float):
    rel, pk = errors(got, ref)
    print(f"{name}: rel L2 {rel:.2e}, max/peak {pk:.2e}")          # pytest -s shows the measured errors
    assert torch.isfinite(got).all(), name
    assert rel < rel_tol and pk < peak_tol, (name, rel, pk)


def assert_lo_within_half_ulp(hi: torch.Tensor, lo: torch.Tensor):
    """|lo| <= ulp(hi) / 2: lo is the rounded remainder of hi = bf16(v), not an independent value (bf16 has 8 significand bits)."""
    h, l = hi.float(), lo.float()
    _, e = torch.frexp(h)                                            # |h| = m 2^e, m in [0.5, 1): ulp = 2^(e - 8)
    bound = torch.ldexp(torch.ones_like(h), (e - 9).to(torch.int32))
    nz = h != 0
    assert (l[nz].abs() <= bound[nz]).all(), float((l[nz].abs() / bound[nz]).max())
