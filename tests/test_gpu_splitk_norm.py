"""The decode step's cluster split-K GEMM with the residual add and the next RMSNorm fused in (tc_gemm_splitk_kernel, through
b2a_tc_gemm_splitk_test) against float64 on the same bf16 weights and hi/lo activation pairs.  For tokens t < N:

    h'[t] = h[t] + W (x_hi[t] + x_lo[t])          xn[t], xn[8 + t] = hi / lo of h'[t] * gain          ss[m_tile, t] = sum h'[t]^2

and for t >= N: h[t] unchanged, xn rows untouched, ss = 0.  Shapes are the o_proj / down_proj GEMMs of Orpheus 3B (hidden 3072,
intermediate 8192), of the Qwen3-0.6B geometry (hidden 1024, 16 x 128 query features, intermediate 3072) and of the test models; the
cluster sizes are what the engine picks (min(5, k-blocks)) plus smaller ones, with k-block counts that do not divide evenly."""
import pytest
import torch

from gemm_reference import EPI_STORE, assert_close, assert_lo_within_half_ulp, hilo_tiles, tc_gemm

pytestmark = pytest.mark.gpu

STAGES = 5          # llama.cu splitk_gemm


def _splitk(b2a, W, X, h, gain, xn, ss, M, N, K, cluster):
    f = b2a._ffi
    st = f.lib().b2a_tc_gemm_splitk_test(f.ptr(W), f.ptr(X), f.ptr(h), f.ptr(gain), f.ptr(xn), f.ptr(ss), M, N, K, cluster, STAGES, None)
    torch.cuda.synchronize()
    assert st == 0, f.lib().b2a_last_error()


def _inputs(M, K, N, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    W = (torch.randn(M, K, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    x = torch.randn(8, K, device="cuda", generator=g)                  # rows >= N hold data too: they must not reach h, xn or ss
    X, xe = hilo_tiles(x, 16)
    h = torch.randn(8, M, device="cuda", generator=g)
    gain = 1.0 + 0.2 * torch.randn(M, device="cuda", generator=g)
    return W, X, xe, h, gain


def _run_and_check(b2a, M, K, N, cluster, seed):
    """One split-K launch on fresh inputs, every output checked against float64."""
    W, X, xe, h0, gain = _inputs(M, K, N, seed)
    h = h0.clone()
    mt = -(-M // 128)
    xn = torch.full((16, M), float("nan"), device="cuda", dtype=torch.bfloat16)
    ss = torch.full((mt, 8), float("nan"), device="cuda")
    _splitk(b2a, W, X, h, gain, xn, ss, M, N, K, cluster)
    ref_h = h0[:N].double() + xe[:N] @ W.double().T
    assert_close("h", h[:N], ref_h, 1e-5, 2e-5)
    assert torch.equal(h[N:], h0[N:])
    ref_xn = ref_h * gain.double()
    assert_close("xn", xn[:N].double() + xn[8:8 + N].double(), ref_xn, 1e-5, 2e-5)
    assert_lo_within_half_ulp(xn[:N], xn[8:8 + N])
    assert xn[N:8].isnan().all() and xn[8 + N:].isnan().all()
    ref_ss = (ref_h ** 2).view(N, mt, 128).sum(-1).T
    assert_close("ss", ss[:, :N], ref_ss, 1e-5, 2e-5)
    assert (ss[:, N:] == 0).all()


CASES = [
    # M, K, cluster, N                                k-blocks % cluster
    (3072, 3072, 5, 8),      # Orpheus o_proj        48 % 5 = 3
    (3072, 8192, 5, 8),      # Orpheus down_proj     128 % 5 = 3
    (3072, 3072, 4, 3),
    (1024, 2048, 5, 3),      # Qwen3-0.6B o_proj     32 % 5 = 2
    (1024, 3072, 5, 1),      # Qwen3-0.6B down_proj  48 % 5 = 3
    (1024, 2048, 2, 8),
    (256, 256, 4, 8),        # test model o_proj: 4 k-blocks, cluster min(5, 4)
    (256, 256, 1, 1),
    (128, 384, 5, 3),        # 6 % 5 = 1
    (128, 384, 4, 8),        # 6 % 4 = 2
    (128, 384, 1, 8),
]


@pytest.mark.parametrize("M,K,cluster,N", CASES)
def test_splitk_norm_matches_float64(b2a, M, K, cluster, N):
    """Measured on an H100 80GB HBM3, worst case over all cases (relative L2 / max over peak): h 1.4e-6 / 1.5e-6, xn 2.9e-6 / 5.6e-6
    (the bf16 hi/lo pair), ss 2.2e-6 / 2.1e-6.  Bounds: 1e-5 / 2e-5, at least 3.5x the worst case."""
    _run_and_check(b2a, M, K, N, cluster, seed=M + K + cluster + N)


@pytest.mark.parametrize("H,nq,nkv,N", [(1024, 16, 8, 8), (256, 2, 1, 3)])
def test_splitk_sums_of_squares_feed_the_qkv_rstd(b2a, H, nq, nkv, N):
    """The step's hand-off: the split-K GEMM leaves xn = hi / lo of h * gain and ss; the next q|k|v GEMM (tc_gemm_kernel<16>,
    stream-K) scales by rsqrt(sum(ss) / H + eps).  Together they must equal a float64 RMSNorm followed by the matmul.
    Measured on an H100 80GB HBM3: relative L2 2.5e-6, max/peak 2.7e-6; bound 1e-5 for both."""
    I = 3 * H                                                       # down_proj: K = intermediate size
    W, X, xe, h0, gain = _inputs(H, I, N, seed=H + N)
    h = h0.clone()
    xn = torch.zeros(16, H, device="cuda", dtype=torch.bfloat16)
    ss = torch.zeros(H // 128, 8, device="cuda")
    _splitk(b2a, W, X, h, gain, xn, ss, H, N, I, min(5, I // 64))
    eps = 1e-5
    ref_h = h0[:N].double() + xe[:N] @ W.double().T
    M = (nq + 2 * nkv) * 128
    Wq = (torch.randn(M, H, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7)) * 0.05).to(torch.bfloat16)
    normed = ref_h / torch.sqrt((ref_h ** 2).mean(-1, keepdim=True) + eps) * gain.double()
    ref = normed @ Wq.double().T
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    out = torch.full((8, M), float("nan"), device="cuda")
    out[:N] = 0
    tc_gemm(b2a, Wq, xn, out, M, N, H, 16, EPI_STORE, 1, 1, min(sms, (M // 128) * (H // 64)), rstd_ss=ss, rstd_parts=H // 128,
            rstd_eps=eps, stages=6)
    assert_close("norm -> qkv", out[:N], ref, 1e-5, 1e-5)
    assert out[N:].isnan().all()
