"""The fused decode step's q|k|v projection as a cluster split-K GEMM (tc_gemm_splitk_kernel in store mode, through
b2a_tc_gemm_splitk_store_test).  Each CTA of a tile's cluster streams the piece of the tile that the stream-K GEMM's CTA streams
(tc_gemm_kernel<16> over the same CTA count), and the leader sums the pieces with that GEMM's arithmetic, so for tokens t < N

    out[t] = rstd[t] * W (x_hi[t] + x_lo[t])          rstd[t] = rsqrt(sum_p rstd_ss[p, t] / K + eps)   (1 without rstd_ss)

is bit-identical to the stream-K launch, and within float64 bounds; rows t >= N of out are untouched.  Also: the launch plan the
engine picks (one CTA per piece, all clusters resident at once), its neighbours in the step fitting on one SM, and the stream-K
GEMM (the fallback) storing into an output that was not zeroed first."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import rel_err
from gemm_reference import EPI_STORE, assert_close, hilo_tiles, tc_gemm
from oracle import llama as ol

pytestmark = pytest.mark.gpu

STAGES = 5                      # llama.cu splitk_stages
ATTN_STATIC_SMEM = 512          # attn_decode_cluster_kernel's static arrays (red_m, red_l)
RESERVED_PER_CTA = 1024


def _splitk_store(b2a, W, X, out, rstd_ss, parts, eps, M, N, K, cluster, sk_ctas):
    f = b2a._ffi
    st = f.lib().b2a_tc_gemm_splitk_store_test(f.ptr(W), f.ptr(X), f.ptr(out), f.ptr(rstd_ss), parts, eps, M, N, K, cluster, sk_ctas,
                                               STAGES, None)
    torch.cuda.synchronize()
    assert st == 0, f.lib().b2a_last_error()


def qkv_plan(b2a, m_tiles, k_blocks):
    """(cluster size or 0, bytes per CTA, clusters resident at once, stream-K CTA count, most pieces of a tile)"""
    out = (C.c_int32 * 5)()
    b2a._ffi.check(b2a._ffi.lib().b2a_debug_qkv_split(m_tiles, k_blocks, out))
    return tuple(int(v) for v in out)


SHAPES = [
    # M, K
    (5120, 3072),        # Orpheus 3B q|k|v: 40 tiles, 48 k-blocks
    (4096, 1024),        # Qwen3 talker / code predictor q|k|v: 32 tiles, 16 k-blocks
    (512, 256),          # test model: 4 tiles, 4 k-blocks, every tile split
    (384, 128),          # 2 k-blocks
]


def _inputs(M, K, N, seed, parts):
    g = torch.Generator(device="cuda").manual_seed(seed)
    W = (torch.randn(M, K, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    x = torch.randn(8, K, device="cuda", generator=g)               # rows >= N hold data too: they must not reach out
    X, xe = hilo_tiles(x, 16)
    ss = torch.rand(parts, 8, device="cuda", generator=g) * K / parts + 0.1
    return W, X, xe, ss


@pytest.mark.parametrize("rstd", [False, True], ids=["plain", "rstd"])
@pytest.mark.parametrize("N", [1, 5, 8])
@pytest.mark.parametrize("M,K", SHAPES)
def test_splitk_store_matches_streamk_and_float64(b2a, M, K, N, rstd):
    """Bit-identical to the stream-K GEMM over the same CTA count; against float64 the bounds of the residual split-K epilogue
    (test_gpu_splitk_norm.py): relative L2 1e-5, max over peak 2e-5."""
    mt, kb = -(-M // 128), K // 64
    cluster, _, _, sk_ctas, pieces = qkv_plan(b2a, mt, kb)
    assert cluster == pieces and sk_ctas > 0
    eps, parts = 1e-5, max(1, K // 128)
    W, X, xe, ss = _inputs(M, K, N, M + K + N + rstd, parts)
    ss = ss if rstd else None
    ref = xe[:N] @ W.double().T
    if rstd:
        ref = ref / torch.sqrt(ss.double().sum(0)[:N, None] / K + eps)
    out = torch.full((8, M), float("nan"), device="cuda")
    _splitk_store(b2a, W, X, out, ss, parts if rstd else 0, eps, M, N, K, cluster, sk_ctas)
    assert_close("out", out[:N], ref, 1e-5, 2e-5)
    assert out[N:].isnan().all()
    sk = torch.full((8, M), float("nan"), device="cuda")
    tc_gemm(b2a, W, X, sk, M, N, K, 16, EPI_STORE, 1, 1, sk_ctas, rstd_ss=ss, rstd_parts=parts if rstd else 0, rstd_eps=eps, stages=6)
    assert torch.equal(out[:N], sk[:N]), float((out[:N] - sk[:N]).abs().max())


def test_splitk_store_rejects_bad_cluster(b2a):
    f = b2a._ffi
    W = torch.zeros(512, 256, device="cuda", dtype=torch.bfloat16)
    X = torch.zeros(16, 256, device="cuda", dtype=torch.bfloat16)
    out = torch.zeros(8, 512, device="cuda")
    # more CTAs than k-blocks; fewer CTAs than the stream-K cut over 16 CTAs gives a tile (4 pieces)
    assert f.lib().b2a_tc_gemm_splitk_store_test(f.ptr(W), f.ptr(X), f.ptr(out), None, 0, 0.0, 512, 8, 256, 5, 0, STAGES, None) != 0
    assert f.lib().b2a_tc_gemm_splitk_store_test(f.ptr(W), f.ptr(X), f.ptr(out), None, 0, 0.0, 512, 8, 256, 3, 16, STAGES, None) != 0


@pytest.mark.parametrize("name,m_tiles,k_blocks", [("orpheus", 40, 48), ("qwen3", 32, 16), ("test model", 4, 4), ("two k-blocks", 3, 2)])
def test_qkv_plan_is_one_wave(b2a, name, m_tiles, k_blocks):
    """The engine's plan: one CTA per stream-K piece of a tile, used when all m_tiles clusters are resident at once.  pytest -s prints
    what the device reports."""
    c, smem, active, sk_ctas, pieces = qkv_plan(b2a, m_tiles, k_blocks)
    print(f"{name}: {m_tiles} tiles, {k_blocks} k-blocks, stream-K over {sk_ctas} CTAs -> clusters of {c}, {smem} B per CTA, "
          f"{active} clusters resident at once")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert sk_ctas == min(sms, m_tiles * k_blocks)
    assert c == pieces and 1 <= c <= 8 and m_tiles <= active
    assert smem == STAGES * 18432 + (c - 1) * 4096 + 512


def test_qkv_falls_back_when_a_tile_has_more_than_8_pieces(b2a):
    """One tile of 16 k-blocks over 16 stream-K CTAs is 16 pieces: more than a cluster may hold, the stream-K GEMM runs."""
    assert qkv_plan(b2a, 1, 8)[0] == 8
    assert qkv_plan(b2a, 1, 16)[:3] == (0, 0, 0)


@pytest.mark.parametrize("G", [1, 2, 3, 4, 6, 8])
def test_qkv_neighbours_fit_on_one_sm(b2a, G):
    """The step's new neighbouring pairs: down split-K + q|k|v split-K (next layer), q|k|v split-K + attention, for every cluster size
    the q|k|v GEMM can be given."""
    per_sm = torch.cuda.get_device_properties(0).shared_memory_per_multiprocessor
    step = (C.c_int32 * 3)()
    b2a._ffi.check(b2a._ffi.lib().b2a_debug_step_smem(G, step))
    down, attn = int(step[1]), int(step[2]) + ATTN_STATIC_SMEM
    for c in range(1, 9):
        chosen, qkv = qkv_plan(b2a, 1, c)[:2]                       # one tile of c k-blocks over c CTAs: c pieces
        assert chosen == c
        for name, a, b in (("down split-K + qkv split-K", down, qkv), ("qkv split-K + attention", qkv, attn)):
            assert a + b + 2 * RESERVED_PER_CTA <= per_sm, (name, c, a, b, per_sm)


def test_streamk_store_needs_no_zeroed_output(b2a):
    """Stream-K with EPI_STORE: the CTA that completes a tile stores the sum of its partials, so the output may hold anything before
    (the step's stream-K fallback does not clear q|k|v)."""
    M, K, N = 512, 256, 8
    g = torch.Generator(device="cuda").manual_seed(5)
    W = (torch.randn(M, K, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    X, xe = hilo_tiles(torch.randn(N, K, device="cuda", generator=g), 16)
    out = torch.full((N + 5, M), 1e30, device="cuda")
    out[N:] = float("nan")
    tc_gemm(b2a, W, X, out, M, N, K, 16, EPI_STORE, 1, 1, 16, stages=6)  # 4 tiles x 4 k-blocks over 16 CTAs: every tile is split
    assert_close("stream-K store", out[:N], xe @ W.double().T, 2e-5, 3e-5)
    assert out[N:].isnan().all()


def test_trace_after_fused_steps_matches_oracle(b2a):
    """The fused step leaves q|k|v holding the last layer's projection; a traced forward after it (the same step, recording the
    residual stream) must not add onto it."""
    cfg = ol.LlamaConfig(hidden_size=256, num_hidden_layers=2, intermediate_size=512, num_attention_heads=2, num_key_value_heads=1,
                         head_dim=128, vocab_size=512)
    W = ol.init_weights(cfg, 3, std=0.05)
    hf = dict(hidden_size=256, num_hidden_layers=2, intermediate_size=512, num_attention_heads=2, num_key_value_heads=1, head_dim=128,
              vocab_size=512, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta, tie_word_embeddings=True,
              rope_scaling={"rope_type": "llama3", "factor": 32.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                            "original_max_position_embeddings": 8192})
    m = b2a.LlamaTTSModel(hf, W, max_batch=2, max_context=64)
    ids = np.random.default_rng(4).integers(0, 512, size=(2, 6)).astype(np.int32)
    ref = ol.LlamaOracle(cfg, W, round_acts=False).forward(torch.as_tensor(ids)).numpy()
    fused = m(ids)
    m.debug_trace(True)
    traced = m(ids)
    m.debug_trace(False)
    assert rel_err(fused, ref) < 1e-4
    assert rel_err(traced, ref) < 1e-4
