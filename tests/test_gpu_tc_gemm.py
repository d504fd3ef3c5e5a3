"""The wgmma + TMA "weights-as-A" GEMM in isolation (b2a_tc_gemm_test, device pointers) against a torch
fp32 reference of the same op: out[N, M] = X[N, K] @ W[M, K]^T.  bf16 inputs, fp32 accumulation: the only
difference from the reference is summation order, so the tolerance is tight (1e-5 relative).

test_epilogue_matches_float64 (b2a_tc_gemm_epilogue_test) runs every epilogue an engine launches (bias, exact-erf GELU, SwiGLU,
residual add, hi/lo bf16 outputs, tile_rows < 128, the fused-RMSNorm rstd scaling, stream-K partial tiles) at the call sites'
shapes, CTA counts and ring depths against float64."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from gemm_reference import ACT_GELU, EPI_ADD, EPI_STORE, EPI_STORE_BF16, EPI_SWIGLU
from gemm_reference import assert_close, assert_lo_within_half_ulp, hilo_rows, hilo_tiles, run_tc_gemm, tc_gemm

pytestmark = pytest.mark.gpu


def _run(b2a, W, X, out, M, N, K, bn, epi, split, hilo, ctas):
    lib = C.CDLL(str(b2a._ffi.LIB_PATH))
    fn = lib.b2a_tc_gemm_test
    fn.restype = C.c_int32
    fn.argtypes = [C.c_void_p] * 3 + [C.c_int32] * 8 + [C.c_void_p]
    st = fn(W.data_ptr(), X.data_ptr(), out.data_ptr(), M, N, K, bn, epi, split, hilo, ctas, None)
    torch.cuda.synchronize()
    assert st == 0, b2a._ffi.lib().b2a_last_error()


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.mark.parametrize("M,K,N,ctas,split", [(128, 64, 8, 1, 0), (256, 128, 8, 2, 0), (384, 512, 5, 3, 0),
                                              (1000, 256, 8, 7, 0), (3072, 3072, 8, 148, 1), (5120, 3072, 8, 148, 1),
                                              (3072, 8192, 8, 148, 1), (640, 1024, 16, 148, 1)])
def test_decode_tile_store_and_streamk(b2a, M, K, N, ctas, split):
    g = torch.Generator(device="cuda").manual_seed(M + K)
    W = (torch.randn(M, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    X = torch.randn(N, K, device="cuda", generator=g).to(torch.bfloat16)
    out = torch.zeros(N, M, device="cuda", dtype=torch.float32)
    _run(b2a, W, X, out, M, N, K, 16, 0, split, 0, ctas)
    ref = X.float() @ W.float().T
    assert _rel(out, ref) < 1e-5, _rel(out, ref)


def test_hilo_gives_fp32_activation_accuracy(b2a):
    M, K, B = 1024, 2048, 8
    g = torch.Generator(device="cuda").manual_seed(0)
    W = (torch.randn(M, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    x = torch.randn(B, K, device="cuda", generator=g)
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    X = torch.cat([hi, lo]).contiguous()
    out = torch.zeros(B, M, device="cuda", dtype=torch.float32)
    _run(b2a, W, X, out, M, B, K, 16, 0, 1, 1, 148)
    ref = x.double() @ W.double().T
    assert _rel(out, ref) < 2e-5, _rel(out, ref)
    only_hi = hi.float() @ W.float().T
    assert _rel(only_hi, ref) > 1e-3          # what bf16-rounded activations would have cost


def test_swiglu_epilogue_hilo_out(b2a):
    I, K, B = 512, 1024, 8
    g = torch.Generator(device="cuda").manual_seed(1)
    Wg = (torch.randn(I, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    Wu = (torch.randn(I, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    W = torch.stack([Wg, Wu], dim=1).reshape(2 * I, K).contiguous()        # rows interleaved gate/up
    x = torch.randn(B, K, device="cuda", generator=g)
    hi = x.to(torch.bfloat16)
    X = torch.cat([hi, (x - hi.float()).to(torch.bfloat16)]).contiguous()
    out = torch.zeros(16, I, device="cuda", dtype=torch.bfloat16)
    _run(b2a, W, X, out, 2 * I, B, K, 16, 2, 0, 1, 8)
    gte, up = x.double() @ Wg.double().T, x.double() @ Wu.double().T
    ref = torch.nn.functional.silu(gte) * up
    got = out[:8].double() + out[8:].double()
    assert _rel(got, ref) < 5e-5, _rel(got, ref)


@pytest.mark.parametrize("M,K,N,ctas", [(256, 128, 128, 2), (512, 256, 300, 4), (1024, 3072, 512, 37)])
def test_prefill_tile_bn128(b2a, M, K, N, ctas):
    g = torch.Generator(device="cuda").manual_seed(N)
    W = (torch.randn(M, K, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    X = torch.randn(N, K, device="cuda", generator=g).to(torch.bfloat16)
    out = torch.zeros(N, M, device="cuda", dtype=torch.float32)
    _run(b2a, W, X, out, M, N, K, 128, 0, 1, 0, ctas)
    ref = X.float() @ W.float().T
    assert _rel(out, ref) < 1e-5, _rel(out, ref)


# ---------------------------------------------------------------------------------------------- epilogue matrix
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cdiv(a, b):
    return -(-a // b)


def _pick_tile_rows(M, sms):
    """llama.cu pick_tile_rows / whisper.cu make_step_map: 128 rows per m-tile unless that leaves over a quarter of the SMs idle."""
    if _cdiv(M, 128) * 4 >= sms * 3:
        return 128
    return max(8, min(128, _cdiv(_cdiv(M, sms), 8) * 8))


def _config(family, M, K, N, sms):
    """The hook arguments each engine call site uses (csrc/llama.cu tc_gemm / pf_gemm, csrc/whisper.cu gemm_step / gemm_big)."""
    kb = K // 64
    if family in ("qkv", "qkv_idle_ctas"):          # decode q|k|v: stream-K store, fused RMSNorm (llama.cu tc_gemm, OP_QKV)
        ctas = min(sms, _cdiv(M, 128) * kb) if family == "qkv" else sms + 7     # the second: more CTAs than (tile, k-block) units
        return dict(bn=16, epi=EPI_STORE, split=1, ctas=ctas, rstd=True, stages=6)
    if family == "gate_up":                         # decode gate/up: SwiGLU to hi/lo bf16, tile_rows rows per m-tile, fused RMSNorm
        tr = _pick_tile_rows(M, sms)
        return dict(bn=16, epi=EPI_SWIGLU, lo_rows=1, tile_rows=tr, ctas=min(sms, _cdiv(M, tr)), rstd=True, stages=6)
    if family == "lm_head":                         # decode lm head: fp32 logits, tile_rows rows per m-tile, fused RMSNorm
        tr = _pick_tile_rows(M, sms)
        return dict(bn=16, epi=EPI_STORE, tile_rows=tr, ctas=min(sms, _cdiv(M, tr)), rstd=True, stages=6)
    if family == "whisper_fc1":                     # Whisper decoder step fc1: bias + GELU to hi/lo bf16, step_rows rows per m-tile
        tr = _pick_tile_rows(M, sms)
        tr = 0 if tr == 128 else tr
        return dict(bn=32, epi=EPI_STORE_BF16, lo_rows=1, bias=True, act=ACT_GELU, tile_rows=tr, ctas=min(sms, _cdiv(M, tr or 128)), stages=8)
    if family == "whisper_add":                     # Whisper decoder step out-proj / fc2: bias + residual add, stream-K
        return dict(bn=32, epi=EPI_ADD, split=1, bias=True, ctas=min(sms, max(1, _cdiv(M, 128) * kb // 4)), stages=8)
    ctas = max(1, min(_cdiv(M, 128), sms // _cdiv(N, 64)))
    if family == "encoder_fc1":                     # Whisper encoder fc1: 64-token hi/lo tiles, bias + GELU to hi/lo bf16
        return dict(bn=128, epi=EPI_STORE_BF16, lo_rows=1, bias=True, act=ACT_GELU, ctas=ctas)
    if family == "encoder_add":                     # Whisper encoder out-proj / fc2: bias + residual add, whole tiles
        return dict(bn=128, epi=EPI_ADD, bias=True, ctas=ctas)
    assert family == "prefill_gate_up"              # Llama batched prefill gate/up: SwiGLU to hi/lo bf16
    return dict(bn=128, epi=EPI_SWIGLU, lo_rows=1, ctas=ctas)


EPILOGUE_CASES = [
    # family, M (weight rows), K, N (tokens)
    ("qkv", 512, 256, 8),                 # test models: hidden 256, 2 + 2 x 1 heads; 2 rstd parts
    ("qkv_idle_ctas", 512, 256, 3),
    ("qkv", 4096, 1024, 5),               # Qwen3-0.6B geometry: 16 + 2 x 8 heads; 8 rstd parts
    ("qkv", 5120, 3072, 8),               # Orpheus 3B: 24 + 2 x 8 heads; 24 rstd parts
    ("gate_up", 1024, 256, 8),            # 2 x intermediate 512: 8 rows per m-tile on 132 SMs
    ("gate_up", 6144, 1024, 3),           # Qwen3-TTS talker: 48 rows per m-tile on 132 SMs
    ("gate_up", 16384, 3072, 8),          # Orpheus: 128 rows per m-tile
    ("lm_head", 156940, 3072, 8),         # Orpheus vocabulary: 128 rows per m-tile, 156940 % 128 = 12
    ("lm_head", 2048, 1024, 8),           # code-predictor vocabulary: 16 rows per m-tile
    ("lm_head", 2044, 256, 2),            # 16 rows per m-tile with a partial last tile
    ("whisper_fc1", 2048, 512, 1),        # Whisper base (d_model 512, ffn 2048), one to sixteen clips
    ("whisper_fc1", 2048, 512, 5),
    ("whisper_fc1", 2048, 512, 16),
    ("whisper_add", 512, 2048, 1),        # fc2: 32 CTAs
    ("whisper_add", 512, 2048, 5),
    ("whisper_add", 512, 512, 16),        # out-proj: 8 CTAs
    ("encoder_fc1", 2048, 512, 100),      # 2 and 24 token tiles (T = 1500)
    ("encoder_fc1", 2048, 512, 1500),
    ("encoder_add", 512, 2048, 100),
    ("encoder_add", 512, 2048, 1500),
    ("prefill_gate_up", 1024, 256, 100),
    ("prefill_gate_up", 1024, 256, 1500),
]


@pytest.mark.parametrize("family,M,K,N", EPILOGUE_CASES, ids=[f"{c[0]}-{c[1]}x{c[2]}-n{c[3]}" for c in EPILOGUE_CASES])
def test_epilogue_matches_float64(b2a, family, M, K, N):
    """Each case against float64 on the same bf16 weights and hi/lo activation pairs: rstd * (W (x_hi + x_lo)) + bias, then GELU /
    SwiGLU / residual add.  Outputs outside the N tokens (and, for hi/lo outputs, outside their rows) must keep the NaN they were
    filled with.  Measured on an H100 80GB HBM3 (132 SMs), worst case over all cases: relative L2 6.7e-6, max/peak 9.2e-6 (both
    Orpheus gate/up, K = 3072); the stream-K stores and adds stay below 1e-6.  Bounds: 2e-5 and 3e-5, about 3x the worst case."""
    sms = _sms()
    c = _config(family, M, K, N, sms)
    bn, epi = c["bn"], c["epi"]
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(M * 7 + K * 3 + N)
    W = (torch.randn(M, K, device=dev, generator=g) * 0.05).to(torch.bfloat16)
    ref = None
    rstd_ss, parts, eps = None, 0, 1e-5
    if c.get("rstd"):
        # the producer left h * gain un-normalised and the per-128-feature sums of squares of h (llama.cu add_rmsnorm_kernel)
        h = torch.randn(N, K, device=dev, generator=g)
        gain = 1.0 + 0.2 * torch.randn(K, device=dev, generator=g)
        x = h * gain
        parts = K // 128
        rstd_ss = torch.zeros(parts, 8, device=dev)
        rstd_ss[:, :N] = (h.double() ** 2).view(N, parts, 128).sum(-1).T.float()
        rstd = 1.0 / torch.sqrt(rstd_ss.double().sum(0)[:N] / K + eps)
    else:
        x = torch.randn(N, K, device=dev, generator=g)
    X, xe = hilo_tiles(x, bn)
    ref = xe @ W.double().T
    if rstd_ss is not None:
        ref = ref * rstd[:, None]
    bias = None
    if c.get("bias"):
        bias = 0.5 * torch.randn(M, device=dev, generator=g)
        ref = ref + bias.double()
    if c.get("act") == ACT_GELU:
        ref = 0.5 * ref * (1.0 + torch.erf(ref / math.sqrt(2.0)))
    if epi == EPI_SWIGLU:
        gte, up = ref[:, 0::2], ref[:, 1::2]                        # weight rows are (gate, up) pairs
        ref = gte * torch.sigmoid(gte) * up
    n_tiles = _cdiv(N, bn // 2)
    ldo = M // 2 if epi == EPI_SWIGLU else M
    if c.get("lo_rows"):
        out = torch.full((n_tiles * bn, ldo), float("nan"), device=dev, dtype=torch.bfloat16)
    else:
        out = torch.full((N + 5, ldo), float("nan"), device=dev)
        if epi == EPI_ADD:
            res = torch.randn(N, M, device=dev, generator=g)
            out[:N] = res
            ref = ref + res.double()
        elif c.get("split"):
            out[:N] = 0                                             # stream-K partial tiles are added into the output
    tc_gemm(b2a, W, X, out, M, N, K, bn, epi, c.get("split", 0), 1, c["ctas"], bias=bias, act=c.get("act", 0),
            tile_rows=c.get("tile_rows", 0), lo_rows=c.get("lo_rows", 0), rstd_ss=rstd_ss, rstd_parts=parts, rstd_eps=eps,
            stages=c.get("stages", 0))
    if c.get("lo_rows"):
        hr, lr = hilo_rows(N, bn)
        hi, lo = out[hr], out[lr]
        assert_close(family, hi.double() + lo.double(), ref, 2e-5, 3e-5)
        assert_lo_within_half_ulp(hi, lo)
        untouched = torch.ones(out.shape[0], dtype=torch.bool, device=dev)
        untouched[hr] = False
        untouched[lr] = False
        assert out[untouched].isnan().all()
    else:
        assert_close(family, out[:N], ref, 2e-5, 3e-5)
        assert out[N:].isnan().all()


@pytest.mark.parametrize("why,kw", [
    ("GELU of a partial K range", dict(bn=16, epi=EPI_STORE, split=1, act=ACT_GELU)),
    ("rstd scaling outside BN = 16", dict(bn=32, epi=EPI_STORE, split=0, rstd=True)),
    ("rstd scaling of bf16 activations", dict(bn=16, epi=EPI_STORE, split=0, hilo=0, rstd=True)),
    ("hi/lo output of an fp32 epilogue", dict(bn=16, epi=EPI_STORE, split=0, lo_rows=1)),
    ("tile_rows with stream-K", dict(bn=16, epi=EPI_STORE, split=1, tile_rows=16)),
    ("tile_rows not a multiple of 8", dict(bn=16, epi=EPI_STORE, split=0, tile_rows=20)),
])
def test_unused_epilogue_combinations_are_rejected(b2a, why, kw):
    M, K, N = 256, 128, 8
    W = torch.zeros(M, K, device="cuda", dtype=torch.bfloat16)
    X = torch.zeros(2 * kw["bn"], K, device="cuda", dtype=torch.bfloat16)
    out = torch.zeros(2 * kw["bn"], M, device="cuda")
    ss = torch.ones(2, 8, device="cuda") if kw.get("rstd") else None
    st = run_tc_gemm(b2a, W, X, out, M, N, K, kw["bn"], kw["epi"], kw["split"], kw.get("hilo", 1), 4, act=kw.get("act", 0),
                            tile_rows=kw.get("tile_rows", 0), lo_rows=kw.get("lo_rows", 0), rstd_ss=ss, rstd_parts=2 if ss is not None else 0)
    assert st == b2a._ffi.ERR_INVALID_INPUT, why
    assert not out.any()
