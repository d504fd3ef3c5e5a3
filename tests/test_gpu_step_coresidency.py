"""The fused decode step's kernels are sized to share an SM with their neighbours, so that each kernel's prefetch before
griddepcontrol.wait runs under the main loop of the kernel before it:

* footprints: for every GQA ratio the engine accepts, each pair of kernels that follow each other in the step (QKV GEMM + attention,
  attention + o split-K, split-K + gate/up GEMM, gate/up GEMM + down split-K, down split-K + next QKV GEMM) plus the 1 KB the system
  keeps per resident CTA fits in the device's shared memory per SM, with the GEMM ring depths the engine launches;
* the attention kernel's staging (K and V of a 64-key chunk in separate ring slots, the warp-partial outputs over a ring slot, the
  Qwen3 q/k norm staged in place) against the float64 oracle at contexts that put the new position first, last and in the middle of
  a chunk for both CTAs of the cluster, for G = 3 and G = 8, with and without the q/k norm."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import llama as ol
from oracle import qwen3_tts as ot

pytestmark = pytest.mark.gpu

ATTN_STATIC_SMEM = 512          # attn_decode_cluster_kernel's static arrays (red_m, red_l)
RESERVED_PER_CTA = 1024
POSITIONS = (0, 1, 63, 64, 65, 127, 128, 129, 191, 192, 575)
CTX = 576


def step_smem(b2a, G):
    out = (C.c_int32 * 3)()
    b2a._ffi.check(b2a._ffi.lib().b2a_debug_step_smem(G, out))
    return int(out[0]), int(out[1]), int(out[2]) + ATTN_STATIC_SMEM


@pytest.mark.parametrize("G", [1, 2, 3, 4, 6, 8])
def test_neighbouring_kernels_fit_on_one_sm(b2a, G):
    per_sm = torch.cuda.get_device_properties(0).shared_memory_per_multiprocessor
    gemm, splitk, attn = step_smem(b2a, G)
    for name, a, b in (("gemm + attention", gemm, attn), ("attention + split-K", attn, splitk), ("split-K + gemm", splitk, gemm)):
        assert a + b + 2 * RESERVED_PER_CTA <= per_sm, (name, a, b, per_sm)
    # the rings were kept: 6 and 5 stages of 128 x 64 weights + 16 x 64 activations, three 64 x 128 fp32 matrices
    assert gemm >= 6 * 18432 and splitk >= 5 * 18432 and attn >= 3 * 32768


def test_step_smem_rejects_unknown_ratio(b2a):
    out = (C.c_int32 * 3)()
    assert b2a._ffi.lib().b2a_debug_step_smem(5, out) != 0


def hf_config(cfg: ol.LlamaConfig) -> dict:
    return dict(hidden_size=cfg.hidden_size, num_hidden_layers=cfg.num_hidden_layers, intermediate_size=cfg.intermediate_size,
                num_attention_heads=cfg.num_attention_heads, num_key_value_heads=cfg.num_key_value_heads, head_dim=cfg.head_dim,
                vocab_size=cfg.vocab_size, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta, tie_word_embeddings=True,
                rope_scaling={"rope_type": "llama3", "factor": 32.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                              "original_max_position_embeddings": 8192})


@pytest.mark.parametrize("nq", [3, 8], ids=["g3", "g8"])
def test_attention_staging_at_chunk_edges(b2a, nq):
    """576 positions through the decode step, one at a time (longer than the batched prompt pass takes): at position p the new k / v
    row is spliced into row p % 64 of the last chunk, which CTA (p / 64) % 2 of the cluster owns."""
    cfg = ol.LlamaConfig(hidden_size=128, num_hidden_layers=1, intermediate_size=256, num_attention_heads=nq, num_key_value_heads=1,
                         head_dim=128, vocab_size=512)
    W = ol.init_weights(cfg, 7, std=0.1)
    m = b2a.LlamaTTSModel(hf_config(cfg), W, max_batch=2, max_context=CTX + 16)
    ids = np.random.default_rng(2).integers(0, 512, size=(2, CTX)).astype(np.int32)
    lg = m(ids)
    ref = ol.LlamaOracle(cfg, W, round_acts=False).forward(torch.as_tensor(ids)).numpy()
    for pos in POSITIONS:
        assert rel_err(lg[:, pos], ref[:, pos]) < 1e-4, pos


@pytest.mark.parametrize("nq", [3, 8], ids=["g3", "g8"])
def test_attention_staging_with_qk_norm(b2a, nq):
    """The same with the Qwen3 talker's per-head q / k RMSNorm, which the kernel stages where RoPE leaves the rotated vectors.  The
    talker returns the last position's logits, so each context is a forward pass of its own from an empty cache."""
    cp = ot.CodePredictorConfig(vocab_size=256, hidden_size=128, intermediate_size=256, num_hidden_layers=1, num_attention_heads=1,
                                num_key_value_heads=1, head_dim=128, num_code_groups=2)
    cfg = ot.TalkerConfig(vocab_size=512, hidden_size=128, intermediate_size=256, num_hidden_layers=1, num_attention_heads=nq,
                          num_key_value_heads=1, head_dim=128, num_code_groups=2, text_hidden_size=128, text_vocab_size=64,
                          codec_eos_token_id=500, code_predictor=cp)
    W = {k: v.to(torch.bfloat16).to(torch.float64) for k, v in ot.init_weights(cfg, 11, std=0.1).items()}
    c = b2a.Qwen3TalkerConfig(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                              num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
                              num_key_value_heads=cfg.num_key_value_heads, head_dim=cfg.head_dim, rms_norm_eps=cfg.rms_norm_eps,
                              rope_theta=cfg.rope_theta, num_code_groups=cfg.num_code_groups, text_hidden_size=cfg.text_hidden_size,
                              text_vocab_size=cfg.text_vocab_size, codec_eos_token_id=cfg.codec_eos_token_id,
                              code_predictor=b2a.Qwen3CodePredictorConfig(
                                  vocab_size=cp.vocab_size, hidden_size=cp.hidden_size, intermediate_size=cp.intermediate_size,
                                  num_hidden_layers=cp.num_hidden_layers, num_attention_heads=cp.num_attention_heads,
                                  num_key_value_heads=cp.num_key_value_heads, head_dim=cp.head_dim, rms_norm_eps=cp.rms_norm_eps,
                                  rope_theta=cp.rope_theta, num_code_groups=cp.num_code_groups))
    m = b2a.Qwen3TTSTalker(c, {k: v.to(torch.bfloat16) for k, v in W.items()}, max_batch=2, max_context=CTX + 16)
    x = torch.from_numpy(np.random.default_rng(3).standard_normal((2, CTX, cfg.hidden_size))).to(torch.bfloat16).to(torch.float64)
    ref, _ = ot.Talker(cfg, W)(x, None)
    for pos in POSITIONS:
        lg, _ = m(x[:, :pos + 1].numpy().astype(np.float32))
        assert rel_err(lg, ref[:, pos].numpy()) < 1e-3, pos       # the talker tests' tolerance
