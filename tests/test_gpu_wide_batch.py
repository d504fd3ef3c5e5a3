"""Calls of 9 to 32 rows: the decode step at widths 16 and 32 (tc_gemm_kernel<32> / <64>, tc_gemm_splitk_kernel<16> / <32>) against the
same prompts run in calls of at most 8 rows (width 8) and against the oracles, for the Llama, VyvoTTS (Qwen3 LM, q/k norm) and Soprano
stacks and the Qwen3-TTS talker with its code predictor.  A row's arithmetic is the same at every width (stream-K and split-K cuts depend
on M, K and the SM count only, each output column's wgmma accumulation is its own, the rstd and s_red reductions keep their order per
token), so greedy tokens and code frames are compared exactly."""
import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import llama as ol
from oracle import qwen3_tts as ot
from oracle import soprano as so
from oracle import vyvo
from test_gpu_llama import TINY, hf_config
from test_gpu_qwen3_talker import CHAT, TTS, bf16_weights, device_model, small_cfg
from test_oracle_qwen3_tts_1p7b import golden_module

pytestmark = pytest.mark.gpu


def chunks(B):
    return [(i, min(i + 8, B)) for i in range(0, B, 8)]


def greedy_params(b2a, n=24):
    return b2a.GenerateParameters(max_tokens=n, temperature=0.0, top_p=1.0, repetition_penalty=1.3, repetition_context_size=20)


@pytest.fixture(scope="module")
def llama32(b2a):
    cfg = ol.LlamaConfig(**TINY)
    W = ol.init_weights(cfg, 1234, std=0.08)
    return cfg, W, b2a.LlamaTTSModel(hf_config(cfg), W, max_batch=32, max_context=256)


@pytest.mark.parametrize("B", [9, 16, 17, 32])
def test_llama_greedy_rows_equal_calls_of_8(b2a, llama32, B):
    cfg, W, m = llama32
    ids = np.random.default_rng(100 + B).integers(0, 2048, size=(B, 10)).astype(np.int32)
    P = greedy_params(b2a)
    wide, _, info = m.generate_batch(ids, P, decode_audio=False)
    narrow = []
    for a, b in chunks(B):
        t, _, _ = m.generate_batch(ids[a:b], P, decode_audio=False)
        narrow += t
    assert info.generation_token_count == 24 * B
    assert np.array_equal(np.asarray(wide), np.asarray(narrow))
    ref = ol.generate_tokens(ol.LlamaOracle(cfg, W, False), ids[[0, B - 1]], 24, temperature=0.0, rep_penalty=1.3, rep_context=20)
    assert [wide[0], wide[B - 1]] == ref


def test_llama_logits_at_32_rows_vs_oracle(llama32):
    cfg, W, m = llama32
    ids = np.random.default_rng(5).integers(0, 2048, size=(32, 12)).astype(np.int32)
    lg = m(ids)
    ref = ol.LlamaOracle(cfg, W, round_acts=False).forward(torch.as_tensor(ids)).numpy()
    assert lg.shape == ref.shape == (32, 12, 2048)
    assert rel_err(lg, ref) < 1e-4, rel_err(lg, ref)
    assert np.array_equal(lg.argmax(-1), ref.argmax(-1))


def test_llama_sampling_rows_are_width_independent(b2a, llama32):
    cfg, W, m = llama32
    ids = np.random.default_rng(7).integers(0, 2048, size=(32, 10)).astype(np.int32)
    P = b2a.GenerateParameters(max_tokens=24, temperature=0.6, top_p=0.8, repetition_penalty=1.3, repetition_context_size=20, seed=42)
    wide, _, _ = m.generate_batch(ids, P, decode_audio=False)
    narrow, _, _ = m.generate_batch(ids[:8], P, decode_audio=False)
    assert wide[:8] == narrow                                  # the noise hashes (seed, row, step): rows 0..7 draw the same
    again, _, _ = m.generate_batch(ids, P, decode_audio=False)
    assert again == wide
    same = np.repeat(ids[:1], 32, axis=0)
    copies, _, _ = m.generate_batch(same, P, decode_audio=False)
    assert len({tuple(t) for t in copies}) > 1                 # 32 copies of one prompt do not all draw the same tokens


def test_launches_per_step_do_not_depend_on_the_width(b2a, llama32):
    cfg, W, m = llama32
    P = greedy_params(b2a, 16)
    counts = {}
    for B in (8, 16, 32):
        ids = np.random.default_rng(B).integers(0, 2048, size=(B, 10)).astype(np.int32)
        per_n = []
        for n in (8, 16):
            n0 = b2a.launch_count()
            m.generate_batch(ids, greedy_params(b2a, n), decode_audio=False)
            per_n.append(b2a.launch_count() - n0)
        counts[B] = per_n[1] - per_n[0]                        # launches of 8 decode steps
    assert counts[8] == counts[16] == counts[32], counts


def test_partly_filled_last_m_tile_at_32_rows(b2a):
    # hidden 192: the o / down GEMMs' second m-tile holds 64 of 128 rows, and the fused norm reduces two partial sums per token
    cfg = ol.LlamaConfig(**{**TINY, "hidden_size": 192})
    W = ol.init_weights(cfg, 77, std=0.08)
    m = b2a.LlamaTTSModel(hf_config(cfg), W, max_batch=32, max_context=64)
    ids = np.random.default_rng(3).integers(0, 2048, size=(32, 8)).astype(np.int32)
    lg = m(ids)
    ref = ol.LlamaOracle(cfg, W, round_acts=False).forward(torch.as_tensor(ids)).numpy()
    assert rel_err(lg, ref) < 1e-4, rel_err(lg, ref)
    assert np.array_equal(lg.argmax(-1), ref.argmax(-1))


@pytest.mark.parametrize("rows,width,gemm,gemm_bytes,splitk,splitk_bytes", [
    (1, 8, 6, 121088, 5, 109056), (8, 8, 6, 121088, 5, 109056),
    (9, 16, 4, 100608, 4, 115200), (16, 16, 4, 100608, 4, 115200),
    (17, 32, 3, 108800, 2, 115328), (32, 32, 3, 108800, 2, 115328)])
def test_step_footprints_per_width(b2a, rows, width, gemm, gemm_bytes, splitk, splitk_bytes):
    import ctypes as C
    out = (C.c_int32 * 6)()
    lib = b2a._ffi.lib()
    b2a._ffi.check(lib.b2a_debug_step_smem_rows(rows, 3, out))
    assert list(out) == [width, gemm, gemm_bytes, splitk, splitk_bytes, 102528]
    old = (C.c_int32 * 3)()
    b2a._ffi.check(lib.b2a_debug_step_smem(3, old))
    assert list(old) == [121088, 109056, 102528]
    # the widths' neighbours that share an SM (233 472 bytes, 1 KB reserved per CTA, 512 static bytes in the attention kernel)
    sm, attn = 233472, 102528 + 512
    assert gemm_bytes + splitk_bytes + 2048 <= sm
    assert attn + gemm_bytes + 2048 <= sm and attn + splitk_bytes + 2048 <= sm


def test_vyvo_32_rows_equal_calls_of_8(b2a):
    cfg = vyvo.Qwen3Config(hidden_size=256, num_hidden_layers=2, intermediate_size=512, head_dim=128, vocab_size=2048,
                           num_attention_heads=4, num_key_value_heads=1, tie_word_embeddings=False,
                           rope_scaling={"type": "linear", "factor": 2.0})
    W = vyvo.init_weights(cfg, 1234, std=0.08)
    m = b2a.Qwen3Model(cfg.to_json(), W, max_batch=32, max_context=128)
    ids = np.random.default_rng(11).integers(0, 2048, size=(32, 12)).astype(np.int32)
    P = greedy_params(b2a)
    wide, _, _ = m.generate_batch(ids, P, decode_audio=False)
    narrow = []
    for a, b in chunks(32):
        narrow += m.generate_batch(ids[a:b], P, decode_audio=False)[0]
    assert wide == narrow
    assert [wide[0], wide[31]] == vyvo.generate_tokens(vyvo.VyvoOracle(cfg, W), ids[[0, 31]], 24, rep_penalty=1.3, rep_context=20)


def test_soprano_32_rows_equal_calls_of_8(b2a):
    cfg = so.SopranoConfig(hidden_size=256, num_hidden_layers=2, intermediate_size=512, num_attention_heads=2, num_key_value_heads=1,
                           head_dim=128, vocab_size=512, decoder_num_layers=2, decoder_dim=128, decoder_intermediate_dim=256, hop_length=64,
                           n_fft=256, upscale=4, input_kernel=3, dw_kernel=3, token_size=256)
    W = so.init_weights(cfg, 1234, std=0.08)
    ids = np.random.default_rng(9).integers(4, 512, size=(32, 9)).astype(np.int32)
    free, _ = so.generate(so.SopranoLM(cfg, W), ids[:1], 12, stop_token=-1)
    stop = next(t for i, t in enumerate(free[0]) if i >= 4 and t not in free[0][:i])     # row 0 stops early: lengths differ
    m = b2a.SopranoModel(cfg.to_json(), W, max_batch=32, max_context=64, stop_token_id=stop)
    P = b2a.GenerateParameters(max_tokens=12, temperature=0.0, top_p=0.95, repetition_penalty=1.5, repetition_context_size=30)
    wide, wwave, _ = m.generate_batch(ids, P)
    hid = m.hidden_states(32)
    assert len({len(t) for t in wide}) > 1
    for a, b in chunks(32):
        t, w, _ = m.generate_batch(ids[a:b], P)
        h = m.hidden_states(b - a)
        assert t == wide[a:b]
        for k in range(b - a):
            assert np.array_equal(h[k], hid[a + k])
            peak = max(np.abs(w[k]).max(), 1e-30)
            assert np.abs(wwave[a + k] - w[k]).max() / peak < 1e-5


def _talker_rows(cfg, W, B, seed):
    ri, rt, rp = ot.prepare_generation_inputs(cfg, W, CHAT, **TTS, language_id=2160)
    x = np.repeat(ri.numpy().astype(np.float32), B, axis=0)
    x[:, -1] += 0.05 * np.random.default_rng(seed).standard_normal((B, x.shape[-1])).astype(np.float32)   # a different last row each
    lens = [3 + (b % 5) for b in range(B)]
    tr = [rt[0, :n].numpy() for n in lens]
    return x, tr, rp[0, 0].numpy()


def _eos_weights(cfg, W, scale):
    # an EOS row of the codec head along a fixed random direction: rows reach EOS at different frames
    W2 = dict(W)
    head = W["codec_head.weight"].clone()
    d = torch.as_tensor(np.random.default_rng(1).standard_normal(cfg.hidden_size), dtype=torch.float64)
    head[cfg.codec_eos_token_id] = (scale * d / d.norm()).to(torch.bfloat16).to(torch.float64)
    W2["codec_head.weight"] = head
    return W2


@pytest.mark.parametrize("geometry", ["0.6b-style", "projected"])
def test_talker_frames_at_16_and_32_rows_equal_calls_of_8(b2a, geometry):
    if geometry == "projected":
        cfg = golden_module().config(384, 256)          # small_to_mtp_projection: talker 384 -> predictor 256 (the 1.7B path)
        W0 = golden_module().weights(cfg)
    else:
        cfg = small_cfg()
        W0 = bf16_weights(cfg, 3)
    P = b2a.Qwen3GenerateParameters(max_tokens=10, temperature=0.0, repetition_penalty=1.05)
    for scale in (2.0, 4.0, 8.0, 16.0):
        m = device_model(b2a, cfg, _eos_weights(cfg, W0, scale), max_batch=32, max_context=96)
        x, tr, pad = _talker_rows(cfg, W0, 32, 5)
        wide, _ = m.generate_codes(x, tr, pad, P)
        lens = [len(c) for c in wide]
        if len(set(lens)) > 1 and min(lens) < 10:
            break
    assert len(set(lens)) > 1, lens
    for B in (16, 32):
        got, _ = m.generate_codes(x[:B], tr[:B], pad, P)
        ref = []
        for a, b in chunks(B):
            ref += m.generate_codes(x[a:b], tr[a:b], pad, P)[0]
        assert all(np.array_equal(g, r) for g, r in zip(got, ref)), B
        assert all(np.array_equal(g, w) for g, w in zip(got, wide[:B]))
