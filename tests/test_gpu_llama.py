"""CUDA Llama/Orpheus step (through the C ABI) vs the oracle: logits within 1e-3 relative L2 of the fp32-activation
oracle on the same bf16 weights (the device path carries activations as bf16 hi/lo pairs and an fp32 KV cache, so it
tracks that value to ~1e-5), greedy tokens bit-exact, logits processors / sampler semantics, end-to-end
tokens -> codes -> waveform.  The oracle's round_acts=True mode (bf16 activations, what MLX itself does) is reported
for scale: it sits ~1e-2 away from both."""
import numpy as np
import pytest
import torch

from conftest import GOLDEN, max_rel_to_peak, rel_err
from oracle import llama as ol
from oracle import snac as osnac

pytestmark = pytest.mark.gpu
TOL = 1e-3

TINY = dict(hidden_size=256, num_hidden_layers=2, intermediate_size=512, num_attention_heads=2,
            num_key_value_heads=1, head_dim=128, vocab_size=2048)


def hf_config(cfg: ol.LlamaConfig) -> dict:
    return dict(hidden_size=cfg.hidden_size, num_hidden_layers=cfg.num_hidden_layers, intermediate_size=cfg.intermediate_size,
                num_attention_heads=cfg.num_attention_heads, num_key_value_heads=cfg.num_key_value_heads, head_dim=cfg.head_dim,
                vocab_size=cfg.vocab_size, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta, tie_word_embeddings=True,
                rope_scaling={"rope_type": "llama3", "factor": 32.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                              "original_max_position_embeddings": 8192})


@pytest.fixture(scope="module")
def tiny(b2a):
    cfg = ol.LlamaConfig(**TINY)
    W = ol.init_weights(cfg, 1234, std=0.08)
    return cfg, W, b2a.LlamaTTSModel(hf_config(cfg), W, max_batch=8, max_context=256)


def test_logits_vs_oracle_and_golden(tiny):
    cfg, W, m = tiny
    g = np.load(GOLDEN / "llama_tiny.npz")
    ids = g["ids"]
    lg = m(ids)
    ref = ol.LlamaOracle(cfg, W, round_acts=False).forward(torch.as_tensor(ids)).numpy()
    bf16_style = ol.LlamaOracle(cfg, W, round_acts=True).forward(torch.as_tensor(ids)).numpy()
    assert lg.shape == ref.shape == (2, 12, 2048)
    assert rel_err(lg, ref) < TOL, rel_err(lg, ref)
    assert rel_err(lg, ref) < 1e-4, rel_err(lg, ref)          # what the hi/lo + fp32-KV path actually achieves
    assert rel_err(lg[:, -1], g["logits_last"]) < TOL
    assert rel_err(bf16_style, ref) > 10 * rel_err(lg, ref)   # a bf16-activation pipeline (MLX) is far noisier
    assert np.array_equal(lg.argmax(-1), ref.argmax(-1))


@pytest.mark.parametrize("B", [1, 3, 8])
def test_batched_equals_serial_and_incremental(tiny, B):
    cfg, W, m = tiny
    ids = np.random.default_rng(B).integers(0, 2048, size=(B, 10)).astype(np.int32)
    full = m(ids)
    one = m(ids[B - 1:B])
    assert rel_err(full[B - 1:B], one) < 1e-5
    a = m(ids[:, :6])
    b = m(ids[:, 6:], reset_cache=False)
    assert rel_err(np.concatenate([a, b], axis=1), full) < 1e-5


def test_greedy_tokens_bit_exact(tiny):
    cfg, W, m = tiny
    g = np.load(GOLDEN / "llama_tiny.npz")
    ids = g["ids"].astype(np.int32)
    P = type(m.default_generation_parameters)
    toks, _, info = m.generate_batch(ids, P(max_tokens=24, temperature=0.0, top_p=1.0, repetition_penalty=1.3,
                                            repetition_context_size=20), decode_audio=False)
    assert np.array_equal(np.asarray(toks), g["greedy"])
    assert info.prompt_token_count == 12 and info.generation_token_count == 48
    # no penalty variant against a live oracle run
    toks2, _, _ = m.generate_batch(ids, P(max_tokens=16, temperature=0.0, top_p=1.0, repetition_penalty=1.0,
                                          repetition_context_size=0), decode_audio=False)
    ref = ol.generate_tokens(ol.LlamaOracle(cfg, W, False), ids, 16, temperature=0.0, rep_penalty=1.0, rep_context=0)
    assert toks2 == ref


def test_top_p_sampler_stays_in_nucleus_and_matches_distribution(tiny):
    cfg, W, m = tiny
    ids = np.random.default_rng(5).integers(0, 2048, size=(1, 8)).astype(np.int32)
    P = type(m.default_generation_parameters)
    logits = ol.LlamaOracle(cfg, W, False).forward(torch.as_tensor(ids)).numpy()[0, -1]
    temp, top_p = 0.6, 0.8
    proc = ol.repetition_penalty(logits, ids[0].tolist()[-20:], 1.3)
    kept = ol.top_p_filter(proc, temp, top_p)
    nucleus = set(np.flatnonzero(kept).tolist())
    # tokens whose membership is numerically ambiguous (within 1e-3 of the boundary mass) are tolerated
    p = np.exp((proc - proc.max()) / temp); p /= p.sum()
    order = np.argsort(-p)
    cum = np.cumsum(p[order])
    amb = set(order[(cum > top_p - 2e-3) & (cum < top_p + 2e-3)].tolist()) | set(order[:1].tolist())
    draws = []
    for seed in range(200):
        t, _, _ = m.generate_batch(ids, P(max_tokens=1, temperature=temp, top_p=top_p, repetition_penalty=1.3,
                                          repetition_context_size=20, seed=seed), decode_audio=False)
        draws.append(t[0][0])
    assert all(d in nucleus or d in amb for d in draws)
    assert len(set(draws)) > 5                                    # it is actually sampling
    top = int(np.argmax(kept))
    freq = draws.count(top) / len(draws)
    expect = kept[top] / kept.sum()
    assert abs(freq - expect) < 4 * np.sqrt(expect * (1 - expect) / len(draws)) + 0.02
    # same seed -> same token; top_p -> 0 degenerates to the argmax
    a, _, _ = m.generate_batch(ids, P(max_tokens=4, temperature=temp, top_p=top_p, seed=7), decode_audio=False)
    b, _, _ = m.generate_batch(ids, P(max_tokens=4, temperature=temp, top_p=top_p, seed=7), decode_audio=False)
    assert a == b
    c, _, _ = m.generate_batch(ids, P(max_tokens=1, temperature=temp, top_p=1e-6, repetition_penalty=1.3,
                                      repetition_context_size=20), decode_audio=False)
    assert c[0][0] == int(np.argmax(proc))


def test_end_to_end_tokens_to_waveform_and_errors(b2a):
    # tiny Orpheus-shaped model with the real vocabulary so parseOutput / SNAC de-interleave are exercised
    cfg = ol.LlamaConfig(hidden_size=256, num_hidden_layers=2, intermediate_size=512, num_attention_heads=2,
                         num_key_value_heads=1, head_dim=128, vocab_size=156940)
    W = ol.init_weights(cfg, 99, std=0.05)
    scfg = osnac.SNACConfig()
    SW = osnac.init_weights(scfg, 1234)
    snac = b2a.SNAC(weights=SW)
    m = b2a.LlamaTTSModel(hf_config(cfg), W, snac=snac, max_batch=8, max_context=256)
    P = type(m.default_generation_parameters)
    ids, _ = m.prepare_input_ids([[11, 22, 33, 44], [55, 66, 77, 88]])
    events = []
    toks, waves, info = m.generate_batch(ids, P(max_tokens=30, temperature=0.0, top_p=1.0, repetition_penalty=1.3,
                                                repetition_context_size=20, mask_eos=True, wrap_codes=True),
                                         on_token=lambda b, s, t: events.append((b, s, t)))
    ref = ol.generate_tokens(ol.LlamaOracle(cfg, W, False), ids, 30, temperature=0.0, rep_penalty=1.3, rep_context=20,
                             mask_eos=True)
    assert toks == ref                                             # greedy tokens bit-exact at the real vocab size
    assert [e[2] for e in events if e[0] == 0] == toks[0]          # .token events in order
    # prompt (7) + 30 generated = 37 tokens -> no start-of-speech -> whole row parsed: 35 codes -> 5 frames
    for b in range(2):
        row = ids[b].tolist() + toks[b]
        cl = ol.parse_output(np.asarray([row]))[0]
        cl = [((c % 4096) + 4096) % 4096 + 4096 * (i % 7) for i, c in enumerate(cl)]
        codes = ol.codes_from_code_list(cl)
        assert waves[b].shape == (codes[0].shape[1] * 4 * 512,)
        y0 = snac.decode(codes, zero_noise=True)[0, 0]
        # generate() draws NoiseBlock noise on the device: compare through the deterministic part only
        assert np.isfinite(waves[b]).all() and abs(np.abs(waves[b]).mean() - np.abs(y0).mean()) < 0.5 * np.abs(y0).mean() + 1e-3
    assert info.codec_time > 0 and info.tokens_per_second > 0
    # error mapping: no SNAC -> modelNotInitialized (LlamaTTS.swift:672-674); context overflow -> invalidInput
    m2 = b2a.LlamaTTSModel(hf_config(cfg), W, snac=None, max_batch=2, max_context=64)
    with pytest.raises(b2a.AudioGenerationError) as e:
        m2.generate([1, 2, 3])
    assert e.value.case == "modelNotInitialized"
    with pytest.raises(b2a.AudioGenerationError) as e:
        m2.generate_batch(ids, P(max_tokens=100), decode_audio=False)
    assert e.value.case == "invalidInput"
    # natural stop: a model that must emit END_OF_SPEECH immediately yields "No audio codes generated"? no --
    # with an empty generation the prompt itself is parsed (reference behaviour); just check it terminates
    toks3, _, info3 = m.generate_batch(ids, P(max_tokens=5, temperature=0.0), decode_audio=False)
    assert all(len(t) <= 5 for t in toks3)


def test_long_context_attention_splits(b2a):
    """Context over many 64-key attention chunks against the oracle: positions on both sides of chunk boundaries, where the
    chunks alternate between the two CTAs of the cluster and their softmax states are merged."""
    cfg = ol.LlamaConfig(hidden_size=128, num_hidden_layers=1, intermediate_size=256, num_attention_heads=3,
                         num_key_value_heads=1, head_dim=128, vocab_size=512)
    W = ol.init_weights(cfg, 5, std=0.1)
    m = b2a.LlamaTTSModel(hf_config(cfg), W, max_batch=2, max_context=400)
    ids = np.random.default_rng(1).integers(0, 512, size=(2, 330)).astype(np.int32)
    lg = m(ids)
    ref = ol.LlamaOracle(cfg, W, round_acts=False).forward(torch.as_tensor(ids)).numpy()
    for pos in (0, 63, 64, 65, 127, 128, 143, 144, 145, 191, 192, 255, 256, 287, 288, 329):
        assert rel_err(lg[:, pos], ref[:, pos]) < 1e-4, pos


# every other GQA ratio the engine accepts (q heads per kv head 1, 2, 3, 4, 6, 8; 3 is the test above), and hidden 192
LONG_CONTEXT_HEADS = [(128, 1, 1), (128, 2, 1), (128, 4, 1), (128, 6, 1), (128, 8, 1), (128, 8, 2), (192, 4, 1)]


@pytest.mark.parametrize("hidden,nq,nkv", LONG_CONTEXT_HEADS, ids=[f"h{h}-q{q}-kv{k}" for h, q, k in LONG_CONTEXT_HEADS])
def test_long_context_attention_every_gqa_ratio(b2a, hidden, nq, nkv):
    """test_long_context_attention_splits for the other GQA ratios.  330 positions (more than one prompt tile of 128) go through the
    decode step one position at a time, so each runs attn_decode_cluster_kernel<G>; at G = 8 the K/V ring is 2 chunks deep and
    wraps many times.  Hidden 192 is not a multiple of 128: the fused step's last m-tile of o_proj / down_proj is half filled, and
    its partial sums of squares cover those 64 rows only."""
    cfg = ol.LlamaConfig(hidden_size=hidden, num_hidden_layers=1, intermediate_size=256, num_attention_heads=nq,
                         num_key_value_heads=nkv, head_dim=128, vocab_size=512)
    W = ol.init_weights(cfg, 5, std=0.1)
    m = b2a.LlamaTTSModel(hf_config(cfg), W, max_batch=2, max_context=400)
    ids = np.random.default_rng(1).integers(0, 512, size=(2, 330)).astype(np.int32)
    lg = m(ids)
    ref = ol.LlamaOracle(cfg, W, round_acts=False).forward(torch.as_tensor(ids)).numpy()
    for pos in (0, 63, 64, 65, 127, 128, 143, 144, 145, 191, 192, 255, 256, 287, 288, 329):
        assert rel_err(lg[:, pos], ref[:, pos]) < 1e-4, pos


@pytest.mark.parametrize("hidden", [256, 192])
def test_debug_trace_matches_oracle_residual_stream(b2a, hidden):
    """b2a_tts_debug_trace (tools/diag_llama.py): the residual stream of the last position at every RMSNorm input -- the embedding,
    then after each layer's o_proj and down_proj, the last being the final norm's input -- as the fused step leaves it in x.  Hidden
    192 has a half-filled last m-tile."""
    cfg = ol.LlamaConfig(**{**TINY, "hidden_size": hidden})
    W = ol.init_weights(cfg, 1234, std=0.08)
    m = b2a.LlamaTTSModel(hf_config(cfg), W, max_batch=8, max_context=64)
    ids = np.random.default_rng(3).integers(0, 2048, size=(2, 12)).astype(np.int32)
    for L in (1, 12):
        m.debug_trace(True)
        lg = m(ids[:, :L])
        tr = m.debug_trace(False, batch=2, read=True)
        ref_tr = []
        ref = ol.LlamaOracle(cfg, W, round_acts=False).forward(torch.as_tensor(ids[:, :L], dtype=torch.long), trace=ref_tr).numpy()
        assert len(ref_tr) == tr.shape[0] == 2 * cfg.num_hidden_layers + 1
        for i, t in enumerate(ref_tr):
            assert rel_err(tr[i], t.numpy()) < 1e-4, (L, i, rel_err(tr[i], t.numpy()))
        assert rel_err(lg, ref) < 1e-4, (L, rel_err(lg, ref))


@pytest.mark.parametrize("hidden,inter", [(200, 512), (256, 520)], ids=["hidden200", "intermediate520"])
def test_widths_off_the_64_grid_are_rejected_at_creation(b2a, hidden, inter):
    """Every GEMM of the Llama and Qwen3 stacks takes K in whole 64-wide k-blocks, so other widths fail at creation, as Whisper's do
    (both constructors of each handle run the same check before touching the weights)."""
    llama = {**hf_config(ol.LlamaConfig(**TINY)), "hidden_size": hidden, "intermediate_size": inter}
    with pytest.raises(b2a.AudioGenerationError) as e:
        b2a.LlamaTTSModel.random_init(llama, max_batch=2, max_context=64)
    assert e.value.case == "invalidInput" and "multiple of 64" in e.value.message
    cp = b2a.Qwen3CodePredictorConfig(vocab_size=2048, hidden_size=hidden, intermediate_size=inter, num_hidden_layers=2,
                                      num_attention_heads=2, num_key_value_heads=1, num_code_groups=4)
    talker = b2a.Qwen3TalkerConfig(vocab_size=3072, hidden_size=hidden, intermediate_size=inter, num_hidden_layers=2, num_attention_heads=2,
                                   num_key_value_heads=1, num_code_groups=4, text_hidden_size=128, text_vocab_size=200, code_predictor=cp)
    with pytest.raises(b2a.AudioGenerationError) as e:
        b2a.Qwen3TTSTalker.random_init(talker, max_batch=2, max_context=64)
    assert e.value.case == "invalidInput" and "multiple of 64" in e.value.message


# (B, L, q heads, kv heads).  The batched prompt pass runs when its attention tile fits: 1024 L + 16384 G bytes <= 220 KB, so
# L <= 128 up to G = 4, L <= 124 at G = 6 and L <= 92 at G = 8.  Every case here takes it; the model built under B2A_PREFILL=step
# replays the decode step (attn_decode_cluster_kernel<G>) instead.
PREFILL_CASES = [pytest.param(3, 37, 2, 1, id="3-37"), pytest.param(8, 64, 2, 1, id="8-64"), pytest.param(1, 2, 2, 1, id="1-2"),
                 pytest.param(2, 128, 2, 1, id="2-128"), pytest.param(2, 50, 1, 1, id="g1-2-50"), pytest.param(3, 37, 3, 1, id="g3-3-37"),
                 pytest.param(2, 100, 4, 1, id="g4-2-100"), pytest.param(2, 124, 6, 1, id="g6-2-124"),
                 pytest.param(3, 92, 8, 1, id="g8-3-92")]


@pytest.mark.parametrize("B,L,nq,nkv", PREFILL_CASES)
def test_batched_prefill_matches_stepwise_and_oracle(b2a, monkeypatch, B, L, nq, nkv):
    """The tensor-core batched prompt pass (64-token hi/lo tiles + causal prompt attention, prefill_attn_kernel<G>) must give the
    same greedy continuation as replaying the decode step per position, and as the oracle; then the KV cache it left must be
    what the decode step expects: one more position fed to both models gives the same logits as each other and as the oracle."""
    cfg = ol.LlamaConfig(**{**TINY, "num_attention_heads": nq, "num_key_value_heads": nkv})
    W = ol.init_weights(cfg, 1234, std=0.08)
    ids = np.random.default_rng(100 + L).integers(0, 2048, size=(B, L)).astype(np.int32)
    P = b2a.GenerateParameters(max_tokens=12, temperature=0.0, top_p=1.0, repetition_penalty=1.0, repetition_context_size=0)
    m_b = b2a.LlamaTTSModel(hf_config(cfg), W, max_batch=8, max_context=192)
    a, _, _ = m_b.generate_batch(ids, P, decode_audio=False)
    monkeypatch.setenv("B2A_PREFILL", "step")
    m_s = b2a.LlamaTTSModel(hf_config(cfg), W, max_batch=8, max_context=192)
    monkeypatch.delenv("B2A_PREFILL")
    s, _, _ = m_s.generate_batch(ids, P, decode_audio=False)
    assert a == s
    ref = ol.generate_tokens(ol.LlamaOracle(cfg, W, False), ids, 12, temperature=0.0, rep_penalty=1.0, rep_context=0)
    assert a == ref
    # the cache now holds the prompt and the first 11 generated tokens: feed the 12th.  The two caches were written by different
    # GEMMs (prompt tiles of 64 tokens vs the fused decode step), so they agree to fp32 rounding: 1.6e-5 at most on an H100.
    nxt = np.asarray([[t[-1]] for t in a], dtype=np.int32)
    lb, ls = m_b(nxt, reset_cache=False), m_s(nxt, reset_cache=False)
    assert rel_err(lb, ls) < 4e-5, rel_err(lb, ls)
    full = np.concatenate([ids, np.asarray(a, dtype=np.int32)], axis=1)
    ref_lg = ol.LlamaOracle(cfg, W, False).forward(torch.as_tensor(full)).numpy()[:, -1:]
    assert rel_err(lb, ref_lg) < 1e-4, rel_err(lb, ref_lg)
    assert rel_err(ls, ref_lg) < 1e-4, rel_err(ls, ref_lg)


def test_streamed_audio_chunks_match_the_one_shot_waveform(b2a):
    """Row N2 (b2a_tts_generate_stream): chunks are produced DURING generation, they tile the utterance exactly, and away from chunk
    ends (the codec's look-ahead) they equal the one-shot decode of the same codes."""
    cfg = ol.LlamaConfig(hidden_size=256, num_hidden_layers=2, intermediate_size=512, num_attention_heads=2,
                         num_key_value_heads=1, head_dim=128, vocab_size=156940)
    W = ol.init_weights(cfg, 99, std=0.05)
    scfg = osnac.SNACConfig()
    scfg.noise = False                                              # NoiseBlock noise is drawn per call: compare the deterministic part
    SW = osnac.init_weights(scfg, 1234)
    snac = b2a.SNAC(weights=SW, noise=False)
    m = b2a.LlamaTTSModel(hf_config(cfg), W, snac=snac, max_batch=2, max_context=512)
    P = type(m.default_generation_parameters)
    ids, _ = m.prepare_input_ids([[11, 22, 33, 44], [55, 66, 77, 88]])
    ids[:, -1] = 128257                                             # START_OF_SPEECH: parseOutput keeps the generated codes only
    p = P(max_tokens=7 * 23 + 3, temperature=0.0, top_p=1.0, repetition_penalty=1.3, repetition_context_size=20, mask_eos=True, wrap_codes=True)
    toks, waves, _ = m.generate_batch(ids, p)
    order = []
    toks_s, chunks, info = m.generate_audio_chunks(ids, p, frames_per_chunk=4, left_context_frames=8,
                                                   on_audio=lambda b, a, fin: order.append(("audio", b, len(a), fin)),
                                                   on_token=lambda b, s, t: order.append(("token", b, s)))
    assert toks_s == toks and info.codec_time > 0
    # audio events are interleaved with token events (emission happens while tokens are still being generated)
    first_audio = next(i for i, e in enumerate(order) if e[0] == "audio")
    last_token = max(i for i, e in enumerate(order) if e[0] == "token")
    assert first_audio < last_token
    assert [e[3] for e in order if e[0] == "audio" and e[1] == 0][-1] is True
    for b in range(2):
        cat = np.concatenate(chunks[b])
        assert len(cat) == len(waves[b]) == 23 * 2048 and all(len(c) == 4 * 2048 for c in chunks[b][:-1])
        peak = np.abs(waves[b]).max()
        err = np.abs(cat - waves[b]) / peak
        edge = np.zeros(len(cat), bool)                             # the last 2 frames of every non-final chunk lack their look-ahead
        pos = 0
        for c in chunks[b][:-1]:
            pos += len(c)
            edge[pos - 2 * 2048: pos] = True
        assert err[~edge].max() < 1e-3, err[~edge].max()
        assert err.max() < 1.0                                      # and the edges are still the same signal, not garbage
