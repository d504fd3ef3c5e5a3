"""Qwen3-TTS voice-cloning (ICL) prompts through the C ABI: codecEmbedIcl's frame rows (b2a_qwen3_talker_embed_code_frames), the
prompt of prepareReferenceConditioning + prepareICLGenerationInputs (Qwen3TTS.swift:709-837), greedy frames from such a prompt against
the teacher-forced oracle, and generate's reference-code cut (:550-565).  Small head_dim-128 talker of test_gpu_qwen3_talker.py."""
import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import qwen3_tts as ot
from test_gpu_qwen3_talker import TTS, bf16_weights, device_model, small_cfg

pytestmark = pytest.mark.gpu
REF_CHAT = [151, 12, 13, 60, 61, 62, 63, 64, 152, 14]                     # "<|im_start|>assistant\n{ref text}<|im_end|>\n"
TARGET_CHAT = [151, 12, 13, 40, 41, 42, 43, 44, 45, 152, 14, 151, 12, 13]   # "...{text}<|im_end|>\n<|im_start|>assistant\n"


@pytest.fixture(scope="module")
def small(b2a):
    cfg = small_cfg()
    W = bf16_weights(cfg, 5)
    return cfg, W, device_model(b2a, cfg, W, max_batch=2, max_context=128)


def ref_codes(cfg, T=6, seed=0):
    rng = np.random.default_rng(seed)
    c = rng.integers(1, cfg.code_predictor.vocab_size, (cfg.num_code_groups, T)).astype(np.int32)
    return c


def frames_f32(cfg, W, codes_tg):
    """codecEmbedIcl's frame rows in float32, summed in the device's order, from the oracle's bf16 tables: codes [n, groups]."""
    e = W["model.codec_embedding.weight"].to(torch.float32).numpy()[codes_tg[:, 0]]
    for g in range(1, codes_tg.shape[1]):
        e = e + W[f"code_predictor.model.codec_embedding.{g - 1}.weight"].to(torch.float32).numpy()[codes_tg[:, g]]
    return e


def icl_prompt(emb_text, emb_codec, emb_frames, cfg, rc, ref_chat, target_chat, tts_bos, tts_eos, tts_pad, language_id=None, speaker=None,
               think=2154, nothink=2155, think_bos=2156, think_eos=2157, pad=2148, bos=2149):
    """prepareReferenceConditioning's slicing + prepareICLGenerationInputs (Qwen3TTS.swift:725-837), restated over row functions."""
    ref_text = ref_chat[min(3, len(ref_chat)):max(min(3, len(ref_chat)), len(ref_chat) - 2)]
    target_text = target_chat[min(3, len(target_chat)):max(min(3, len(target_chat)), len(target_chat) - 5)]
    tts = emb_text([tts_bos, tts_eos, tts_pad])
    text = np.concatenate([emb_text(ref_text + target_text), tts[1:2]], 0) + emb_codec([pad])
    codec = np.concatenate([emb_codec([bos]), emb_frames(rc.T)], 0) + tts[2:3]
    prefill = [think, think_bos, language_id, think_eos] if language_id is not None else [nothink, think_bos, think_eos]
    prefix = np.concatenate([emb_codec(prefill)] + ([speaker[None]] if speaker is not None else []) + [emb_codec([pad, bos])], 0)
    combined = np.concatenate([np.repeat(tts[2:3], prefix.shape[0] - 2, 0), tts[0:1]], 0) + prefix[:-1]
    return np.concatenate([emb_text(target_chat[:3]), combined, text, codec], 0), tts[2:3]


def oracle_rows(cfg, W):
    t = ot.Talker(cfg, W)
    et = lambda ids: t.embed_text(torch.as_tensor([list(ids)]))[0].numpy()
    ec = lambda ids: t.embed_codec(torch.as_tensor([list(ids)]))[0].numpy()
    p = ot.CodePredictor(cfg, W)

    def ef(c):
        e = ec(c[:, 0])
        for g in range(1, c.shape[1]):
            e = e + p.embed(g - 1, torch.as_tensor(c[:, g])).numpy()
        return e
    return et, ec, ef


def test_embed_code_frames(small):
    cfg, W, m = small
    rc = ref_codes(cfg, 9).T.copy()                                          # [9, G]
    rc[0, 0] = cfg.vocab_size - 1                                           # c0 reaches the talker's (larger) codec table
    assert np.array_equal(m.embed_code_frames(rc), frames_f32(cfg, W, rc))
    assert np.array_equal(m.embed_code_frames(rc[:, :2]), frames_f32(cfg, W, rc[:, :2]))     # fewer groups: the reference's break
    assert np.array_equal(m.embed_code_frames(rc[:, :1]), m.embed_codec(rc[:, 0]))
    _, _, ef = oracle_rows(cfg, W)
    assert rel_err(m.embed_code_frames(rc), ef(rc)) < 1e-6
    from mlx_audio_swift_b200 import _ffi
    for bad in (np.concatenate([rc, rc[:, :1]], 1), np.full((2, cfg.num_code_groups), cfg.code_predictor.vocab_size, np.int32), np.zeros((0, 4), np.int32)):
        with pytest.raises(_ffi.AudioGenerationError) as e:
            m.embed_code_frames(bad)
        assert e.value.case == "invalidInput"


@pytest.mark.parametrize("language_id", [None, 2160])
@pytest.mark.parametrize("with_speaker", [False, True])
def test_icl_prompt_bit_exact_and_vs_oracle(small, language_id, with_speaker):
    cfg, W, m = small
    rc = ref_codes(cfg)
    spk = np.random.default_rng(1).standard_normal(cfg.hidden_size).astype(np.float32) if with_speaker else None
    inp, trail, pad = m.prepare_icl_generation_inputs(rc, REF_CHAT, TARGET_CHAT, **TTS, language_id=language_id, speaker_embedding=spk)
    ref, ref_pad = icl_prompt(m.embed_text, m.embed_codec, m.embed_code_frames, cfg, rc, REF_CHAT, TARGET_CHAT, **TTS, language_id=language_id, speaker=spk)
    assert np.array_equal(inp, ref) and np.array_equal(trail, ref_pad) and np.array_equal(pad, ref_pad[0])
    L = 3 + (4 if language_id else 3) + (1 if with_speaker else 0) + 1 + (5 + 6 + 1) + (1 + rc.shape[1])
    assert inp.shape == (L, cfg.hidden_size)
    o, o_pad = icl_prompt(*oracle_rows(cfg, W), cfg, rc, REF_CHAT, TARGET_CHAT, **TTS, language_id=language_id,
                          speaker=spk.astype(np.float64) if with_speaker else None)
    assert rel_err(inp, o) < 1e-5 and rel_err(pad, o_pad[0]) < 1e-5
    assert np.array_equal(m.prepare_icl_generation_inputs(rc[None], REF_CHAT, TARGET_CHAT, **TTS, language_id=language_id, speaker_embedding=spk)[0], inp)


def test_base_checkpoint_needs_a_speaker_embedding(small):
    from mlx_audio_swift_b200 import _ffi
    cfg, W, m = small
    m.config.tts_model_type = "base"
    try:
        with pytest.raises(_ffi.AudioGenerationError) as e:
            m.prepare_icl_generation_inputs(ref_codes(cfg), REF_CHAT, TARGET_CHAT, **TTS)
        assert e.value.case == "invalidInput" and "speaker" in e.value.message
        spk = np.zeros(cfg.hidden_size, np.float32)
        assert m.prepare_icl_generation_inputs(ref_codes(cfg), REF_CHAT, TARGET_CHAT, **TTS, speaker_embedding=spk)[0].shape[0] > 0
    finally:
        m.config.tts_model_type = ""


def test_greedy_frames_from_icl_prompt_vs_oracle(b2a, small):
    cfg, W, m = small
    rc = ref_codes(cfg, 5, seed=3)
    o, o_pad = icl_prompt(*oracle_rows(cfg, W), cfg, rc, REF_CHAT, TARGET_CHAT, **TTS, language_id=2160)
    ri, rp = torch.from_numpy(o)[None], torch.from_numpy(o_pad)[None]
    P = b2a.Qwen3GenerateParameters(max_tokens=10, temperature=0.0, repetition_penalty=1.05, mask_eos=True)
    codes, info = m.generate_codes(o[None].astype(np.float32), [o_pad.astype(np.float32)], o_pad[0].astype(np.float32), P)
    ref = ot.generate_codes(cfg, W, ri, rp, rp, max_tokens=10, temperature=0.0, repetition_penalty=1.05, stop_on_eos=False).numpy()
    assert codes[0].shape == ref.shape == (10, cfg.num_code_groups)
    assert np.array_equal(codes[0], ref), (codes[0], ref)


def test_generate_cuts_the_reference_audio(b2a, small):
    from mlx_audio_swift_b200 import qwen3_tts_codec as q
    cfg, W, m = small
    dcfg = q.Qwen3TTSTokenizerDecoderConfig(codebook_size=2048, codebook_dim=32, latent_dim=64, decoder_dim=128, hidden_size=64, intermediate_size=128,
                                            num_attention_heads=2, num_key_value_heads=2, num_hidden_layers=1, num_quantizers=cfg.num_code_groups,
                                            upsample_rates=[8, 5, 4, 3], upsampling_ratios=[2, 2])
    tok = q.Qwen3TTSSpeechTokenizer(dcfg, weights=q.random_init_weights(dcfg))
    model = b2a.Qwen3TTSModel(m, tok)
    rc = ref_codes(cfg, 7, seed=4)
    inp, trail, pad = m.prepare_icl_generation_inputs(rc, REF_CHAT, TARGET_CHAT, **TTS, language_id=2160)
    P = b2a.Qwen3GenerateParameters(max_tokens=9, temperature=0.0, mask_eos=True)
    gen = m.generate_codes(inp[None], [trail], pad, P)[0][0]
    audio = model.generate(inp, trail, pad, P, ref_codes=rc)
    full, lengths = tok.decode(np.concatenate([rc.T, gen], 0)[None])
    valid = full[0, :int(lengths[0])] if 0 < int(lengths[0]) < full.shape[1] else full[0]
    cut = int(rc.shape[1] / (rc.shape[1] + gen.shape[0]) * valid.shape[0])
    assert cut > 0 and audio.shape == (valid.shape[0] - cut,) and np.array_equal(audio, valid[cut:])
    w, l = tok.decode(gen[None])                                                                       # without ref_codes: no prefix, no cut
    assert np.array_equal(model.generate(inp, trail, pad, P), w[0, :int(l[0])] if 0 < int(l[0]) < w.shape[1] else w[0])
    events = list(model.generate_stream(inp, trail, pad, P, streaming_interval=0.4, ref_codes=rc))     # streaming: no ref prefix, no cut
    streamed = np.concatenate([e[1] for e in events if e[0] == "audio"])
    assert streamed.shape == (gen.shape[0] * 1920,)
