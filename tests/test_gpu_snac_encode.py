"""CUDA SNAC encode (through the C ABI) against the float64 reference (tests/snac_encoder_reference.py) and its golden, and voice
cloning prompts for Orpheus built from a device-encoded reference clip.

Latent z: max |diff| / max |ref| and relative L2 below 1e-3 (the bf16 hi/lo tensor-core products track fp32 to ~1e-5).  Codes:
bit-exact against the ordered-fp32 code search run on the device's own z; against the float64 end-to-end reference a code may
differ only where that level's float64 search is a near-tie, or inside the time span of a differing code of a coarser level
(whose residual the finer levels then search)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import snac_encoder_reference as ser
from conftest import GOLDEN, max_rel_to_peak, rel_err
from oracle import llama as ol
from oracle import snac as osnac

pytestmark = pytest.mark.gpu
TOL = 1e-3
TIE_GAP = 1e-3    # float64 distance gap (normalised vectors, distances in [0, 4]) below which a level's search counts as a near-tie


@pytest.fixture(scope="module")
def model(b2a):
    cfg = osnac.SNACConfig()
    W = {**osnac.init_weights(cfg, 1234), **ser.init_encoder_weights(cfg, 4321)}
    return cfg, W, b2a.SNAC(weights=W)


def device_latent(b2a, m, audio):
    a = np.ascontiguousarray(audio[:, 0], dtype=np.float32)
    B, n = a.shape
    z = np.empty((B, 768, m.encoded_length(n)), dtype=np.float32)
    b2a._ffi.check(b2a._ffi.lib().b2a_snac_encode_latent_test(m._h, b2a._ffi.ptr(a), B, n, b2a._ffi.ptr(z)))
    return z


def search_gaps(cfg, W, z):
    """The float64 residual VQ along the reference's own path: codes and, per level, the gap between the two smallest distances."""
    codes, gaps = [], []
    with torch.no_grad():
        res = osnac._t(z)
        for i, s in enumerate(cfg.vq_strides):
            q = f"quantizer.quantizers.{i}"
            x = F.avg_pool1d(res, s, s) if s > 1 else res
            e = osnac.wn_conv1d(W, q + ".in_proj", x).permute(0, 2, 1).numpy()            # [B, Ts, D]
            e = e / np.maximum(np.linalg.norm(e, axis=-1, keepdims=True), 1e-12)
            c = W[q + ".codebook.weight"].astype(np.float64)
            c = c / np.maximum(np.linalg.norm(c, axis=1, keepdims=True), 1e-12)
            d = (e ** 2).sum(-1, keepdims=True) - 2 * e @ c.T + (c ** 2).sum(1)
            idx = d.argmin(-1)
            part = np.partition(d, 1, axis=-1)
            codes.append(idx.astype(np.int32)); gaps.append(part[..., 1] - part[..., 0])
            zq = osnac.wn_conv1d(W, q + ".out_proj", osnac._t(W[q + ".codebook.weight"])[torch.as_tensor(idx)].transpose(1, 2))
            res = res - (torch.repeat_interleave(zq, s, dim=2) if s > 1 else zq)
    return codes, gaps


def assert_codes_explained(cfg, dev, ref, gaps):
    """Every device / reference code difference is a near-tie of its level or lies under a coarser level's difference."""
    for b in range(ref[0].shape[0]):
        bad_steps = np.zeros(ref[-1].shape[1] * cfg.vq_strides[-1], dtype=bool)      # latent steps under a coarser mismatch
        for i, s in enumerate(cfg.vq_strides):
            diff = np.flatnonzero(dev[i][b] != ref[i][b])
            for j in diff:
                assert gaps[i][b, j] < TIE_GAP or bad_steps[j * s:(j + 1) * s].any(), (b, i, j, gaps[i][b, j])
            for j in diff:
                bad_steps[j * s:(j + 1) * s] = True


@pytest.mark.parametrize("B,n", [(1, 2048), (3, 12000), (2, 50000)])
def test_latent_and_codes_vs_reference(b2a, model, B, n):
    cfg, W, m = model
    audio = ser.synth_clip(B, n, seed=n)
    z = device_latent(b2a, m, audio)
    zr = ser.encode_latent(cfg, W, audio)
    assert z.shape == zr.shape == (B, 768, -(-n // 2048) * 4)
    assert max_rel_to_peak(z, zr) < TOL and rel_err(z, zr) < TOL, (max_rel_to_peak(z, zr), rel_err(z, zr))
    codes = m.encode(audio)
    assert [c.shape for c in codes] == [(B, zr.shape[2] // s) for s in cfg.vq_strides]
    _, from_z = osnac.quantize(cfg, W, z)                 # the device's search is the ordered-fp32 one, bit for bit
    assert all(np.array_equal(a, b) for a, b in zip(codes, from_z))
    ref, gaps = search_gaps(cfg, W, zr)
    assert_codes_explained(cfg, codes, ref, gaps)


def test_golden(b2a, model):
    cfg, W, m = model
    g = np.load(GOLDEN / "snac_encode.npz")
    audio = ser.synth_clip(2, 5000, 3)                            # tests/golden/make_golden_snac_encode.py
    z = device_latent(b2a, m, audio)
    assert tuple(g["z_shape"]) == z.shape
    peak = max(abs(g["z_stats"][2]), abs(g["z_stats"][3]))
    assert np.abs(z.reshape(-1)[:16] - g["z_first"]).max() < TOL * peak
    zs = np.array([z.mean(), np.abs(z).mean(), z.min(), z.max()])
    assert np.abs(zs - g["z_stats"]).max() < TOL * peak
    codes = m.encode_audio(audio)
    _, gaps = search_gaps(cfg, W, ser.encode_latent(cfg, W, audio))
    assert_codes_explained(cfg, codes, [g[f"codes{i}"] for i in range(3)], gaps)


def test_batched_equals_serial_and_deterministic(model):
    cfg, W, m = model
    audio = ser.synth_clip(4, 30000, seed=9)
    audio[2] *= 0.3
    full = m.encode(audio)
    again = m.encode(audio)
    assert all(np.array_equal(a, b) for a, b in zip(full, again))
    for b in range(4):
        one = m.encode(audio[b:b + 1])
        assert all(np.array_equal(f[b:b + 1], o) for f, o in zip(full, one))


def test_device_entry_matches_host_entry(model):
    cfg, W, m = model
    audio = ser.synth_clip(2, 20000, seed=5)
    host = m.encode(audio)
    T = m.encoded_length(20000)
    d_codes = [torch.empty((2, T // s), dtype=torch.int32, device="cuda") for s in cfg.vq_strides]
    m.encode_dev(torch.from_numpy(audio).cuda(), d_codes, stream=m.stream)
    torch.cuda.synchronize()
    assert all(np.array_equal(h, d.cpu().numpy()) for h, d in zip(host, d_codes))


def test_full_size_properties(b2a, model):
    """B = 8 x 30 s: finite latent; a 10 s prefix of a clip gives the whole clip's codes away from the cut (finite receptive field);
    a 1 s prefix against the reference."""
    cfg, W, m = model
    n = 30 * 24000
    audio = ser.synth_clip(8, n, seed=1)
    z = device_latent(b2a, m, audio)
    assert z.shape == (8, 768, m.encoded_length(n)) and np.isfinite(z).all()
    codes = m.encode(audio)
    assert [c.shape for c in codes] == [(8, z.shape[2] // s) for s in cfg.vq_strides]
    pre = m.encode(audio[3:4, :, :240000])
    keep = (m.encoded_length(240000) - 32) // 4 * 4               # latent steps clear of the cut's receptive field
    for i, s in enumerate(cfg.vq_strides):
        assert np.array_equal(pre[i][0, :keep // s], codes[i][3, :keep // s]), i
    short = audio[5:6, :, :24000]
    zs, zr = device_latent(b2a, m, short), ser.encode_latent(cfg, W, short)
    assert max_rel_to_peak(zs, zr) < TOL
    assert max_rel_to_peak(z[5:6, :, :32], zr[:, :, :32]) < TOL


# geometries whose widths are all padded, including the last one: encoder_dim 50 -> stages 50 / 100 / 200 / 400 at 64 / 128 / 256 / 448
# channels and latent 800 stored at 832; encoder_dim 8 -> latent 32 stored at 64 (the final depthwise conv reads the padded rows)
@pytest.mark.parametrize("enc_dim,rates,vq,n", [(50, (2, 4, 8, 8), (4, 2, 1), 12000), (8, (2, 2), (2, 1), 3000)],
                         ids=["latent800", "latent32"])
def test_padded_geometries_vs_reference(b2a, enc_dim, rates, vq, n):
    cfg = osnac.SNACConfig(encoder_dim=enc_dim, encoder_rates=rates, decoder_dim=64, decoder_rates=(2,), vq_strides=vq)
    W = {**osnac.init_weights(cfg, 5), **ser.init_encoder_weights(cfg, 6)}
    m = b2a.SNAC(encoder_dim=enc_dim, encoder_rates=rates, decoder_dim=64, decoder_rates=(2,), vq_strides=vq, weights=W)
    audio = ser.synth_clip(2, n, seed=4)
    a = np.ascontiguousarray(audio[:, 0])
    T = m.encoded_length(n)
    z = np.empty((2, cfg.latent, T), dtype=np.float32)
    b2a._ffi.check(b2a._ffi.lib().b2a_snac_encode_latent_test(m._h, b2a._ffi.ptr(a), 2, n, b2a._ffi.ptr(z)))
    zr = ser.encode_latent(cfg, W, audio)
    assert z.shape == zr.shape
    assert max_rel_to_peak(z, zr) < TOL and rel_err(z, zr) < TOL, (max_rel_to_peak(z, zr), rel_err(z, zr))
    codes = m.encode(audio)
    _, from_z = osnac.quantize(cfg, W, z)
    assert all(np.array_equal(c, f) for c, f in zip(codes, from_z))
    ref, gaps = search_gaps(cfg, W, zr)
    assert_codes_explained(cfg, codes, ref, gaps)


def test_device_entries_reject_mismatched_buffers(b2a, model):
    cfg, W, m = model
    T = m.encoded_length(4096)
    wave = torch.zeros((1, 1, 4096), device="cuda")
    good = [torch.empty((1, T // s), dtype=torch.int32, device="cuda") for s in cfg.vq_strides]
    bad_sets = [good[:2], good[:2] + [torch.empty((1, T - 1), dtype=torch.int32, device="cuda")],
                good[:2] + [torch.empty((1, T), dtype=torch.int64, device="cuda")], good[:2] + [good[2].cpu()]]
    for codes in bad_sets:
        with pytest.raises(b2a.AudioGenerationError) as e:
            m.encode_dev(wave, codes, stream=m.stream)
        assert e.value.case == "invalidInput"
    for w in (wave.double(), wave.cpu(), torch.zeros((1, 2, 4096), device="cuda")):
        with pytest.raises(b2a.AudioGenerationError) as e:
            m.encode_dev(w, good, stream=m.stream)
        assert e.value.case == "invalidInput"
    m.encode_dev(wave, good, stream=m.stream)
    torch.cuda.synchronize()
    with pytest.raises(b2a.AudioGenerationError) as e:
        m.decode_dev(good[:2], torch.empty((1, 1, T * 512), device="cuda"))
    assert e.value.case == "invalidInput"
    with pytest.raises(b2a.AudioGenerationError) as e:
        m.decode_dev(good, torch.empty((1, 1, T * 512 - 1), device="cuda"))
    assert e.value.case == "invalidInput"


def test_errors_and_decoder_only_handle(b2a, model):
    cfg, W, m = model
    with pytest.raises(b2a.AudioGenerationError) as e:
        m.encode(np.zeros((1, 1, 0), dtype=np.float32))
    assert e.value.case == "audioEncodingFailed"
    dec_only = b2a.SNAC(weights=osnac.init_weights(cfg, 1234))
    assert dec_only.encoded_length(4096) == 0
    with pytest.raises(b2a.AudioGenerationError) as e:
        dec_only.encode(ser.synth_clip(1, 4096))
    assert e.value.case == "modelNotInitialized"
    codes = osnac.synth_codes(cfg, 2, 16, seed=2)
    a, b = dec_only.decode(codes, zero_noise=True), m.decode(codes, zero_noise=True)
    assert np.array_equal(a, b)
    assert max_rel_to_peak(a, np.load(GOLDEN / "snac.npz")["wave_nonoise"]) < TOL
    # a malformed encoder tensor leaves the decoder working and encode reports the model as not initialised
    bad = dict(W)
    bad["encoder.block.layers.2.block.layers.4.weight_v"] = np.zeros((3, 3, 3), dtype=np.float32)
    mb = b2a.SNAC(weights=bad)
    assert np.array_equal(mb.decode(codes, zero_noise=True), b)
    with pytest.raises(b2a.AudioGenerationError) as e:
        mb.encode(ser.synth_clip(1, 4096))
    assert e.value.case == "modelNotInitialized"


def _hf(cfg):
    return dict(hidden_size=cfg.hidden_size, num_hidden_layers=cfg.num_hidden_layers, intermediate_size=cfg.intermediate_size,
                num_attention_heads=cfg.num_attention_heads, num_key_value_heads=cfg.num_key_value_heads, head_dim=cfg.head_dim,
                vocab_size=cfg.vocab_size, rms_norm_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta, tie_word_embeddings=True,
                rope_scaling={"rope_type": "llama3", "factor": 32.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                              "original_max_position_embeddings": 8192})


@pytest.mark.parametrize("n_ref,text_len", [(4096, 5), (12000, 80)], ids=["batched-prefill", "stepwise-prefill"])
def test_orpheus_cloning_prompt_and_greedy_generation(b2a, model, n_ref, text_len):
    """prepareInputIds with refAudio / refText (LlamaTTS.swift:446-553) from a device-encoded reference: the framing equals the
    reference restatement on the same codes, and greedy generation from that prompt equals the teacher-forced oracle, for a prompt
    of <= 128 tokens (batched prefill) and one of more (token-by-token prefill)."""
    scfg, SW, snac = model
    cfg = ol.LlamaConfig(hidden_size=256, num_hidden_layers=2, intermediate_size=512, num_attention_heads=2,
                         num_key_value_heads=1, head_dim=128, vocab_size=156940)
    W = ol.init_weights(cfg, 99, std=0.05)
    m = b2a.LlamaTTSModel(_hf(cfg), W, snac=snac, max_batch=4, max_context=320)
    ref_audio = ser.synth_clip(1, n_ref, seed=n_ref)[0, 0]
    code_list = m.encode_audio_to_code_list(ref_audio)
    assert code_list == ol.code_list_from_codes(snac.encode(ref_audio[None, None]))
    ref_text = list(range(1000, 1000 + text_len))
    prompts = [[11, 22, 33, 44], [55, 66]]
    ids, mask = m.prepare_input_ids(prompts, code_list, ref_text)
    assert np.array_equal(ids, ser.prepare_input_ids_ref(prompts, ref_text, code_list))
    assert np.array_equal(mask, ids != 128263)
    assert (ids.shape[1] <= 128) == (n_ref == 4096)
    P = b2a.GenerateParameters(max_tokens=10, temperature=0.0, top_p=1.0, repetition_penalty=1.3, repetition_context_size=20,
                               mask_eos=True)
    toks, _, info = m.generate_batch(ids, P, decode_audio=False)
    ref = ol.generate_tokens(ol.LlamaOracle(cfg, W, False), ids, 10, temperature=0.0, rep_penalty=1.3, rep_context=20, mask_eos=True)
    assert toks == ref and info.prompt_token_count == ids.shape[1]
    # parseOutput crops after the last start-of-speech over prompt + generated tokens (the reference block's SOS here)
    full = np.concatenate([ids, np.asarray(toks, dtype=np.int32)], axis=1)
    assert m.parse_output(full) == ol.parse_output(full)
    # the generate entry points clone only when both the audio and its transcript are given
    P = b2a.GenerateParameters(max_tokens=10, temperature=0.0, top_p=1.0, repetition_penalty=1.3, repetition_context_size=20,
                               mask_eos=True, wrap_codes=True)
    ev = [v for k, v in m.generate_stream(prompts[0], P, ref_audio=ref_audio, ref_text_ids=ref_text) if k == "token"]
    one, _ = m.prepare_input_ids(prompts[:1], code_list, ref_text)
    assert ev == m.generate_batch(one, P, decode_audio=False)[0][0]
    plain = [v for k, v in m.generate_stream(prompts[0], P, ref_audio=ref_audio) if k == "token"]
    assert plain == m.generate_batch(m.prepare_input_ids(prompts[:1])[0], P, decode_audio=False)[0][0]
