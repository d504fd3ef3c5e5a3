"""Qwen3-TTS speaker encoder through the C ABI (b2a_qwen3_speaker_encoder_*): the 1024-point log-mel front-end, the ECAPA-TDNN
against the float64 reference (tests/qwen3_speaker_encoder_reference.py, itself pinned against transformers' ECAPA_TimeDelayNet in
test_oracle_qwen3_tts_speaker.py), determinism, the golden fixture, the errors, directory loading and the voice-cloning prompt
built from reference audio.  Tolerance: max |diff| / max |ref| and relative L2 below 1e-3."""
import json

import numpy as np
import pytest
import torch

import qwen3_speaker_encoder_reference as ser
from conftest import GOLDEN, max_rel_to_peak, rel_err
from oracle import dsp
from test_gpu_qwen3_talker import bf16_weights, device_model, small_cfg
from test_gpu_qwen3_tts_icl import REF_CHAT, TARGET_CHAT, TTS

pytestmark = pytest.mark.gpu
TOL = 1e-3
SMALL = dict(enc_channels=[96, 96, 96, 192], enc_kernel_sizes=[5, 3, 3, 3], enc_dilations=[1, 2, 3, 1], enc_attention_channels=80,
             enc_res2net_scale=4, enc_se_channels=72, enc_dim=48)


def model(b2a, seed=7, **kw):
    from mlx_audio_swift_b200.qwen3_tts import random_init_speaker_encoder_weights
    cfg = b2a.Qwen3SpeakerEncoderConfig(**kw)
    W = random_init_speaker_encoder_weights(cfg, seed=seed)
    return cfg, W, b2a.Qwen3TTSSpeakerEncoder(cfg, W)


@pytest.fixture(scope="module")
def small(b2a):
    return model(b2a, **SMALL)


@pytest.fixture(scope="module")
def shipped(b2a):
    return model(b2a, seed=11)


def errors(label, got, want):
    peak, l2 = max_rel_to_peak(got, want), rel_err(got, want)
    print(f"{label}: max/peak {peak:.2e}, rel L2 {l2:.2e}")
    assert peak < TOL and l2 < TOL


# ------------------------------------------------------------------ mel front-end at n_fft = 1024
@pytest.mark.parametrize("B,n", [(2, 513), (3, 1024), (2, 24017), (2, 30 * 24000)])
def test_logmel_1024_vs_oracle(b2a, B, n):
    lm = b2a.LogMel("core", 24000, 1024, 256, 128)
    x = ser.synth_clip(B, n, seed=n)
    got = lm(x)
    assert got.shape == (B, 1 + n // 256, 128) and lm.frames(n) == 1 + n // 256
    for b in range(B):
        want = dsp.compute_mel_spectrogram(x[b], 24000, 1024, 256, 128)
        assert max_rel_to_peak(got[b], want) < TOL, (b, max_rel_to_peak(got[b], want))


def test_logmel_1024_rejects_short_clips_and_other_sizes(b2a):
    from mlx_audio_swift_b200 import _ffi
    lm = b2a.LogMel("core", 24000, 1024, 256, 128)
    with pytest.raises(_ffi.AudioGenerationError) as e:
        lm(np.zeros((1, 512), np.float32))
    assert e.value.case == "invalidInput"
    for n_fft in (512, 2048):
        with pytest.raises(_ffi.AudioGenerationError) as e:
            b2a.LogMel("core", 24000, n_fft, 256, 128)
        assert e.value.case == "invalidInput"


def test_streaming_mel_1024_vs_oracle(b2a):
    x = ser.synth_clip(1, 60000, seed=2)[0]
    cuts = [0, 300, 1500, 9000, 33333, 60000]
    m, o = b2a.IncrementalMelSpectrogram(24000, 1024, 256, 128), dsp.IncrementalMelSpectrogram(24000, 1024, 256, 128)
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        a, r = m.process(x[lo:hi]), o.process(x[lo:hi])
        assert (a is None) == (r is None)
        if a is not None:
            assert a.shape == r.shape and max_rel_to_peak(a, r) < TOL
    a, r = m.flush(), o.flush()
    assert a.shape == r.shape and max_rel_to_peak(a, r) < TOL
    assert m.total_frames == o.total_frames


# ------------------------------------------------------------------ the network against float64
@pytest.mark.parametrize("geometry,B,n", [("small", 2, 30000), ("small", 1, 1024), ("shipped", 2, 4 * 24000), ("shipped", 1, 1024)])
def test_embed_mel_vs_float64(b2a, small, shipped, geometry, B, n):
    cfg, W, m = small if geometry == "small" else shipped
    mel = np.stack([ser.log_mel(r) for r in ser.synth_clip(B, n, seed=B + n)])
    got = m.embed_mel(mel.astype(np.float32))
    assert got.shape == (B, cfg.enc_dim)
    errors(f"embed_mel {geometry} B={B} n={n}", got, ser.forward(cfg, W, mel))


@pytest.mark.parametrize("geometry,B,n", [("small", 2, 30000), ("shipped", 2, 4 * 24000), ("shipped", 1, 10 * 24000)])
def test_embed_audio_vs_float64(b2a, small, shipped, geometry, B, n):
    cfg, W, m = small if geometry == "small" else shipped
    x = ser.synth_clip(B, n, seed=n)
    got = m.embed(x)
    errors(f"embed {geometry} B={B} n={n}", got, ser.embed(cfg, W, x))
    assert np.array_equal(m(x), got[0])                                   # extractSpeakerEmbedding: row 0
    assert np.array_equal(m(x[0]), got[0]) and np.array_equal(m(x[:, None, :]), got[0])


def test_deterministic_batched_serial_dev_host(b2a, shipped):
    cfg, W, m = shipped
    x = ser.synth_clip(3, 3 * 24000 + 77, seed=4)
    batched = m.embed(x)
    assert np.array_equal(batched, m.embed(x))                           # two calls
    for b in range(3):
        assert np.array_equal(m.embed(x[b:b + 1]), batched[b:b + 1]), b  # batched == serial
    d_x = torch.from_numpy(x).cuda()
    d_out = torch.empty((3, cfg.enc_dim), dtype=torch.float32, device="cuda")
    m.embed_dev(d_x, d_out, stream=m.stream)
    torch.cuda.ExternalStream(m.stream).synchronize()
    assert np.array_equal(d_out.cpu().numpy(), batched)                  # device entry == host entry
    mel = b2a.LogMel("core", 24000, 1024, 256, 128)(x)
    assert np.array_equal(m.embed_mel(mel), batched)                     # the two halves compose to the whole


def test_golden(b2a):
    import sys
    sys.path.insert(0, str(GOLDEN))
    import make_golden_qwen3_speaker as mg
    g = np.load(GOLDEN / "qwen3_speaker.npz")
    cfg, W = mg.weights()
    got = b2a.Qwen3TTSSpeakerEncoder(cfg, W).embed(mg.clip())
    errors("golden", got, g["embedding"])


# ------------------------------------------------------------------ errors
def test_errors(b2a, small, shipped):
    from mlx_audio_swift_b200 import _ffi
    cfg, W, m = small

    def case(fn):
        with pytest.raises(_ffi.AudioGenerationError) as e:
            fn()
        return e.value.case

    bad = [dict(SMALL, mel_dim=80), dict(SMALL, enc_res2net_scale=5), dict(SMALL, enc_channels=[96, 96, 96, 160]),
           dict(SMALL, enc_kernel_sizes=[4, 3, 3, 3]), dict(SMALL, enc_channels=[96, 96, 96])]
    for kw in bad:
        assert case(lambda: b2a.Qwen3TTSSpeakerEncoder(b2a.Qwen3SpeakerEncoderConfig(**kw), W)) == "invalidInput", kw
    assert case(lambda: m.embed(np.zeros((1, 0), np.float32))) == "invalidInput"            # empty
    assert case(lambda: m.embed(np.zeros((2, 512), np.float32))) == "invalidInput"          # too few samples for the mel
    assert case(lambda: m.embed(np.zeros((1, 767), np.float32))) == "invalidInput"          # T = 3 <= the widest pad (dilation 3)
    assert m.embed(ser.synth_clip(1, 768)).shape == (1, cfg.enc_dim)                        # T = 4
    assert case(lambda: shipped[2].embed(np.zeros((1, 1023), np.float32))) == "invalidInput"  # shipped: T = 4 <= 4 (dilation 4)
    assert case(lambda: m.embed_mel(np.zeros((1, 3, 128), np.float32))) == "invalidInput"   # T = 3 <= 3 (dilation 3)
    assert case(lambda: m.embed_mel(np.zeros((1, 8, 80), np.float32))) == "invalidInput"
    partial = {k: v for k, v in W.items() if k != "blocks.2.se_block.conv2.bias"}
    assert case(lambda: b2a.Qwen3TTSSpeakerEncoder(cfg, partial)) == "modelNotInitialized"
    wrong = dict(W, **{"asp.conv.weight": W["asp.conv.weight"][:-1]})
    assert case(lambda: b2a.Qwen3TTSSpeakerEncoder(cfg, wrong)) == "modelNotInitialized"
    assert case(lambda: b2a.Qwen3TTSSpeakerEncoder(cfg, {})) == "modelNotInitialized"


# ------------------------------------------------------------------ loading
def write_dir(path, cfg, W, model_type="base", with_speaker=True):
    from safetensors.numpy import save_file
    path.mkdir(exist_ok=True)
    sec = {k: v for k, v in cfg.__dict__.items() if k != "mel_dim"}
    (path / "config.json").write_text(json.dumps({"tts_model_type": model_type, "speaker_encoder_config": sec}))
    ck = {"talker.model.norm.weight": np.ones(4, np.float32)}
    if with_speaker:
        ck.update({"speaker_encoder." + k: np.ascontiguousarray(v) for k, v in W.items()})
    save_file(ck, str(path / "model.safetensors"))


def test_directory_loading(b2a, small, tmp_path):
    from mlx_audio_swift_b200 import _ffi
    cfg, W, m = small
    write_dir(tmp_path / "base", cfg, W)
    d = b2a.Qwen3TTSSpeakerEncoder.from_model_directory(tmp_path / "base")
    assert d.config == cfg
    x = ser.synth_clip(2, 20000, seed=6)
    assert np.array_equal(d.embed(x), m.embed(x))
    for name, kw in (("custom", dict(model_type="custom_voice")), ("nospk", dict(with_speaker=False))):
        write_dir(tmp_path / name, cfg, W, **kw)
        with pytest.raises(_ffi.AudioGenerationError) as e:
            b2a.Qwen3TTSSpeakerEncoder.from_model_directory(tmp_path / name)
        assert e.value.case == "modelNotInitialized", name


# ------------------------------------------------------------------ the voice-cloning prompt from reference audio
def test_prepare_reference_conditioning(b2a):
    from mlx_audio_swift_b200 import qwen3_tts_codec as q
    tcfg = small_cfg()
    talker = device_model(b2a, tcfg, bf16_weights(tcfg, 5), max_batch=2, max_context=160)
    talker.config.tts_model_type = "base"
    _, _, spk = model(b2a, seed=3, **dict(SMALL, enc_dim=tcfg.hidden_size))
    ecfg = q.Qwen3TTSTokenizerEncoderConfig(hidden_size=64, num_filters=8, num_attention_heads=2, num_key_value_heads=2, intermediate_size=128,
                                            num_hidden_layers=2, codebook_size=64, codebook_dim=16, num_quantizers=8,
                                            valid_num_quantizers=tcfg.num_code_groups)
    enc = q.Qwen3TTSSpeechTokenizerEncoder(ecfg, weights=q.random_init_encoder_weights(ecfg, seed=7, layer_scale=0.3))
    dcfg = q.Qwen3TTSTokenizerDecoderConfig(codebook_size=2048, codebook_dim=32, latent_dim=64, decoder_dim=128, hidden_size=64, intermediate_size=128,
                                            num_attention_heads=2, num_key_value_heads=2, num_hidden_layers=1, num_quantizers=tcfg.num_code_groups,
                                            upsample_rates=[8, 5, 4, 3], upsampling_ratios=[2, 2])
    tok = q.Qwen3TTSSpeechTokenizer(dcfg, weights=q.random_init_weights(dcfg), encoder=enc)
    audio = ser.synth_clip(1, 24000, seed=12)[0]
    with pytest.raises(b2a.AudioGenerationError) as e:                   # a Base talker without a speaker encoder
        b2a.Qwen3TTSModel(talker, tok).prepare_reference_conditioning(audio, REF_CHAT, TARGET_CHAT, **TTS)
    assert "speaker" in e.value.message
    model_ = b2a.Qwen3TTSModel(talker, tok, speaker_encoder=spk)
    inp, trail, pad, rc = model_.prepare_reference_conditioning(audio, REF_CHAT, TARGET_CHAT, **TTS, language_id=2160)
    x = spk(audio)
    codes = tok.encode(audio)
    assert np.array_equal(rc, codes[0]) and rc.shape == (tcfg.num_code_groups, enc.encoded_length(audio.shape[0]))
    want = talker.prepare_icl_generation_inputs(codes, REF_CHAT, TARGET_CHAT, **TTS, language_id=2160, speaker_embedding=x)
    assert np.array_equal(inp, want[0]) and np.array_equal(trail, want[1]) and np.array_equal(pad, want[2])
    assert np.array_equal(inp[3 + 4], x + pad)            # role (3 rows), think / think_bos / language / think_eos, then the x-vector
    P = b2a.Qwen3GenerateParameters(max_tokens=6, temperature=0.0, mask_eos=True)
    out = model_.generate(inp, trail, pad, P, ref_codes=rc)
    assert out.ndim == 1 and out.shape[0] > 0 and np.isfinite(out).all()
