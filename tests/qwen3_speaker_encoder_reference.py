"""Float64 restatement of the Qwen3-TTS speaker encoder (Sources/MLXAudioTTS/Models/Qwen3TTS/Qwen3TTSSpeakerEncoder.swift, an
ECAPA-TDNN) and of its front-end in extractSpeakerEmbedding (Qwen3TTS.swift:839-881: computeMelSpectrogram with n_fft 1024,
hop 256, 128 mels).  Channels-first [B, C, T] as the Swift module runs; weights are the module's keys in torch layout [out, in, k]
(random_init_speaker_encoder_weights).  Pinned against transformers' ECAPA_TimeDelayNet in test_oracle_qwen3_tts_speaker.py.

The Swift reflectPad1D clamps its pad to T - 1; every conv here has T > pad (the library rejects shorter inputs), where the clamp
is inactive and the padding is plain reflection."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import dsp

EPS = 1e-12


def log_mel(audio, sample_rate: int = 24000) -> np.ndarray:
    """computeMelSpectrogram(audio, sampleRate, nFft: 1024, hopLength: 256, nMels: 128) -> [T, 128] float64 (the power, filterbank
    and log run in float64 on the float32 window and filterbank the device uses)."""
    return np.asarray(dsp.compute_mel_spectrogram(np.asarray(audio, np.float32), sample_rate, 1024, 256, 128), dtype=np.float64)


def frames(n: int) -> int:
    return 1 + n // 256


def _w(W, k):
    return torch.as_tensor(np.asarray(W[k], dtype=np.float64))


def _reflect(x, pad):
    """reflectPad1D (:6-16) on [B, C, T]: clamp the pad to T - 1."""
    T = x.shape[-1]
    p = min(pad, max(T - 1, 0))
    if pad <= 0 or T <= 1 or p <= 0:
        return x
    left = x[..., 1:p + 1].flip(-1)
    right = x[..., T - 1 - p:T - 1].flip(-1)
    return torch.cat([left, x, right], dim=-1)


def _tdnn(W, p, x, k, d):
    """TimeDelayNetBlock: reflect pad (k - 1) d / 2, conv, ReLU."""
    x = _reflect(x, (k - 1) * d // 2)
    return torch.relu(F.conv1d(x, _w(W, p + ".conv.weight"), _w(W, p + ".conv.bias"), dilation=d))


def _conv1(W, p, x):
    return F.conv1d(x, _w(W, p + ".weight"), _w(W, p + ".bias"))


def forward(cfg, W, mel) -> np.ndarray:
    """Qwen3TTSSpeakerEncoder.callAsFunction (:299-322): mel [B, T, mel_dim] -> [B, enc_dim] float64."""
    x = torch.as_tensor(np.asarray(mel, dtype=np.float64)).transpose(1, 2)
    ch, ks, ds, s = cfg.enc_channels, cfg.enc_kernel_sizes, cfg.enc_dilations, cfg.enc_res2net_scale
    x = _tdnn(W, "blocks.0", x, ks[0], ds[0])
    hidden = [x]
    for i in range(1, len(ch) - 1):
        p = f"blocks.{i}."
        res = x
        h = _tdnn(W, p + "tdnn1", x, 1, 1)
        chunks = torch.chunk(h, s, dim=1)
        outs, part = [], None
        for j in range(s):                                       # Res2NetBlock (:73-95)
            if j == 0:
                part = chunks[0]
            elif j == 1:
                part = _tdnn(W, p + f"res2net_block.blocks.{j - 1}", chunks[1], ks[i], ds[i])
            else:
                part = _tdnn(W, p + f"res2net_block.blocks.{j - 1}", chunks[j] + part, ks[i], ds[i])
            outs.append(part)
        h = _tdnn(W, p + "tdnn2", torch.cat(outs, dim=1), 1, 1)
        se = h.mean(dim=2, keepdim=True)                         # SqueezeExcitationBlock (:121-128)
        se = torch.sigmoid(_conv1(W, p + "se_block.conv2", torch.relu(_conv1(W, p + "se_block.conv1", se))))
        x = h * se + res
        hidden.append(x)
    x = _tdnn(W, "mfa", torch.cat(hidden[1:], dim=1), ks[-1], ds[-1])
    T = x.shape[-1]                                              # AttentiveStatisticsPooling (:209-232)
    mean = x.mean(dim=2, keepdim=True)
    std = torch.sqrt(((x - mean) ** 2).mean(dim=2, keepdim=True) + EPS)
    att = torch.cat([x, mean.expand(-1, -1, T), std.expand(-1, -1, T)], dim=1)
    att = _conv1(W, "asp.conv", torch.tanh(_tdnn(W, "asp.tdnn", att, 1, 1)))
    att = torch.softmax(att, dim=2)
    m = (att * x).sum(dim=2, keepdim=True)
    sd = torch.sqrt(torch.clamp((att * (x - m) ** 2).sum(dim=2, keepdim=True), min=EPS))
    pooled = torch.cat([m, sd], dim=1)
    return _conv1(W, "fc", pooled)[..., 0].numpy()


def embed(cfg, W, audio) -> np.ndarray:
    """audio [B, n] -> [B, enc_dim]: the float64 mel of each row, then the network."""
    a = np.atleast_2d(np.asarray(audio, np.float32))
    return forward(cfg, W, np.stack([log_mel(r, cfg.sample_rate) for r in a]))


def sanitize(weights: dict) -> dict:
    """Qwen3TTSSpeakerEncoder.sanitize (:324-354): keys after the first "speaker_encoder" component (key.split(".") drops empty
    pieces); a 3-D ".weight" that fails checkArrayShapeQwen3 transposed (0, 2, 1)."""
    from mlx_audio_swift_b200.qwen3_tts import check_array_shape
    out = {}
    for k, v in weights.items():
        parts = [p for p in k.split(".") if p]
        if "speaker_encoder" not in parts:
            continue
        rest = parts[parts.index("speaker_encoder") + 1:]
        if not rest:
            continue
        key = ".".join(rest)
        v = np.asarray(v)
        if key.endswith(".weight") and v.ndim == 3 and not check_array_shape(v.shape):
            v = v.transpose(0, 2, 1)
        out[key] = v
    return out


def synth_clip(B: int, n: int, seed: int = 0, sr: int = 24000) -> np.ndarray:
    """[B, n] float32: 0.5 sin(2 pi f t) + 0.1 N(0, 1) with a different pitch per row."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    rows = [0.5 * np.sin(2 * np.pi * (150.0 + 70.0 * b) * t) + 0.1 * rng.standard_normal(n) for b in range(B)]
    return np.clip(np.stack(rows), -1.0, 1.0).astype(np.float32)
