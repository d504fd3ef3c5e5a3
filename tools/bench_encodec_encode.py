"""Encodec encode throughput (b2a_encodec_encode / b2a_encodec_encode_dev) on the 24 kHz model (default) or the 48 kHz stereo model
(--model 48khz: time_group_norm, 1 s chunks with 1 % overlap, normalize) with random-init weights.  Prints ONE JSON line with an
entry per bandwidth.

Workload: B clips of S seconds, 0.5 sin(2 pi 220 t) + 0.1 N(0, 1) (seeded), encoded at 1.5 kbps (2 codebooks) and 24 kbps (32
codebooks) at 24 kHz, at 3 kbps (2 codebooks) and 24 kbps (16) at 48 kHz, where S defaults to 30.7 s (31 whole chunks).  Both entry points are timed with CUDA events recorded on the handle's stream after warm-up: `dev` (waveform and codes
in HBM) and `host` (host waveform in, host codes out, copies included).  Rates are audio-seconds per second of device time.

flops: 2 x the multiply-adds of the encoder (stem, resnet blocks, strided convs, LSTM input and recurrent products, last conv) per
chunk plus the code search's dot products (frames x n_q x codebook_size x dim), counted from shapes.

    python tools/bench_encodec_encode.py [--model 24khz|48khz] [--batch 8] [--seconds S] [--warmup 2] [--iters 5]"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import mlx_audio_swift_b200 as m  # noqa: E402


def encoder_macs(cfg, n: int) -> int:
    """Multiply-adds of EncodecEncoder on one clip of n samples (one residual layer per stage)."""
    F = cfg.num_filters
    macs = cfg.kernel_size * cfg.audio_channels * F * n
    L, c = n, F
    for r in reversed(cfg.upsampling_ratios):
        hid = c // cfg.compress
        macs += L * (cfg.residual_kernel_size * c * hid + hid * c + (c * c if cfg.use_conv_shortcut else 0))
        L = -(-L // r)
        macs += L * (2 * r * c) * (2 * c)
        c *= 2
    macs += cfg.num_lstm_layers * L * 8 * c * c              # Wx and Wh, 4 gates each
    macs += L * cfg.last_kernel_size * c * cfg.hidden_size
    return macs


def config_48khz():
    """facebook/encodec_48khz's config.json."""
    return m.EncodecConfig(audio_channels=2, use_causal_conv=False, normalize=True, norm_type="time_group_norm", sampling_rate=48000,
                           chunk_length_s=1.0, overlap=0.01, target_bandwidths=[3.0, 6.0, 12.0, 24.0])


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=["24khz", "48khz"], default="24khz")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--seconds", type=float, default=None, help="default: 30 (24khz), 30.7 (48khz: 31 whole 1 s chunks)")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    assert m.device_count() > 0, "the encode benchmark needs a CUDA device"
    big = a.model == "48khz"
    cfg = config_48khz() if big else m.EncodecConfig()
    codec = m.Encodec(cfg, weights=m.Encodec.random_init_weights(cfg, 1234, n_codebooks=16 if big else 32, encoder=True))
    if a.seconds is None:
        a.seconds = 30.7 if big else 30.0
    n = int(round(a.seconds * cfg.sampling_rate))
    t = np.arange(n) / cfg.sampling_rate
    rng = np.random.default_rng(0)
    ch = cfg.audio_channels
    audio = (0.5 * np.sin(2 * np.pi * 220.0 * t)[None, :, None] + 0.1 * rng.standard_normal((a.batch, n, ch))).astype(np.float32)
    nc, T = codec.encoded_shape(n)
    d_audio = torch.from_numpy(audio).cuda()
    stream = torch.cuda.ExternalStream(codec.stream)

    def timed(fn):
        for _ in range(a.warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(a.iters):
            fn()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / a.iters

    audio_s = a.batch * a.seconds
    runs = []
    chunk = codec.chunk_length if nc > 1 else n
    for bw in ((3.0, 24.0) if big else (1.5, 24.0)):
        nq = codec.num_quantizers_for_bandwidth(bw)
        d_codes = torch.empty((nc, a.batch, nq, T), dtype=torch.int32, device="cuda")
        ms_dev = timed(lambda: codec.encode_dev(d_audio, d_codes, stream=codec.stream, bandwidth=bw))
        ms_host = timed(lambda: codec.encode(audio, bandwidth=bw))
        same = np.array_equal(codec.encode(audio, bandwidth=bw)[0], d_codes.cpu().numpy())
        flops = 2 * a.batch * nc * (encoder_macs(cfg, chunk) + T * nq * cfg.codebook_size * cfg.codebook_dim)
        runs.append({"bandwidth_kbps": bw, "n_q": nq, "dev_ms": round(ms_dev, 3), "host_ms": round(ms_host, 3),
                     "dev_audio_s_per_s": round(audio_s / (ms_dev / 1e3), 1), "host_audio_s_per_s": round(audio_s / (ms_host / 1e3), 1),
                     "flops": flops, "dev_tflops": round(flops / (ms_dev / 1e3) / 1e12, 2), "host_equals_dev": same})
    line = {"workload": f"encodec_{a.model} encode, B={a.batch} x {a.seconds:g} s", "chunks": nc, "frames": T, "runs": runs, **gpu_info()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
