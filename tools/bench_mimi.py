"""Mimi encode / decode time (b2a_mimi_*) at mimi_202407(32) with random-init weights.  Prints ONE JSON line.

Workloads: 8 x 30 s encode and one-shot decode (batch throughput; codes and waveform in HBM, timed with CUDA events on the
handle's stream after warm-up), and the streaming decoder one code frame per call at batch 1 and 8 -- the Marvis shape
(MimiStreamingDecoder.decodeFrames) -- as the mean wall time of a synchronised decode_step_dev over 100 frames, with the kernel
launches of one step.  The card name and power limit are read in the same run.

flops: 2 x the multiply-adds counted from shapes: the decoder's output projections, upsample, transformer (q|k|v, attention over
the causal half, out projection, MLP) and SEANet decoder; the encoder's as tools/bench_qwen3_encode.py counts them.

    python tools/bench_mimi.py [--warmup 2] [--iters 5]"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]
import mlx_audio_swift_b200 as m  # noqa: E402
from oracle import mimi as om  # noqa: E402
from tools.bench_qwen3_encode import encoder_flops, gpu_info  # noqa: E402


def decoder_flops(cfg, T: int) -> dict:
    """Multiply-adds x 2 of decoding T code frames, by stage."""
    D, s = cfg.dimension, cfg.downsample_stride
    Tl = T * s
    quant = T * 2 * cfg.codebook_dim * D + Tl * 2 * D
    tr = cfg.num_layers * (Tl * (4 * D * D + 2 * D * cfg.dim_feedforward) + Tl * (Tl + 1) // 2 * 2 * D)
    L = len(cfg.ratios)
    c = cfg.n_filters << L
    sea = Tl * cfg.kernel_size * D * c
    n = Tl
    for r in cfg.ratios:
        sea += n * (2 * r) * c * (c // 2)            # transposed conv: every input frame meets every tap
        n *= r
        c //= 2
        hid = c // cfg.compress
        sea += n * (cfg.residual_kernel_size * c * hid + hid * c)
    sea += n * cfg.last_kernel_size * c
    return {"quantizer_upsample": 2 * quant, "transformer": 2 * tr, "seanet": 2 * sea}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    assert m.device_count() > 0, "the Mimi benchmark needs a CUDA device"
    cfg = om.mimi_202407(32)
    codec = m.Mimi(om.init_weights(cfg, 1234), 32, max_batch=8, max_cache_frames=400)
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

    out = {"workload": "mimi_202407(32), random weights"}
    B, secs = 8, 30.0
    n = int(secs * cfg.sample_rate)
    t = np.arange(n) / cfg.sample_rate
    rng = np.random.default_rng(0)
    audio = (0.5 * np.sin(2 * np.pi * 220.0 * t)[None, None, :] + 0.1 * rng.standard_normal((B, 1, n))).astype(np.float32)
    T = codec.encoded_length(n)
    d_audio = torch.from_numpy(audio).cuda()
    d_codes = torch.empty((B, 32, T), dtype=torch.int32, device="cuda")
    d_wave = torch.empty((B, 1, T * 1920), dtype=torch.float32, device="cuda")
    ms_enc = timed(lambda: codec.encode_dev(d_audio, d_codes, stream=codec.stream))
    ms_dec = timed(lambda: codec.decode_dev(d_codes, d_wave, stream=codec.stream))
    efl = {k: B * v for k, v in encoder_flops(
        type("E", (), dict(num_filters=cfg.n_filters, hidden_size=cfg.dimension, intermediate_size=cfg.dim_feedforward,
                           kernel_size=cfg.kernel_size, upsampling_ratios=list(cfg.ratios), compress=cfg.compress,
                           residual_kernel_size=cfg.residual_kernel_size, last_kernel_size=cfg.last_kernel_size,
                           num_hidden_layers=cfg.num_layers, downsample_stride=cfg.downsample_stride, codebook_dim=cfg.codebook_dim,
                           num_code_groups=32, codebook_size=cfg.codebook_size)), n).items()}
    dfl = {k: B * v for k, v in decoder_flops(cfg, T).items()}
    out["encode_8x30s"] = {"frames": T, "ms": round(ms_enc, 3), "audio_s_per_s": round(B * secs / (ms_enc / 1e3), 1), "flops": efl,
                           "tflops": round(sum(efl.values()) / (ms_enc / 1e3) / 1e12, 2)}
    out["decode_8x30s"] = {"frames": T, "ms": round(ms_dec, 3), "audio_s_per_s": round(B * T * 0.08 / (ms_dec / 1e3), 1), "flops": dfl,
                           "gflop_per_audio_s": round(sum(dfl.values()) / (B * T * 0.08) / 1e9, 2),
                           "tflops": round(sum(dfl.values()) / (ms_dec / 1e3) / 1e12, 2)}
    frames = 100
    for Bs in (1, 8):
        codes = torch.from_numpy(np.random.default_rng(Bs).integers(0, 2048, (Bs, 32, frames)).astype(np.int32)).cuda()
        steps = [codes[:, :, i:i + 1].contiguous() for i in range(frames)]
        w1 = torch.empty((Bs, 1, 1920), dtype=torch.float32, device="cuda")
        codec.reset()
        for i in range(5):
            codec.decode_step_dev(steps[i], w1, stream=codec.stream)
        codec.reset()
        torch.cuda.synchronize()
        l0 = m.launch_count()
        codec.decode_step_dev(steps[0], w1, stream=codec.stream)
        launches = m.launch_count() - l0
        torch.cuda.synchronize()
        dt = []
        for i in range(1, frames):
            t0 = time.perf_counter()
            codec.decode_step_dev(steps[i], w1, stream=codec.stream)
            stream.synchronize()
            dt.append(time.perf_counter() - t0)
        dt = np.array(dt) * 1e3
        out[f"decode_frames_b{Bs}"] = {"ms_per_frame_mean": round(float(dt.mean()), 3), "ms_per_frame_p50": round(float(np.median(dt)), 3),
                                       "ms_per_frame_max": round(float(dt.max()), 3), "launches_per_step": launches,
                                       "x_real_time": round(80.0 / float(dt.mean()), 1)}
    print(json.dumps({**out, **gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
