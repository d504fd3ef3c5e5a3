"""SNAC encode throughput (b2a_snac_encode / b2a_snac_encode_dev) on the 24 kHz model with random-init weights.  Prints ONE JSON line.

Workload: B clips of S seconds at 24 kHz, 0.5 sin(2 pi 220 t) + 0.1 N(0, 1) (seeded).  Both entry points are timed with CUDA events
recorded on the handle's stream after warm-up: `dev` (waveform and codes in HBM) and `host` (host waveform in, host codes out, copies
included).  Rates are audio-seconds per second of device time.

flops: 2 x the multiply-adds of the model at its real widths (stem, residual units, strided convs, final depthwise conv, in_proj,
code search and the quantizer's out_proj lookups), counted from shapes.  tc_flops: what the tensor cores execute -- the 1x1 and strided
convs at the padded widths (48 -> 64, 96 -> 128 channels), three bf16 products per fp32 product (Wh Xh, Wh Xl, Wl Xh).
bytes: the activation traffic of this implementation's kernel sequence at the padded widths: every fp32 tensor read and written by
each kernel, the bf16 hi/lo operands (4 B per value) and the strided convs' 2-frame operands; weights, halos and L2 reuse excluded.

    python tools/bench_snac_encode.py [--batch 8] [--seconds 30] [--warmup 2] [--iters 5]"""
import argparse
import json
import math
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import mlx_audio_swift_b200 as m  # noqa: E402

ENC_DIM, RATES, LATENT, VQ, CODEBOOK, CB_DIM = 48, (2, 4, 8, 8), 768, (4, 2, 1), 4096, 8


def padded(c):
    return 64 if c <= 64 else 128 if c <= 128 else -(-c // 64) * 64


def work(n_samples: int):
    """(flops, tc_flops, bytes) for ONE clip of n_samples (already padded to a multiple of 2048)."""
    macs = 7 * ENC_DIM * n_samples
    tc_macs = 0
    byts = 4 * n_samples + 4 * padded(ENC_DIM) * n_samples                # stem: waveform in, fp32 out
    t, c = n_samples, ENC_DIM
    for s in RATES:
        cp, cpo = padded(c), padded(2 * c)
        macs += 3 * (7 * c + c * c) * t + (2 * c) * (2 * s * c) * (t // s)
        tc_macs += 3 * cp * cp * t + cpo * 2 * s * cp * (t // s + 1)
        if cp in (64, 128):
            byts += 3 * 8 * cp * t                                        # fused unit: fp32 in + out
        else:
            byts += 3 * 4 * 5 * cp * t                                    # dw7 (x in, hi/lo out) + GEMM (hi/lo in, x read-modify-write)
        byts += 2 * 8 * cp * t                                            # 2-frame hi/lo operand written (each value twice) and read back
        byts += 4 * cpo * (t // s)                                        # strided conv fp32 out
        t, c = t // s, 2 * c
    macs += 7 * LATENT * t
    byts += 8 * LATENT * t                                                # final depthwise conv: NLC in, NCT out
    for s in VQ:
        macs += (LATENT * CB_DIM + CODEBOOK * CB_DIM) * (t // s) + LATENT * CB_DIM * t
    return 2 * macs, 2 * 3 * tc_macs, byts


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    assert m.device_count() > 0, "the encode benchmark needs a CUDA device"
    codec = m.SNAC(weights=m.SNAC.random_init_weights(1234, encoder=True))
    n = int(a.seconds * 24000)
    t = np.arange(n) / 24000.0
    rng = np.random.default_rng(0)
    audio = (0.5 * np.sin(2 * np.pi * 220.0 * t)[None, None] + 0.1 * rng.standard_normal((a.batch, 1, n))).astype(np.float32)
    T = codec.encoded_length(n)
    d_audio = torch.from_numpy(audio).cuda()
    d_codes = [torch.empty((a.batch, T // s), dtype=torch.int32, device="cuda") for s in VQ]
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

    ms_dev = timed(lambda: codec.encode_dev(d_audio, d_codes, stream=codec.stream))
    ms_host = timed(lambda: codec.encode(audio))
    host_codes = codec.encode(audio)
    same = all(np.array_equal(h, d.cpu().numpy()) for h, d in zip(host_codes, d_codes))
    flops, tc_flops, byts = (a.batch * x for x in work(T * 512))
    audio_s = a.batch * a.seconds
    line = {"workload": f"snac_24khz encode, B={a.batch} x {a.seconds:g} s", "t_latent": T,
            "dev_ms": round(ms_dev, 3), "host_ms": round(ms_host, 3),
            "dev_audio_s_per_s": round(audio_s / (ms_dev / 1e3), 1), "host_audio_s_per_s": round(audio_s / (ms_host / 1e3), 1),
            "flops": flops, "tc_flops": tc_flops, "bytes": byts,
            "dev_tflops": round(flops / (ms_dev / 1e3) / 1e12, 2), "dev_tc_tflops": round(tc_flops / (ms_dev / 1e3) / 1e12, 2),
            "dev_gb_per_s": round(byts / (ms_dev / 1e3) / 1e9, 1), "host_equals_dev": same, **gpu_info()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
