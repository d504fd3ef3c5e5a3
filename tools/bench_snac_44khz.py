"""SNAC 44.1 kHz (published geometry, random-init weights with LocalMHA) encode and decode of B clips of S seconds.  Prints ONE JSON
line: device time per call (CUDA events on the handle's stream after warm-up), audio-seconds per second, the decode's model work
counted from shapes, and with --profile (a run of its own, torch.profiler) the share of kernel time spent in LocalMHA's kernels.

decode_flops: 2 x the multiply-adds of the decoder at its real widths -- depthwise + 1x1 input convs, LocalMHA (to_qkv, q k^T, p v,
to_out), per DecoderBlock the transposed conv (k = 2s), NoiseBlock linear and three residual units (depthwise k7 + 1x1), final conv.

    python tools/bench_snac_44khz.py [--batch 8] [--seconds 30] [--warmup 1] [--iters 3] [--profile]"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import mlx_audio_swift_b200 as m  # noqa: E402

ENC_DIM, ENC_RATES, LATENT, DEC_DIM, DEC_RATES, VQ, WINDOW, SR = 64, (2, 3, 8, 8), 1024, 1536, (8, 8, 3, 2), (8, 4, 2, 1), 32, 44100
ATTN_KERNELS = ("dw_layernorm_kernel", "local_attn_kernel")


def decode_flops(t_latent: int) -> float:
    t, c = t_latent, DEC_DIM
    macs = 7 * LATENT * t + LATENT * c * t
    macs += 4 * c * c * t + 2 * WINDOW * c * t                          # to_qkv + to_out, q k^T + p v
    for s in DEC_RATES:
        co = c // 2
        macs += c * 2 * s * co * t                                       # transposed conv, k = 2s, over the input frames
        t = t * s - s % 2
        macs += co * co * t + 3 * (7 * co + co * co) * t
        c = co
    macs += 7 * c * t
    return 2.0 * macs


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="torch.profiler run: LocalMHA's share of kernel time (no timings)")
    a = ap.parse_args()
    assert m.device_count() > 0, "the benchmark needs a CUDA device"
    W = m.SNAC.random_init_weights(1234, latent=LATENT, decoder_dim=DEC_DIM, decoder_rates=DEC_RATES, vq_strides=VQ, encoder=True,
                                   encoder_dim=ENC_DIM, encoder_rates=ENC_RATES, attn_window_size=WINDOW)
    codec = m.SNAC(SR, ENC_DIM, ENC_RATES, None, DEC_DIM, DEC_RATES, WINDOW, 4096, 8, VQ, True, True, weights=W)
    n = int(a.seconds * SR)
    t = np.arange(n) / SR
    rng = np.random.default_rng(0)
    audio = (0.5 * np.sin(2 * np.pi * 220.0 * t)[None, None] + 0.1 * rng.standard_normal((a.batch, 1, n))).astype(np.float32)
    T = codec.encoded_length(n)
    d_audio = torch.from_numpy(audio).cuda()
    d_codes = [torch.empty((a.batch, T // s), dtype=torch.int32, device="cuda") for s in VQ]
    d_wave = torch.empty((a.batch, 1, codec.decoded_length(T)), dtype=torch.float32, device="cuda")
    s = torch.cuda.ExternalStream(codec.stream)

    def enc():
        codec.encode_dev(d_audio, d_codes, stream=codec.stream)

    def dec():
        codec.decode_dev(d_codes, d_wave, seed=1, stream=codec.stream)

    for _ in range(a.warmup):
        enc(); dec()
    torch.cuda.synchronize()
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        res = {}
        for name, fn in (("encode", enc), ("decode", dec)):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            tot = attn = gemm = 0.0
            for ev in prof.key_averages():
                dt = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
                tot += dt
                if any(k in ev.key for k in ATTN_KERNELS):
                    attn += dt
            res[name] = {"kernel_us": tot, "attn_core_us": attn, "attn_core_share": attn / tot if tot else 0.0,
                         "top": [(ev.key[:60], (ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total))
                                 for ev in sorted(prof.key_averages(), key=lambda e: -(e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total))[:8]]}
        print(json.dumps({"bench": "snac44_profile", "batch": a.batch, "seconds": a.seconds, **res, **gpu_info()}))
        return
    out = {}
    for name, fn in (("encode", enc), ("decode", dec)):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(s):
            e0.record(s)
            for _ in range(a.iters):
                fn()
            e1.record(s)
        e1.synchronize()
        ms = e0.elapsed_time(e1) / a.iters
        out[name] = {"ms": ms, "audio_s_per_s": a.batch * a.seconds / (ms / 1e3)}
    fl = decode_flops(T) * a.batch
    out["decode"].update({"model_tflop": fl / 1e12, "model_tflop_per_clip": fl / a.batch / 1e12, "achieved_tflops": fl / (out["decode"]["ms"] / 1e3) / 1e12})
    print(json.dumps({"bench": "snac44", "batch": a.batch, "seconds": a.seconds, "t_latent": T, **out, **gpu_info()}))


if __name__ == "__main__":
    main()
