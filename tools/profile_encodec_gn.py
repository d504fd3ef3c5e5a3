"""Share of device time taken by the time_group_norm kernels (gn_stats_kernel, gn_apply_kernel) in one 48 kHz encode and one 48 kHz
decode of 8 clips x 30.7 s (31 chunks) at 24 kbps, from a torch.profiler trace (CUDA activities) in a run of its own, plus the bytes
those kernels move, counted from shapes: statistics read every conv output once, the apply reads it (two outputs in a resnet, the
trimmed rows of a transposed conv) and writes the result.  Prints ONE JSON line.

    python tools/profile_encodec_gn.py [--batch 8]"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import mlx_audio_swift_b200 as m  # noqa: E402
from bench_encodec_encode import config_48khz  # noqa: E402


def gn_bytes(cfg, rows: int, chunk: int, frames: int) -> dict:
    """fp32 bytes read + written by gn_stats_kernel / gn_apply_kernel over `rows` chunk rows (decoder from `frames` code frames,
    encoder from `chunk` samples)."""
    F = cfg.num_filters

    def normed(E):                       # stats read E, apply read E + write E
        return 4 * E, 8 * E

    def resnet(L, dim):
        hid = dim // cfg.compress
        s1, a1 = normed(L * hid)
        return s1 + 4 * L * dim * (2 if cfg.use_conv_shortcut else 1), a1 + 12 * L * dim      # apply: two addends read, one write

    dec_s = dec_a = 0
    c = F * 2 ** len(cfg.upsampling_ratios)
    s, a = normed(frames * c); dec_s += s; dec_a += a
    L = frames
    for r in cfg.upsampling_ratios:
        co = c // 2
        dec_s += 4 * (L + 1) * r * co; dec_a += 8 * L * r * co              # untrimmed statistics, trimmed apply
        L *= r
        s, a = resnet(L, co); dec_s += s; dec_a += a
        c = co
    s, a = normed(L * cfg.audio_channels); dec_s += s; dec_a += a
    enc_s = enc_a = 0
    L, c = chunk, F
    s, a = normed(L * F); enc_s += s; enc_a += a
    for r in reversed(cfg.upsampling_ratios):
        s, a = resnet(L, c); enc_s += s; enc_a += a
        L = -(-L // r)
        s, a = normed(L * 2 * c); enc_s += s; enc_a += a
        c *= 2
    s, a = normed(L * cfg.hidden_size); enc_s += s; enc_a += a
    return {"decode_stats": rows * dec_s, "decode_apply": rows * dec_a, "encode_stats": rows * enc_s, "encode_apply": rows * enc_a}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    a = ap.parse_args()
    assert m.device_count() > 0, "the profile needs a CUDA device"
    from torch.profiler import ProfilerActivity, profile
    cfg = config_48khz()
    codec = m.Encodec(cfg, weights=m.Encodec.random_init_weights(cfg, 1234, n_codebooks=16, encoder=True))
    n = 30 * codec.chunk_stride + codec.chunk_length
    rng = np.random.default_rng(0)
    t = np.arange(n) / cfg.sampling_rate
    audio = (0.5 * np.sin(2 * np.pi * 220.0 * t)[None, :, None] + 0.1 * rng.standard_normal((a.batch, n, 2))).astype(np.float32)
    nc, T = codec.encoded_shape(n)
    d_audio = torch.from_numpy(audio).cuda()
    d_codes = torch.empty((nc, a.batch, 16, T), dtype=torch.int32, device="cuda")
    d_scales = torch.empty((nc, a.batch), dtype=torch.float32, device="cuda")
    wave = torch.empty((a.batch, n, 2), device="cuda")

    def run(which):
        if which == "encode":
            codec.encode_dev(d_audio, d_codes, d_scales, stream=codec.stream, bandwidth=24.0)
        else:
            codec.decode_dev(d_codes, wave, d_scales, stream=codec.stream)
        torch.cuda.synchronize()

    out = {"workload": f"encodec_48khz, B={a.batch} x {n / 48000:.1f} s ({nc} chunks), 24 kbps"}
    for which in ("encode", "decode"):
        run(which); run(which)                                    # warm-up: every shape of the profiled call
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(which)
        total = gn_stats = gn_apply = 0.0
        for e in prof.key_averages():
            us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            if e.key.startswith("Memcpy") or e.key.startswith("Memset"):
                continue
            total += us
            if "gn_stats_kernel" in e.key:
                gn_stats += us
            elif "gn_apply_kernel" in e.key:
                gn_apply += us
        out[which] = {"kernel_ms": round(total / 1e3, 3), "gn_stats_ms": round(gn_stats / 1e3, 3), "gn_apply_ms": round(gn_apply / 1e3, 3),
                      "gn_share": round((gn_stats + gn_apply) / max(total, 1e-9), 4)}
    b = gn_bytes(cfg, nc * a.batch, codec.chunk_length, T)
    for which in ("encode", "decode"):
        moved = b[f"{which}_stats"] + b[f"{which}_apply"]
        ms = out[which]["gn_stats_ms"] + out[which]["gn_apply_ms"]
        out[which].update({"gn_bytes": moved, "gn_GBps": round(moved / (ms * 1e-3) / 1e9, 1) if ms else None})
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip().splitlines()[0]
    out["gpu"] = gpu
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
