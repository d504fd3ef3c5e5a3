"""Qwen3-TTS speaker-encoder time (b2a_qwen3_speaker_encoder_embed / _embed_dev: the 1024-point log-mel and the ECAPA-TDNN) at the
shipped geometry with random-init weights.  Prints ONE JSON line with an entry per workload.

Workloads: 1 x 10 s (the voice-cloning latency: the x-vector is computed before the first generated frame) and 8 x 30 s (batch
throughput), 24 kHz audio 0.5 sin(2 pi 220 t) + 0.1 N(0, 1) (seeded).  Both entry points are timed with CUDA events recorded on the
handle's stream after warm-up: `dev` (waveform and embeddings in HBM) and `host` (host waveform in, host embeddings out, copies
included).  The card name and power limit are read in the same run.

flops: 2 x the multiply-adds of the network's convs per frame, counted from shapes as the reference module runs them (the ASP TDNN
over all 3 C inputs, before the library folds its time-constant part into a per-clip bias; the SE and fc matrix-vector products
are per clip and left out).  launches: kernels per call, from the library's launch counter.

    python tools/bench_qwen3_speaker.py [--warmup 2] [--iters 10]"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import mlx_audio_swift_b200 as m  # noqa: E402
from mlx_audio_swift_b200.qwen3_tts import random_init_speaker_encoder_weights  # noqa: E402


def macs_per_frame(cfg) -> int:
    ch, ks, s = cfg.enc_channels, cfg.enc_kernel_sizes, cfg.enc_res2net_scale
    total = ks[0] * cfg.mel_dim * ch[0]
    for i in range(1, len(ch) - 1):
        w = ch[i] // s
        total += ch[i - 1] * ch[i] + (s - 1) * ks[i] * w * w + ch[i] * ch[i]
    total += ks[-1] * ch[-1] * ch[-1] + 3 * ch[-1] * cfg.enc_attention_channels + cfg.enc_attention_channels * ch[-1]
    return total


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    assert m.device_count() > 0, "the speaker-encoder benchmark needs a CUDA device"
    cfg = m.Qwen3SpeakerEncoderConfig()
    enc = m.Qwen3TTSSpeakerEncoder(cfg, random_init_speaker_encoder_weights(cfg, 1234))
    stream = torch.cuda.ExternalStream(enc.stream)

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

    runs = []
    for B, secs in ((1, 10.0), (8, 30.0)):
        n = int(secs * cfg.sample_rate)
        t = np.arange(n) / cfg.sample_rate
        rng = np.random.default_rng(0)
        audio = (0.5 * np.sin(2 * np.pi * 220.0 * t)[None, :] + 0.1 * rng.standard_normal((B, n))).astype(np.float32)
        T = enc.frames(n)
        d_audio = torch.from_numpy(audio).cuda()
        d_out = torch.empty((B, cfg.enc_dim), dtype=torch.float32, device="cuda")
        ms_dev = timed(lambda: enc.embed_dev(d_audio, d_out, stream=enc.stream))
        ms_host = timed(lambda: enc.embed(audio))
        l0 = m.launch_count()
        host = enc.embed(audio)
        launches = m.launch_count() - l0
        same = np.array_equal(host, d_out.cpu().numpy())
        flops = 2 * B * T * macs_per_frame(cfg)
        runs.append({"workload": f"B={B} x {secs:g} s", "frames": T, "dev_ms": round(ms_dev, 3), "host_ms": round(ms_host, 3),
                     "dev_audio_s_per_s": round(B * secs / (ms_dev / 1e3), 1), "macs_per_frame": macs_per_frame(cfg), "flops": flops,
                     "dev_tflops": round(flops / (ms_dev / 1e3) / 1e12, 2), "launches": launches, "host_equals_dev": same})
    print(json.dumps({"workload": "qwen3_tts speaker encoder (shipped geometry, random weights)", "runs": runs, **gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
