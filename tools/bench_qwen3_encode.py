"""Qwen3-TTS speech-tokenizer encode time (b2a_speech_tokenizer_encoder_encode / _encode_dev) at the shipped geometry with
random-init weights.  Prints ONE JSON line with an entry per workload.

Workloads: 8 x 30 s (batch throughput) and 1 x 10 s (the voice-cloning latency: the reference clip is encoded before the first
generated frame), 24 kHz audio 0.5 sin(2 pi 220 t) + 0.1 N(0, 1) (seeded).  Both entry points are timed with CUDA events recorded on
the handle's stream after warm-up: `dev` (waveform and codes in HBM) and `host` (host waveform in, host codes out, copies included).
The card name and power limit are read in the same run.

flops: 2 x the multiply-adds of the SEANet encoder, the transformer (q|k|v, attention scores and values over the causal half,
out projection, MLP), the downsample and the code search (input projections + frames x groups x codebook_size x codebook_dim),
counted from shapes.

    python tools/bench_qwen3_encode.py [--warmup 2] [--iters 5]"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import mlx_audio_swift_b200 as m  # noqa: E402
from mlx_audio_swift_b200 import qwen3_tts_codec as q  # noqa: E402


def encoder_flops(cfg, n: int) -> dict:
    F, H, I = cfg.num_filters, cfg.hidden_size, cfg.intermediate_size
    seanet = cfg.kernel_size * F * n
    L, c = n, F
    for r in reversed(cfg.upsampling_ratios):
        hid = c // cfg.compress
        seanet += L * (cfg.residual_kernel_size * c * hid + hid * c)
        L = -(-L // r)
        seanet += L * (2 * r * c) * (2 * c)
        c *= 2
    seanet += L * cfg.last_kernel_size * c * H
    tr = cfg.num_hidden_layers * (L * (4 * H * H + 2 * H * I) + L * (L + 1) // 2 * 2 * H)
    T = -(-L // cfg.downsample_stride)
    tail = T * 2 * cfg.downsample_stride * H * H + T * 2 * H * cfg.codebook_dim + T * cfg.num_code_groups * cfg.codebook_size * cfg.codebook_dim
    return {"seanet": 2 * seanet, "transformer": 2 * tr, "downsample_and_search": 2 * tail}


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    assert m.device_count() > 0, "the encode benchmark needs a CUDA device"
    cfg = q.Qwen3TTSTokenizerEncoderConfig()
    enc = q.Qwen3TTSSpeechTokenizerEncoder(cfg, weights=q.random_init_encoder_weights(cfg, 1234))
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
    for B, secs in ((8, 30.0), (1, 10.0)):
        n = int(secs * cfg.sampling_rate)
        t = np.arange(n) / cfg.sampling_rate
        rng = np.random.default_rng(0)
        audio = (0.5 * np.sin(2 * np.pi * 220.0 * t)[None, None, :] + 0.1 * rng.standard_normal((B, 1, n))).astype(np.float32)
        T = enc.encoded_length(n)
        d_audio = torch.from_numpy(audio).cuda()
        d_codes = torch.empty((B, enc.num_code_groups, T), dtype=torch.int32, device="cuda")
        ms_dev = timed(lambda: enc.encode_dev(d_audio, d_codes, stream=enc.stream))
        ms_host = timed(lambda: enc.encode(audio))
        same = np.array_equal(enc.encode(audio), d_codes.cpu().numpy())
        fl = {k: B * v for k, v in encoder_flops(cfg, n).items()}
        total = sum(fl.values())
        runs.append({"workload": f"B={B} x {secs:g} s", "frames": T, "dev_ms": round(ms_dev, 3), "host_ms": round(ms_host, 3),
                     "dev_audio_s_per_s": round(B * secs / (ms_dev / 1e3), 1), "flops": fl, "dev_tflops": round(total / (ms_dev / 1e3) / 1e12, 2),
                     "host_equals_dev": same})
    print(json.dumps({"workload": "qwen3_tts speech-tokenizer encode (shipped geometry, random weights)", "runs": runs, **gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
