"""Qwen3-TTS talker + code predictor frame loop at the 0.6B or the 1.7B geometry (random-init bf16 weights, EOS masked so every run
does the same work).  Prints ONE JSON line per batch size: host time of the frame loop per frame after warm-up (the median of --iters
runs of --frames frames; b2a_qwen3_talker_generate's generate_time, which ends in a device synchronise), times real time (a frame is
80 ms of audio per row), and the weight bytes one frame streams, counted from shapes, with their share of the H100 SXM data-sheet
HBM3 bandwidth (3.35 TB/s).  The card's name and power limit are read in the same call.

Weight bytes per frame: the talker's layers and codec head once, the predictor's layers 16 times (position 0 + 15 code positions),
its 15 lm heads once each, and at 1.7B the small_to_mtp_projection once (the projected embedding rows are gathers).

    python tools/bench_qwen3_talker.py --geometry 1.7b --batch 1,4,8,16,32 [--frames 512] [--warmup 1] [--iters 3]"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import mlx_audio_swift_b200 as m  # noqa: E402
from tools.bench_snac_44khz import gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
FRAME_S = 0.08
PROMPT_ROWS, TRAILING_ROWS = 10, 24


def geometry(name: str):
    """0.6B: Qwen3TTSConfig.swift's defaults.  1.7B: talker 2048 / MLP 6144 / 28 layers / 16 q : 8 kv heads, text_hidden_size 2048,
    the same predictor (1024 / 3072 / 5 layers) -- the published config.json as recalled, not checked against a real one."""
    if name == "0.6b":
        return m.Qwen3TalkerConfig()
    if name == "1.7b":
        return m.Qwen3TalkerConfig(hidden_size=2048, intermediate_size=6144, num_hidden_layers=28, num_attention_heads=16,
                                   num_key_value_heads=8, text_hidden_size=2048)
    raise SystemExit(f"unknown geometry {name!r}")


def stack_bytes(hidden, inter, layers, nq, nkv, hd=128):
    return 2 * layers * (hidden * (nq + 2 * nkv) * hd + nq * hd * hidden + 3 * hidden * inter)


def weight_bytes_per_frame(c) -> int:
    cp = c.code_predictor
    talker = stack_bytes(c.hidden_size, c.intermediate_size, c.num_hidden_layers, c.num_attention_heads, c.num_key_value_heads)
    talker += 2 * c.vocab_size * c.hidden_size
    pred = stack_bytes(cp.hidden_size, cp.intermediate_size, cp.num_hidden_layers, cp.num_attention_heads, cp.num_key_value_heads)
    heads = (c.num_code_groups - 1) * 2 * cp.vocab_size * cp.hidden_size
    proj = 2 * cp.hidden_size * c.hidden_size if cp.hidden_size != c.hidden_size else 0
    return talker + c.num_code_groups * pred + heads + proj


def run(cfg, name, B, frames, warmup, iters):
    talker = m.Qwen3TTSTalker.random_init(cfg, max_batch=B, max_context=PROMPT_ROWS + frames + 32, std=0.02, seed=77)
    rng = np.random.default_rng(9)
    H = cfg.hidden_size
    embeds = (0.05 * rng.standard_normal((B, PROMPT_ROWS, H))).astype(np.float32)
    trailing = list((0.05 * rng.standard_normal((B, TRAILING_ROWS, H))).astype(np.float32))
    pad = (0.05 * rng.standard_normal(H)).astype(np.float32)
    P = m.Qwen3GenerateParameters(max_tokens=frames, temperature=0.9, top_k=50, top_p=1.0, repetition_penalty=1.05, seed=1, mask_eos=True)
    times = []
    for i in range(warmup + iters):
        codes, info = talker.generate_codes(embeds, trailing, pad, P)
        assert all(len(c) == frames for c in codes)
        if i >= warmup:
            times.append(info.generate_time)
    del talker
    ms = float(np.median(times)) / frames * 1e3
    wb = weight_bytes_per_frame(cfg)
    return {"geometry": name, "batch": B, "frames": frames, "iters": iters, "ms_per_frame": ms,
            "ms_per_frame_runs": [t / frames * 1e3 for t in times], "x_realtime_per_row": FRAME_S * 1e3 / ms,
            "x_realtime_total": B * FRAME_S * 1e3 / ms, "weight_bytes_per_frame": wb,
            "hbm_floor_ms_per_frame": wb / HBM_BYTES_PER_S * 1e3, "hbm_fraction": wb / HBM_BYTES_PER_S / (ms * 1e-3),
            "hbm_peak": "3.35 TB/s (H100 SXM data sheet)",
            "talker": {"hidden": cfg.hidden_size, "layers": cfg.num_hidden_layers, "predictor_hidden": cfg.code_predictor.hidden_size}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--geometry", default="1.7b", choices=["0.6b", "1.7b"])
    ap.add_argument("--batch", default="1,4,8", help="comma-separated batch sizes (<= 32)")
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--iters", type=int, default=3)
    a = ap.parse_args()
    assert m.device_count() > 0, "the benchmark needs a CUDA device"
    cfg = geometry(a.geometry)
    for B in (int(b) for b in a.batch.split(",")):
        r = run(cfg, a.geometry, B, a.frames, a.warmup, a.iters)
        r.update(gpu_info())
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
