"""Orpheus-3B prompt pass (time to the first token) at prompt lengths on both sides of the SIMT prompt attention's 128-position cap.

Two random-init models with the same weights: the default one (batched prefill: prompts of <= 128 positions with the SIMT prompt
attention, longer ones with the wgmma one, csrc/prompt_attn_tc.cuh) and one built under B2A_PREFILL=step (the decode step replayed per
prompt position).  For each batch and prompt length both run generate_batch with max_tokens = 1 alternately; the time is the library's
prefill_time (host clock from before the first prompt kernel to a stream synchronise after the first token is sampled), median over
--reps calls after one warm-up call per shape.

    python tools/bench_prefill.py [--batch 1 8] [--lengths 64 128 129 256 512 913 1536] [--reps 5] [--out FILE.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import mlx_audio_swift_b200 as m  # noqa: E402
from bench import ORPHEUS  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--lengths", type=int, nargs="+", default=[64, 128, 129, 256, 512, 913, 1536])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert m.device_count() > 0, "bench_prefill needs a CUDA device"
    ctx, mb = max(a.lengths) + 8, max(a.batch)
    fast = m.LlamaTTSModel.random_init(ORPHEUS, max_batch=mb, max_context=ctx)
    os.environ["B2A_PREFILL"] = "step"
    step = m.LlamaTTSModel.random_init(ORPHEUS, max_batch=mb, max_context=ctx)
    del os.environ["B2A_PREFILL"]
    P = m.GenerateParameters(max_tokens=1, temperature=0.0, top_p=1.0, repetition_penalty=1.0, repetition_context_size=0)
    gpu = card()
    print(f"card: {gpu}")
    rows = []
    for B in a.batch:
        for L in a.lengths:
            ids = np.random.default_rng(L).integers(0, 128000, size=(B, L)).astype(np.int32)
            t = {"batched": [], "step": []}
            for name, model in (("batched", fast), ("step", step)):
                model.generate_batch(ids, P, decode_audio=False)                 # warm-up
            toks = {}
            for _ in range(a.reps):
                for name, model in (("batched", fast), ("step", step)):
                    tk, _, info = model.generate_batch(ids, P, decode_audio=False)
                    t[name].append(info.prefill_time)
                    toks[name] = tk
            r = {"batch": B, "prompt": L, "prefill_ms": 1e3 * statistics.median(t["batched"]),
                 "step_replay_ms": 1e3 * statistics.median(t["step"]), "same_first_token": toks["batched"] == toks["step"]}
            r["speedup"] = r["step_replay_ms"] / r["prefill_ms"]
            rows.append(r)
            print(json.dumps(r), flush=True)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps({"card": gpu, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
