"""Per-kernel timeline of one Orpheus-3B decode step (the 144-launch CUDA graph bench.py times), from torch.profiler.

    python tools/step_timeline.py OUT_DIR [--iters N]

Builds bench.py's model (bench.ORPHEUS, batch 8), and for contexts 64, 320 and 576 runs `tts.time_steps(8, ctx, N)` twice: once with
the profiler off (the CUDA-event ms per step) and once, after that warm-up, under torch.profiler with CUDA activities.  The kernel
records of the profiled run are folded by their position in the step; OUT_DIR/step_timeline.json gets, per position, the kernel
name, the median duration, the median gap from the previous kernel's end to this kernel's start (negative: the two overlap), the
bytes the kernel has to move (weights once, fp32 K/V at that context, the logits; activations of a few hundred KB are left out) and
bytes / duration; and per step the sum of durations, the sum of positive gaps and the event-timed ms.  The card's name, power
limit and maximum SM clock are read with nvidia-smi and written beside the numbers: an absolute time means nothing without them.
Tracing perturbs the step, so compare sum_dur_us + sum_pos_gap_us with event_ms_per_step before reading the table as a budget.
There is no CPU path: without a CUDA device the tool fails."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

CONTEXTS = (64, 320, 576)


def step_bytes(cfg: dict, batch: int, ctx: int) -> list:
    """(kernel role, bytes it must move) for every launch of the fused decode step, in launch order."""
    H, I, hd = cfg["hidden_size"], cfg["intermediate_size"], cfg["head_dim"]
    nq, nkv, L, V = cfg["num_attention_heads"], cfg["num_key_value_heads"], cfg["num_hidden_layers"], cfg["vocab_size"]
    out = [("embed", batch * H * (2 + 4 + 4)), ("norm", batch * H * (4 + 4))]
    for _ in range(L):
        out += [("qkv", 2 * (nq + 2 * nkv) * hd * H),
                ("attention", 2 * batch * nkv * (ctx + 1) * hd * 4),      # fp32 K and V rows 0..ctx of this layer
                ("o", 2 * H * nq * hd), ("gate_up", 2 * 2 * I * H), ("down", 2 * H * I)]
    out += [("lm_head", 2 * V * H), ("sampler", batch * V * 4)]
    return out


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       check=True, capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"name": name, "power_limit": power, "clocks_max_sm": clock}


def kernel_records(torch, fn) -> list:
    """(name, start us, duration us) of every kernel `fn` runs, in start order."""
    from torch.profiler import ProfilerActivity, profile
    with tempfile.TemporaryDirectory() as tmp:
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        path = Path(tmp) / "trace.json"
        prof.export_chrome_trace(str(path))
        events = json.loads(path.read_text())["traceEvents"]
    ks = [(e["name"], float(e["ts"]), float(e["dur"])) for e in events if e.get("cat") == "kernel" and e.get("ph") == "X"]
    return sorted(ks, key=lambda k: k[1])


def fold(ks: list, n_launch: int, replays: int) -> tuple:
    """Median duration and gap per position over the last `replays` steps of the record (the first replay is a warm-up)."""
    assert len(ks) >= n_launch * (replays + 1), f"{len(ks)} kernel records, expected at least {n_launch * (replays + 1)}"
    ks = ks[-n_launch * replays:]
    steps = [ks[i * n_launch:(i + 1) * n_launch] for i in range(replays)]
    names = [k[0] for k in steps[0]]
    assert all([k[0] for k in s] == names for s in steps), "kernel order differs between replays: the fold is off by some launches"
    dur = np.array([[k[2] for k in s] for s in steps])
    start = np.array([[k[1] for k in s] for s in steps])
    gap = np.full_like(dur, np.nan)
    gap[:, 1:] = start[:, 1:] - (start[:, :-1] + dur[:, :-1])
    flat_s, flat_d = start.reshape(-1), dur.reshape(-1)
    gap[1:, 0] = flat_s[n_launch::n_launch] - (flat_s[n_launch - 1:-1:n_launch] + flat_d[n_launch - 1:-1:n_launch])
    return names, np.median(dur, axis=0), np.nanmedian(gap, axis=0), (start[:, -1] + dur[:, -1] - start[:, 0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--iters", type=int, default=24, help="graph replays per context (the first is a warm-up)")
    args = ap.parse_args()

    import torch
    import bench
    import mlx_audio_swift_b200 as m

    assert torch.cuda.is_available() and m.device_count() > 0, "step_timeline needs a CUDA device: there is no CPU path"
    cfg = dict(bench.ORPHEUS)
    rows = bench.BATCH
    tts = m.LlamaTTSModel.random_init(cfg, snac=None, device=0, max_batch=rows, max_context=max(CONTEXTS) + args.iters + 16,
                                      std=0.02, seed=1234)
    n_launch = 2 + 5 * cfg["num_hidden_layers"] + 2
    result = {"card": card(), "workload": bench.workload_name(cfg), "batch": rows, "launches_per_step": n_launch,
              "iters": args.iters, "contexts": {}}
    for ctx in CONTEXTS:
        tts.time_steps(rows, ctx, args.iters)                      # warm-up: modules loaded, graph captured once before
        event_ms = tts.time_steps(rows, ctx, args.iters)           # profiler off
        ks = kernel_records(torch, lambda: tts.time_steps(rows, ctx, args.iters))
        names, dur, gap, span = fold(ks, n_launch, args.iters - 1)
        roles = step_bytes(cfg, rows, ctx)
        table = [{"pos": i, "role": roles[i][0], "kernel": names[i], "dur_us": round(float(dur[i]), 3),
                  "gap_us": None if np.isnan(gap[i]) else round(float(gap[i]), 3), "bytes": int(roles[i][1]),
                  "gb_per_s": round(roles[i][1] / (float(dur[i]) * 1e-6) / 1e9, 1)} for i in range(n_launch)]
        by_role = {}
        for r in table:
            d = by_role.setdefault(r["role"], {"kernel": r["kernel"], "n": 0, "dur_us": [], "gap_us": [], "bytes": r["bytes"]})
            d["n"] += 1
            d["dur_us"].append(r["dur_us"])
            if r["gap_us"] is not None:
                d["gap_us"].append(r["gap_us"])
        for d in by_role.values():
            d["sum_dur_us"] = round(float(np.sum(d["dur_us"])), 1)
            d["dur_us"] = round(float(np.median(d["dur_us"])), 3)
            d["sum_gap_us"] = round(float(np.sum(d["gap_us"])), 1)
            d["gap_us"] = round(float(np.median(d["gap_us"])), 3) if d["gap_us"] else None
            d["gb_per_s"] = round(d["bytes"] / (d["dur_us"] * 1e-6) / 1e9, 1)
        gaps = np.array([r["gap_us"] for r in table if r["gap_us"] is not None])
        result["contexts"][str(ctx)] = {
            "event_ms_per_step": event_ms, "traced_ms_per_step": round(float(np.median(span)) * 1e-3, 4),
            "sum_dur_us": round(float(dur.sum()), 1), "sum_pos_gap_us": round(float(gaps[gaps > 0].sum()), 1),
            "sum_overlap_us": round(float(-gaps[gaps < 0].sum()), 1), "bytes_per_step": int(sum(b for _, b in roles)),
            "by_role": by_role, "kernels": table}
        c = result["contexts"][str(ctx)]
        print(f"ctx {ctx}: {event_ms:.3f} ms/step by events, {c['traced_ms_per_step']:.3f} traced; kernels {c['sum_dur_us']:.0f} us, "
              f"gaps {c['sum_pos_gap_us']:.0f} us, overlap {c['sum_overlap_us']:.0f} us")
        for role, d in by_role.items():
            print(f"  {role:10s} x{d['n']:3d}  {d['dur_us']:9.2f} us  gap {d['gap_us']}  {d['gb_per_s']:8.1f} GB/s  {d['kernel'][:60]}")
    out = Path(args.out_dir)
    out.mkdir(parents=True, exist_ok=True)
    (out / "step_timeline.json").write_text(json.dumps(result, indent=1))
    print(f"{result['card']}  ->  {out / 'step_timeline.json'}")


if __name__ == "__main__":
    main()
