"""
What the embedding-neighbour search costs on one H100 (a study, not part of bench.py): engine.embedding_neighbours all-vs-all
(k = 10) on seeded post-ReLU-like rows generated on the device, after a warm-up of the same shape, with the card's name and
power limit read in the same run.  Reports time, pairs/s, algorithmic TFLOP/s (2 * 512 flop per pair, one pass) and the share
of the 3-pass TF32 floor (3 * 2 * 512 flop per pair at the data sheet's 495 TFLOP/s), a per-kernel breakdown from
torch.profiler in a separate run, and a CPU baseline (fp32 torch.matmul + topk) at a small n.

    python tools/neighbours_throughput.py [--sizes 100000 300000 1000000] [--k 10] [--cpu-n 20000] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

TF32_PEAK = 495e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                   # noqa: BLE001
        q = f"unavailable ({e})"
    return q


def rows(torch, n, seed, device):
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn((n, 512), generator=g, device=device).clamp_(min=0)
    return x * (torch.rand((n, 512), generator=g, device=device) < 0.3)


def main():
    import torch
    from genomad_b200 import engine
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 300_000, 1_000_000])
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--cpu-n", type=int, default=20_000)
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    res = {"card": card(), "k": args.k, "chunk": engine.NEIGHBOURS_CHUNK, "all_vs_all": []}
    for n in args.sizes:
        x = rows(torch, n, n, "cuda")
        engine.embedding_neighbours(x[: min(n, 20_000)], None, args.k)          # warm-up: module load, workspace
        times = []
        for _ in range(2 if n <= 300_000 else 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sim, idx = engine.embedding_neighbours(x, None, args.k)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        t = min(times)
        pairs = float(n) * (n - 1)
        r = {"n": n, "seconds": times, "pairs_per_s": pairs / t, "tflops_1pass": pairs * 1024 / t / 1e12,
             "share_of_3pass_tf32_floor": pairs * 3 * 1024 / TF32_PEAK / t}
        res["all_vs_all"].append(r)
        print(json.dumps(r), flush=True)
        del x, sim, idx
        torch.cuda.empty_cache()
    # per-kernel breakdown at the first size
    n = args.sizes[0]
    x = rows(torch, n, n, "cuda")
    engine.embedding_neighbours(x, None, args.k)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        engine.embedding_neighbours(x, None, args.k)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA":
            kern[e.key] = kern.get(e.key, 0.0) + e.device_time_total / 1e3     # ms
    res["kernels_ms_at_n"] = {"n": n, "ms": kern}
    print(json.dumps(res["kernels_ms_at_n"]), flush=True)
    # CPU baseline: fp32 matmul + topk, all-vs-all
    m = args.cpu_n
    xc = rows(torch, m, 7, "cpu")
    t0 = time.perf_counter()
    xn = xc / xc.norm(dim=1, keepdim=True).clamp(min=1e-30)
    s = xn @ xn.T
    s.fill_diagonal_(-float("inf"))
    torch.topk(s, args.k, dim=1)
    tc = time.perf_counter() - t0
    res["cpu_baseline"] = {"n": m, "threads": torch.get_num_threads(), "seconds": tc, "pairs_per_s": float(m) * (m - 1) / tc}
    print(json.dumps(res["cpu_baseline"]), flush=True)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
