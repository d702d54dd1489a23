"""
What integrated gradients cost on one H100 (a study, not part of bench.py): Classifier.integrated_gradients_ascii at m = 8 and
32 against attribute_ascii and predict_ascii on the same device-resident seeded windows, run alternately after a warm-up, with
the probabilities checked bitwise against predict_ascii and the card's name and power limit read in the same run.

    python tools/ig_throughput.py [--windows 1024] [--seed 0] [--reps 3] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                   # noqa: BLE001
        q = f"unavailable ({e})"
    return q


def main():
    import torch
    from genomad_b200 import engine, synth
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=1024)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    idx = synth.subsample_indices(args.windows, 1_000_000, seed=args.seed)
    a = torch.from_numpy(synth.windows_numpy(idx, seed=args.seed)).cuda()
    c = engine.Classifier(None, device=0, max_batch=1024)
    c._attr_ctx(engine.ATTR_MAX_BATCH)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out

    calls = {"predict_ascii": lambda: (c.predict_ascii(a),),
             "attribute_ascii": lambda: c.attribute_ascii(a, 2),
             "ig_m8": lambda: c.integrated_gradients_ascii(a, 2, 8, "zero"),
             "ig_m32": lambda: c.integrated_gradients_ascii(a, 2, 32, "zero")}
    ref = c.predict_ascii(a)
    for name, fn in calls.items():                           # warm-up, and the probabilities bitwise predict_ascii's
        out = fn()
        assert torch.equal(out[0], ref), name
    times = {k: [] for k in calls}
    for _ in range(args.reps):
        for name, fn in calls.items():
            times[name].append(timed(fn)[0])
    c.check_status()
    res = {"card": card(), "windows": args.windows, "reps": args.reps, "attr_chunk": engine.ATTR_MAX_BATCH,
           "seconds": times, "windows_per_s": {k: args.windows / float(np.median(v)) for k, v in times.items()}}
    base = res["windows_per_s"]["predict_ascii"]
    res["cost_in_forwards"] = {k: base / v for k, v in res["windows_per_s"].items()}
    print(json.dumps(res, indent=1))
    if args.out:
        args.out.write_text(json.dumps(res, indent=1))
    c.close()


if __name__ == "__main__":
    main()
