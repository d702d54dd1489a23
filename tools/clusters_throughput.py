"""
What greedy embedding clustering costs on one H100 (a study, not part of bench.py): embedding_clusters.cluster on seeded rows
generated on the device, the card's name and power limit read in the same run.  Cases:
    a  1 M rows in 100 k near-duplicate families (2 % multiplicative noise on sparse post-ReLU-like rows), t = 0.99
    b  300 k all-distinct sparse rows, t = 0.99: every row is a representative, the worst case for covering
    c  the first 100 k rows of a
For each: the time split into covering (embedding_neighbours at k = 1 against the representatives), mask + resolve
(gnm_cluster_block) and the final assignment (k = 1 search of the members against the representatives), each phase timed with a
device synchronise on both sides; the pairs each phase evaluates and pairs/s; and the all-vs-all embedding_neighbours time
(k = 10) at the same n.  Also an fp32 CPU statement of the same greedy (blocked matmuls + a sequential in-block pass) at a small n.

    python tools/clusters_throughput.py [--cases a b c] [--cpu-n 20000] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from neighbours_throughput import card, rows  # noqa: E402

T = 0.99


def families(torch, n, n_fam, seed, device):
    g = torch.Generator(device=device).manual_seed(seed)
    base = rows(torch, n_fam, seed, device)
    fam = torch.randint(0, n_fam, (n,), generator=g, device=device)
    return base[fam] * (1 + 0.02 * torch.randn((n, 512), generator=g, device=device))


class Phases:
    """Wraps the module's phase functions with synchronised timers and pair counters."""

    def __init__(self, torch, EC, EN, engine):
        self.t = {"covering": 0.0, "mask_resolve": 0.0, "final": 0.0}
        self.pairs = {"covering": 0, "mask_resolve": 0, "final": 0}
        self.torch = torch
        cov, blk, search = EC._covered, engine.cluster_block, EN.search

        def timed(name, fn, pairs):
            def run(*a, **k):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = fn(*a, **k)
                torch.cuda.synchronize()
                self.t[name] += time.perf_counter() - t0
                self.pairs[name] += pairs(*a)
                return out
            return run

        EC._covered = timed("covering", cov, lambda b, r, *_: b.shape[0] * r.shape[0])
        engine.cluster_block = timed("mask_resolve", blk, lambda b, *_: b.shape[0] * (b.shape[0] - 1) // 2)
        EN.search = timed("final", search, lambda q, r, *_: q.shape[0] * r.shape[0])


def cpu_greedy(torch, x, t, block=1024):
    """fp32 CPU greedy with the same definition: covering by matmul, a sequential in-block pass, a final matmul + argmax."""
    xn = x / x.norm(dim=1, keepdim=True).clamp(min=1e-30)
    reps = []
    for a in range(0, len(xn), block):
        b = xn[a:a + block]
        cov = ((b @ xn[reps].T).max(dim=1).values >= t) if reps else torch.zeros(len(b), dtype=torch.bool)
        s = (b @ b.T >= t).numpy()
        cov = cov.numpy()
        new = []
        for j in range(len(b)):
            if not cov[j] and not any(s[j, i] for i in new):
                new.append(j)
        reps += [a + j for j in new]
    r = torch.tensor(reps)
    members = torch.ones(len(xn), dtype=torch.bool)
    members[r] = False
    (xn[members] @ xn[r].T).max(dim=1)
    return len(reps)


def main():
    import numpy as np
    import torch
    from genomad_b200 import dist, embedding_clusters as EC, embedding_neighbours as EN, engine
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="+", default=["c", "b", "a"])
    ap.add_argument("--cpu-n", type=int, default=20_000)
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    res = {"card": card(), "min_similarity": T, "block": engine.CLUSTER_MAX_BLOCK, "cases": []}
    print(json.dumps({"card": res["card"]}), flush=True)
    ph = Phases(torch, EC, EN, engine)
    info = dist.DistInfo()
    EC.cluster(rows(torch, 20_000, 1, "cuda").cpu().numpy(), T, info)                  # warm-up: module load, every kernel
    for case in args.cases:
        if case == "b":
            x = rows(torch, 300_000, 2, "cuda")
        else:
            x = families(torch, 1_000_000, 100_000, 3, "cuda")
            if case == "c":
                x = x[:100_000].clone()
        n = x.shape[0]
        xh = x.cpu().numpy()
        for k in ph.t:
            ph.t[k], ph.pairs[k] = 0.0, 0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ri, sim, reps = EC.cluster(xh, T, info)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        r = {"case": case, "n": n, "representatives": int(len(reps)), "seconds_total": total,
             "seconds": dict(ph.t), "pairs": dict(ph.pairs),
             "pairs_per_s": {k: (ph.pairs[k] / ph.t[k] if ph.t[k] else None) for k in ph.t},
             "largest_cluster": int(np.bincount(np.searchsorted(reps, ri)).max())}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        engine.embedding_neighbours(x, None, 10)
        torch.cuda.synchronize()
        r["all_vs_all_k10_seconds"] = time.perf_counter() - t0
        res["cases"].append(r)
        print(json.dumps(r), flush=True)
        del x, xh
        torch.cuda.empty_cache()
    cpu = []
    for name, xc in (("distinct", rows(torch, args.cpu_n, 7, "cpu")), ("families", families(torch, args.cpu_n, args.cpu_n // 10, 8, "cpu"))):
        t0 = time.perf_counter()
        nr = cpu_greedy(torch, xc, T)
        cpu.append({"rows": name, "n": args.cpu_n, "representatives": nr, "threads": torch.get_num_threads(),
                    "seconds": time.perf_counter() - t0})
        print(json.dumps(cpu[-1]), flush=True)
    res["cpu_fp32_greedy"] = cpu
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
