"""
What the embedding map costs on one H100 (a study, not part of bench.py): engine.embedding_map's stages on seeded post-ReLU-like
rows generated on the device (tools/neighbours_throughput.rows), k = 15 and umap-learn's default epochs, the card's name and
power limit read in the same run.  Each stage is timed with a device synchronise on both sides: the all-vs-all kNN search, the
memberships, the graph bookkeeping, the PCA (normalisation, covariance, eigenvectors), the initialisation and the layout
epochs; then the whole engine.embedding_map call on its own.  Also the CSR edge count and the layout's edge-visits per second.

    python tools/embedding_map_throughput.py [--sizes 100000 1000000] [--out FILE.json]
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


def main():
    import torch
    from genomad_b200 import engine as E
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--k", type=int, default=15)
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    res = {"card": card(), "k": args.k, "cases": []}
    warm = rows(torch, 2000, 1, "cuda")
    E.embedding_map(warm, args.k, 20, 0)                        # loads the modules, sets the kernels' attributes
    for n in args.sizes:
        x = rows(torch, n, 7, "cuda")
        epochs = E.map_default_epochs(n)
        t = {}

        def timed(name, fn, *a):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn(*a)
            torch.cuda.synchronize()
            t[name] = time.perf_counter() - t0
            return out

        sim, idx = timed("knn", E.embedding_neighbours, x, None, args.k)
        m = timed("membership", E.map_membership, sim, idx)
        g = timed("graph", E.map_graph, m.union, idx, epochs)
        xh, center, _, V = timed("pca", E.map_pca, x)
        Y = timed("init", E.map_init, xh, center, V, 0)
        Y = timed("epochs", E.map_epochs, g, Y, epochs, 0)
        del m, xh
        total = timed("embedding_map", E.embedding_map, x, args.k, epochs, 0)
        assert torch.equal(total, Y), "the staged run and the one call differ"
        nnz = int(g.col.numel())
        visits = sum(int(((torch.floor(e / g.eps) > torch.floor((e - 1) / g.eps))).sum()) for e in range(1, epochs))
        case = {"n": n, "epochs": epochs, "csr_entries": nnz, "sampled_entries": visits,
                "seconds": {k_: round(v, 4) for k_, v in t.items()},
                "layout_share_of_knn": round(t["epochs"] / t["knn"], 4),
                "sampled_entries_per_s": round(visits / t["epochs"], 1)}
        print(json.dumps(case), flush=True)
        res["cases"].append(case)
        del sim, idx, g, Y, total, x
        torch.cuda.empty_cache()
    print(json.dumps({"card": res["card"]}))
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
