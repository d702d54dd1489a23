"""
What the embedding index costs and finds on one H100 (a study, not part of bench.py), the card's name and power limit read in the
same run.  Inputs: seeded post-ReLU-like rows generated on the device (tools/neighbours_throughput.rows) and encoder embeddings
of synth windows.  For each input:
  * the build (engine.ivf_build's stages, each timed with a device synchronise on both sides) at L = ceil(4 sqrt(n)), 20
    iterations, seed 0;
  * all-vs-all k = 10 through the index at each nprobe, and the exact search (engine.embedding_neighbours) in the same run, with
    recall@10 against the exact lists;
  * at the first input, embedding-map's whole engine call with and without the index (--map-nprobe), and a per-kernel breakdown
    of one index search from torch.profiler in a separate run.

With --large-n N (and --skip-1m to run only it): N seeded rows, all-vs-all at each --large-nprobe, recall@10 on the first
--large-sample rows against their exact search.

    python tools/embedding_index_throughput.py [--n 1000000] [--encoder-n 262144] [--nprobe 1 4 16 32 64] [--out FILE.json]
    python tools/embedding_index_throughput.py --skip-1m --large-n 10000000 [--large-sample 10000] [--out FILE.json]
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


def recall(idx, ref):
    import torch
    hits = (idx[:, :, None] == ref[:, None, :]) & (ref[:, None, :] >= 0)
    return float(hits.any(1).sum(1).double().div(torch.clamp((ref >= 0).sum(1), min=1)).mean())


def timed(torch, t, name, fn, *a, **kw):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn(*a, **kw)
    torch.cuda.synchronize()
    t[name] = t.get(name, 0.0) + time.perf_counter() - t0
    return out


def build(torch, E, x, L, iters, seed, t):
    train = timed(torch, t, "training_rows", E.ivf_training_rows, x.shape[0], L, seed, x.device)
    xhat = timed(torch, t, "normalize", E.ivf_normalize, x.index_select(0, train).contiguous())
    cent = xhat[:L].clone()
    for _ in range(iters):
        best, assign = timed(torch, t, "assign", E.ivf_assign, xhat, cent)
        cent = timed(torch, t, "centroids", E.ivf_centroids, xhat, assign, L)
        cent, _ = timed(torch, t, "reseed", E.ivf_reseed, cent, xhat, train, best, assign)
    _, assign = timed(torch, t, "final_assign", E.ivf_assign, x, cent)
    order, off = timed(torch, t, "layout", E.ivf_layout, assign, L)
    return E.IvfIndex(cent, order, off)


def study(torch, E, name, x, nprobes, res):
    n = x.shape[0]
    L = E.ivf_default_lists(n)
    t = {}
    ix = build(torch, E, x, L, 20, 0, t)
    sizes = torch.diff(ix.offsets)
    case = {"input": name, "n": n, "lists": L, "build_seconds": {k: round(v, 4) for k, v in t.items()},
            "build_total_s": round(sum(t.values()), 3), "list_rows_min_median_max": [int(sizes.min()), int(sizes.median()),
                                                                                   int(sizes.max())],
            "empty_lists": int((sizes == 0).sum())}
    E.ivf_search(x[:1000], x, ix, 10, 4)                              # warm-up: modules, kernel attributes
    s = {}
    _, exact = timed(torch, s, "exact", E.embedding_neighbours, x, None, 10)
    case["exact_s"] = round(s["exact"], 3)
    case["search"] = []
    for p in nprobes:
        s = {}
        _, idx = timed(torch, s, "ivf", E.ivf_search, x, None, ix, 10, p)
        r = {"nprobe": p, "seconds": round(s["ivf"], 4), "speedup_vs_exact": round(case["exact_s"] / s["ivf"], 2),
             "recall_at_10": round(recall(idx, exact), 5)}
        case["search"].append(r)
        print(json.dumps({"input": name, **r}), flush=True)
        del idx
    del exact
    torch.cuda.empty_cache()
    res["cases"].append(case)
    print(json.dumps({k: v for k, v in case.items() if k != "search"}), flush=True)
    return ix


def large(torch, E, args, res):
    """All-vs-all through the index at n rows, recall@10 on the first `large_sample` rows (the exact search of that sample)."""
    n, m = args.large_n, args.large_sample
    x = rows(torch, n, 7, "cuda")
    L = E.ivf_default_lists(n)
    t = {}
    ix = build(torch, E, x, L, 20, 0, t)
    case = {"input": "seeded rows (large)", "n": n, "lists": L, "build_seconds": {k: round(v, 4) for k, v in t.items()},
            "build_total_s": round(sum(t.values()), 3), "recall_sample": m, "search": []}
    s = {}
    _, exact = timed(torch, s, "exact_sample", E.embedding_neighbours, x[:m], x, 10, self_index0=0)
    case["exact_sample_s"] = round(s["exact_sample"], 3)
    E.ivf_search(x[:1000], x, ix, 10, 4)
    for p in args.large_nprobe:
        s = {}
        _, idx = timed(torch, s, "ivf", E.ivf_search, x, None, ix, 10, p)
        r = {"nprobe": p, "seconds": round(s["ivf"], 3), "recall_at_10_sample": round(recall(idx[:m], exact), 5)}
        case["search"].append(r)
        print(json.dumps({"input": case["input"], **r}), flush=True)
        del idx
        torch.cuda.empty_cache()
    res["cases"].append(case)
    print(json.dumps({k: v for k, v in case.items() if k != "search"}), flush=True)
    del x, ix, exact
    torch.cuda.empty_cache()


def main():
    import torch
    from genomad_b200 import engine as E, synth
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--encoder-n", type=int, default=262_144)
    ap.add_argument("--nprobe", type=int, nargs="+", default=[1, 4, 16, 32, 64])
    ap.add_argument("--map-nprobe", type=int, default=16)
    ap.add_argument("--large-n", type=int, default=0, help="also a case of this many seeded rows, recall on a query sample")
    ap.add_argument("--large-sample", type=int, default=10_000)
    ap.add_argument("--large-nprobe", type=int, nargs="+", default=[1, 4, 16, 32])
    ap.add_argument("--skip-1m", action="store_true", help="only the large case")
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    res = {"card": card(), "k": 10, "cases": []}
    print(json.dumps(res), flush=True)
    if args.large_n:
        large(torch, E, args, res)
    if args.skip_1m:
        if args.out:
            args.out.parent.mkdir(parents=True, exist_ok=True)
            args.out.write_text(json.dumps(res, indent=1) + "\n")
        return
    x = rows(torch, args.n, 7, "cuda")
    ix = study(torch, E, "seeded rows", x, args.nprobe, res)

    # embedding-map's engine call, exact and through the index
    t = {}
    E.embedding_map(x[:2000], 15, 20, 0)
    timed(torch, t, "map_exact", E.embedding_map, x, 15, 200, 0)

    def map_ivf():
        s, i = E.ivf_search(x, None, ix, 15, args.map_nprobe)
        return E.map_layout(x, s, i, 200, 0)
    timed(torch, t, "map_index", map_ivf)
    res["map"] = {"n": args.n, "k": 15, "epochs": 200, "nprobe": args.map_nprobe, "exact_s": round(t["map_exact"], 3),
                  "index_s": round(t["map_index"], 3), "index_build_excluded": True}
    print(json.dumps(res["map"]), flush=True)

    # per-kernel breakdown of one index search (separate run)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        E.ivf_search(x, None, ix, 10, 32)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA":
            kern[e.key] = round(kern.get(e.key, 0.0) + e.device_time_total / 1e3, 3)
    res["kernels_ms_nprobe32"] = dict(sorted(kern.items(), key=lambda kv: -kv[1])[:16])
    print(json.dumps(res["kernels_ms_nprobe32"]), flush=True)
    del x, ix
    torch.cuda.empty_cache()

    if args.encoder_n:
        clf = E.Classifier(None, device=0, max_batch=1024)
        embs = []
        for a in range(0, args.encoder_n, 1024):
            embs.append(clf.embed_ascii(synth.windows_torch(a, min(1024, args.encoder_n - a), 1, "cuda"))[1].clone())
        clf.close()
        study(torch, E, "encoder embeddings of synth windows", torch.cat(embs).contiguous(), args.nprobe, res)
    print(json.dumps({"card": res["card"]}))
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
