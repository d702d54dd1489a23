"""
What clustering through the embedding index costs on one H100, against the exact greedy (a study, not part of bench.py):
embedding_clusters.cluster with and without an index, on rows generated on the device, the card's name and power limit read in
the same run.  Cases:
    families   1 M rows in 100 k near-duplicate families (tools/clusters_throughput.families), t = 0.99
    distinct   1 M all-distinct seeded rows (tools/neighbours_throughput.rows), t = 0.99
    encoder    encoder embeddings of synth windows (the index study's input), t = 0.99
    large      10 M seeded rows, index only; the exact time is extrapolated from a sampled covering run, labelled as such
For each run: the time per phase (probes, covering, block step, final assignment; each with a device synchronise on both sides),
R, peak device memory, and against the exact clustering the fraction of rows with the same representative and co-membership
precision and recall on a seeded sample of member pairs.  Index builds are timed apart.  Every shape is warmed up first.

    python tools/clusters_index_throughput.py [--n 1000000] [--encoder-n 262144] [--large-n 10000000] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from clusters_throughput import families  # noqa: E402
from neighbours_throughput import card, rows  # noqa: E402

T = 0.99


class Phases:
    """Synchronised timers around the index path's engine calls: the first calls of cluster_slots_search are the blocks'
    covering, the rest the final assignment."""

    def __init__(self, torch, EC, E):
        self.torch, self.E, self.EC = torch, E, EC
        self.orig = {k: getattr(E, k) for k in ("ivf_probes", "cluster_slots_search", "cluster_block_probed")}
        self.calls = []
        for k, fn in self.orig.items():
            setattr(E, k, self._timed(k, fn))

    def _timed(self, name, fn):
        def run(*a, **kw):
            self.torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn(*a, **kw)
            self.torch.cuda.synchronize()
            self.calls.append((name, time.perf_counter() - t0))
            return out
        return run

    def split(self, n, block):
        blocks = -(-n // block)
        out = {"probes": 0.0, "covering": 0.0, "block_step": 0.0, "final": 0.0}
        seen = 0
        for name, dt in self.calls:
            if name == "ivf_probes":
                out["probes"] += dt
            elif name == "cluster_block_probed":
                out["block_step"] += dt
            else:
                out["covering" if seen < blocks else "final"] += dt
                seen += 1
        self.calls = []
        return {k: round(v, 3) for k, v in out.items()}

    def close(self):
        for k, fn in self.orig.items():
            setattr(self.E, k, fn)


def agreement(exact, got, seed=0, sample=200_000):
    """Same-representative fraction; co-membership precision (index co-members that are exact co-members) and recall (exact
    co-members that are index co-members) over a seeded sample of (member, its representative) pairs of each clustering."""
    import numpy as np
    re_, ri = exact[0], got[0]
    rng = np.random.default_rng(seed)
    mem_i = np.flatnonzero(ri != np.arange(len(ri)))
    mem_e = np.flatnonzero(re_ != np.arange(len(re_)))
    pi = rng.choice(mem_i, min(sample, len(mem_i)), replace=False) if len(mem_i) else mem_i
    pe = rng.choice(mem_e, min(sample, len(mem_e)), replace=False) if len(mem_e) else mem_e
    precision = float((re_[pi] == re_[ri[pi]]).mean()) if len(pi) else 1.0
    recall = float((ri[pe] == ri[re_[pe]]).mean()) if len(pe) else 1.0
    return {"same_representative": round(float((re_ == ri).mean()), 5), "comembership_precision": round(precision, 5),
            "comembership_recall": round(recall, 5), "pairs_sampled": [int(len(pi)), int(len(pe))]}


def index_of(torch, E, x):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ix = E.ivf_build(x, E.ivf_default_lists(x.shape[0]), 20, 0)
    torch.cuda.synchronize()
    return {"centroids": ix.centroids.cpu().numpy(), "rows": ix.rows.cpu().numpy(), "offsets": ix.offsets.cpu().numpy(),
            "lists": ix.centroids.shape[0], "sha256": "-"}, round(time.perf_counter() - t0, 3)


def timed_cluster(torch, EC, emb, info, **kw):
    torch.cuda.reset_peak_memory_stats()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = EC.cluster(emb, T, info, **kw)
    torch.cuda.synchronize()
    return out, round(time.perf_counter() - t0, 3), round(torch.cuda.max_memory_allocated() / 2**30, 2)


def study(torch, E, EC, info, name, emb, nprobes, res, exact=True):
    torch.cuda.empty_cache()
    n = emb.shape[0]
    ix, t_build = index_of(torch, E, torch.from_numpy(emb).cuda())
    torch.cuda.empty_cache()
    EC.cluster(emb[:20_000], T, info)                                          # warm-up of every shape
    case = {"case": name, "n": n, "t": T, "lists": ix["lists"], "index_build_s": t_build, "runs": []}
    ex = None
    if exact:
        ex, dt, peak = timed_cluster(torch, EC, emb, info)
        case["runs"].append({"mode": "exact", "s": dt, "R": int(len(ex[2])), "peak_gib": peak})
        print(json.dumps(case["runs"][-1]), flush=True)
    ph = Phases(torch, EC, E)
    try:
        for p in nprobes:
            EC.cluster(emb[:8192], T, info, index=_sub_index(ix, 8192), nprobe=min(p, _sub_index(ix, 8192)["lists"]))
            ph.calls = []
            got, dt, peak = timed_cluster(torch, EC, emb, info, index=ix, nprobe=p)
            run = {"mode": f"index nprobe {p}", "s": dt, "R": int(len(got[2])), "peak_gib": peak, "phases_s": ph.split(n, 8192)}
            if ex is not None:
                run.update(agreement(ex, got))
            case["runs"].append(run)
            print(json.dumps(run), flush=True)
    finally:
        ph.close()
    res["cases"].append(case)
    return emb


def _sub_index(ix, m):
    """An index of the first m rows: their lists from ix (same centroids), for warm-up calls."""
    import numpy as np
    home = np.empty(len(ix["rows"]), np.int64)
    home[ix["rows"]] = np.repeat(np.arange(ix["lists"]), np.diff(ix["offsets"]))
    h = home[:m]
    return {"centroids": ix["centroids"], "rows": np.argsort(h, kind="stable"),
            "offsets": np.concatenate([[0], np.cumsum(np.bincount(h, minlength=ix["lists"]))]), "lists": ix["lists"], "sha256": "-"}


def exact_extrapolation(torch, E, x, reps=1_000_000, q=8192):
    """Exact covering rate: q rows against `reps` representatives at k = 1 (the exact path's covering call), and the time
    n^2 / 2 pairs would take at that rate."""
    E.embedding_neighbours(x[:q], x[q:q + 4096], 1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    E.embedding_neighbours(x[:q], x[q:q + reps], 1)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    rate = q * reps / dt
    n = x.shape[0]
    return {"sampled_pairs": q * reps, "sampled_s": round(dt, 4), "pairs_per_s": f"{rate:.3g}",
            "extrapolated_exact_covering_s_for_n2_over_2": round(n * n / 2 / rate, 1), "label": "extrapolation, not a measurement"}


def main():
    import torch
    from genomad_b200 import dist, embedding_clusters as EC, engine as E, synth
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--encoder-n", type=int, default=262_144)
    ap.add_argument("--large-n", type=int, default=10_000_000)
    ap.add_argument("--nprobe", type=int, nargs="+", default=[8, 16, 32])
    ap.add_argument("--large-nprobe", type=int, nargs="+", default=[16, 32])
    ap.add_argument("--cases", nargs="+", default=["families", "distinct", "encoder", "large"])
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    info = dist.DistInfo()
    res = {"card": card(), "t": T, "cases": []}
    print(json.dumps(res), flush=True)

    def save():
        if args.out:
            args.out.parent.mkdir(parents=True, exist_ok=True)
            args.out.write_text(json.dumps(res, indent=1) + "\n")

    if "families" in args.cases:
        study(torch, E, EC, info, "1 M rows in 100 k families", families(torch, args.n, 100_000, 3, "cuda").cpu().numpy(),
              args.nprobe, res)
        save()
    if "distinct" in args.cases:
        study(torch, E, EC, info, "all-distinct seeded rows", rows(torch, args.n, 5, "cuda").cpu().numpy(), [args.nprobe[-1]],
              res)
        save()
    if "encoder" in args.cases and args.encoder_n:
        clf = E.Classifier(None, device=0, max_batch=1024)
        embs = []
        for a in range(0, args.encoder_n, 1024):
            embs.append(clf.embed_ascii(synth.windows_torch(a, min(1024, args.encoder_n - a), 1, "cuda"))[1].clone())
        clf.close()
        study(torch, E, EC, info, "encoder embeddings of synth windows", torch.cat(embs).cpu().numpy(), args.nprobe, res)
        save()
    if "large" in args.cases and args.large_n:
        x = rows(torch, args.large_n, 9, "cuda")
        res["large_exact"] = exact_extrapolation(torch, E, x)
        print(json.dumps(res["large_exact"]), flush=True)
        emb = x.cpu().numpy()
        del x
        study(torch, E, EC, info, f"{args.large_n:,} seeded rows", emb, args.large_nprobe, res, exact=False)
        save()
    res["card_after"] = card()
    print(json.dumps({"card": res["card"], "card_after": res["card_after"]}))
    save()


if __name__ == "__main__":
    main()
