"""
Cost of the per-window score export on one H100 (a study, not part of bench.py).  On the seeded contig set of
tools/contig_throughput.py (10,000 contigs, lengths log-uniform on [1 kb, 500 kb]) it times

  plan      gnm_contig_windows_stride on device-resident sequences at strides 6000, 1000 and 100     ms, ms per Gbp
  scores    Classifier.window_scores at stride 1000 (plan + gnm_forward_windows) against gnm_forward_ascii on the same
            windows gathered beforehand (first --score-contigs contigs)                               windows/s
  module    nn-classification on the set as FASTA, with --write-window-scores (stride 6000) and without, alternating
            runs                                                                                      s
  tsv       the native window-score table writer                                                     rows/s

and prints the card's name and power limit with the numbers (one JSON line; --out also writes it to a file).

    python tools/window_scores_throughput.py [--contigs 10000] [--seed 0] [--reps 3] [--runs 5] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--contigs", type=int, default=10000)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--score-contigs", type=int, default=1000)
    ap.add_argument("--tsv-rows", type=int, default=10_000_000)
    ap.add_argument("--out", type=str, default="")
    a = ap.parse_args()

    import torch
    from contig_throughput import card, make_contigs
    from genomad_b200 import engine, nn_classification
    if not torch.cuda.is_available():
        raise SystemExit("needs an H100")
    seq_h, offs_h = make_contigs(a.contigs, a.seed)
    gbp = seq_h.size / 1e9
    clf = engine.Classifier(None, device=0, max_batch=1024)
    seq, offs = torch.from_numpy(seq_h).cuda(), torch.from_numpy(offs_h).cuda()

    def timed(fn, reps=a.reps):
        fn(); torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); ts.append(time.perf_counter() - t0)
        return float(np.median(ts))

    out = {"card": card(), "contigs": a.contigs, "seed": a.seed, "gbp": round(gbp, 4)}
    # ---- device planning
    for s in (6000, 1000, 100):
        r = {}
        t = timed(lambda: r.update(p=clf.contig_windows(seq, offs, stride=s)))
        out[f"plan_s{s}"] = {"windows": int(r["p"][0].numel()), "ms": round(t * 1e3, 3), "ms_per_gbp": round(t * 1e3 / gbp, 3)}
        del r
    torch.cuda.empty_cache()

    # ---- window_scores at stride 1000 against forward_ascii on the same windows, gathered beforehand
    k = min(a.score_contigs, a.contigs)
    sub = (seq[: int(offs_h[k])], offs[: k + 1])
    res = {}
    t_ws = timed(lambda: res.update(w=clf.window_scores(sub, stride=1000)), reps=2)
    start, length, _woff = clf.contig_windows(sub[0], sub[1], stride=1000)
    ascii_w = clf.gather_windows(sub[0], start, length)
    t_as = timed(lambda: res.update(a=clf.predict_ascii(ascii_w)), reps=2)
    assert torch.equal(res["w"].probs, res["a"]), "window_scores and forward_ascii differ"
    n_ws = int(start.numel())
    out["scores_s1000"] = {"contigs": k, "gbp": round(int(offs_h[k]) / 1e9, 4), "windows": n_ws,
                           "window_scores_windows_per_s": round(n_ws / t_ws), "forward_ascii_windows_per_s": round(n_ws / t_as),
                           "window_scores_over_ascii": round(t_as / t_ws, 4)}
    del ascii_w, res, start, length
    clf.check_status()
    clf.close()
    torch.cuda.empty_cache()

    # ---- module wall clock with and without --write-window-scores (stride 6000), alternating
    tmp = Path(tempfile.mkdtemp(prefix="gnm_ws_"))
    try:
        fa = tmp / "set.fna"
        with open(fa, "wb") as fh:
            for i in range(a.contigs):
                s = seq_h[offs_h[i]:offs_h[i + 1]].tobytes()
                fh.write(b">c%d\n" % i + b"\n".join(s[j:j + 80] for j in range(0, len(s), 80)) + b"\n")
        threads = min(32, len(os.sched_getaffinity(0)))
        walls = {"off": [], "on": []}
        nn_classification.main(fa, tmp / "warm", False, 128, False, threads, False, False)       # classifier + page cache
        for r in range(a.runs):
            for mode in ("off", "on"):
                d = tmp / f"{mode}{r}"
                t0 = time.perf_counter()
                nn_classification.main(fa, d, False, 128, False, threads, False, False, write_window_scores=(mode == "on"))
                walls[mode].append(time.perf_counter() - t0)
                shutil.rmtree(d)
        med = {m: float(np.median(v)) for m, v in walls.items()}
        out["module_s6000"] = {"runs": a.runs, "threads": threads, "off_s": [round(x, 3) for x in walls["off"]],
                               "on_s": [round(x, 3) for x in walls["on"]], "median_off_s": round(med["off"], 3),
                               "median_on_s": round(med["on"], 3), "on_over_off": round(med["on"] / med["off"], 4)}
        # ---- the table writer
        rng = np.random.default_rng(1)
        n = a.tsv_rows
        n_c = max(1, n // 50)
        offsets = np.linspace(0, n, n_c + 1).astype(np.int32)
        names = [f"contig_{i}" for i in range(n_c)]
        starts = rng.integers(0, 10 ** 7, n).astype(np.int64)
        lengths = np.full(n, 6000, np.int32)
        probs = rng.random((n, 3), dtype=np.float32)
        t0 = time.perf_counter()
        nn_classification._write_window_tsv(tmp / "w.tsv", names, offsets, starts, lengths, probs, threads)
        t_tsv = time.perf_counter() - t0
        out["tsv_writer"] = {"rows": n, "threads": threads, "s": round(t_tsv, 3), "rows_per_s": round(n / t_tsv),
                             "bytes": (tmp / "w.tsv").stat().st_size}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        nn_classification.release_classifiers()
    print(json.dumps(out))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
