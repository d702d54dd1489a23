"""
What novelty attributions and window novelty cost on one H100 (a study, not part of bench.py), in one process, each pair run
alternately after a warm-up:

  api     Head.attribute_novelty_ascii vs Head.attribute_ascii on --windows seeded windows, a C = --classes head whose novelty
          model is fitted on those windows' own embeddings: gradient x input, and integrated gradients at m = --steps
  module  nn-classification --head H --write-novelty-attributions vs --write-head-attributions, and --write-window-novelty
          --window-stride 1000 vs --window-stride 1000, on the first --contigs seeded contigs of tools/contig_throughput.py

Writes <out>/head_novelty_attributions_h100.{md,json}; the card's name, power limit and clocks are read in the same run.

    python tools/novelty_attribution_throughput.py [--windows 4096] [--classes 7] [--steps 8] [--contigs 1000] [--reps 3]
                                                   [--out profiles]
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
sys.path.insert(0, str(ROOT / "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=4096)
    ap.add_argument("--classes", type=int, default=7)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--contigs", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=str(ROOT / "profiles"))
    a = ap.parse_args()
    import numpy as np
    import torch
    from attribution_throughput import alternate
    from contig_throughput import make_contigs
    from head_outputs_throughput import card, write_fasta
    from genomad_b200 import engine, nn_classification as nnc, synth, weights as W
    assert torch.cuda.is_available(), "needs an H100"
    res = {"card": card(), "windows": a.windows, "classes": a.classes, "ig_steps": a.steps, "reps": a.reps}
    win = synth.windows_numpy(synth.subsample_indices(a.windows, 1_000_000, seed=0), seed=0)
    d_win = torch.from_numpy(win).cuda()
    sync = torch.cuda.synchronize
    clf = engine.Classifier(None, device=0, max_batch=1024)
    clf._attr_ctx(engine.ATTR_MAX_BATCH)
    emb = clf.embed_ascii(d_win)[1]
    rng = np.random.default_rng(0)
    lab = rng.integers(0, a.classes, a.windows).astype(np.int32)
    lab[:a.classes] = np.arange(a.classes)
    fit = engine.novelty_fit(clf, emb, torch.arange(a.windows, device="cuda"), torch.from_numpy(lab).cuda(), a.classes)
    head = engine.Head(clf, W.HeadFile(W.initial_head(a.classes, 0), tuple(f"k{i}" for i in range(a.classes)), ""))
    head.set_novelty(fit.center, fit.whitening, fit.means)
    tg = rng.integers(0, a.classes, a.windows).astype(np.int32)
    res["attr_max_batch"] = clf.attr_max_batch
    calls = {"gxi": (lambda: (head.attribute_ascii(d_win, 2), sync()),
                     lambda: (head.attribute_novelty_ascii(d_win, tg), sync())),
             "ig": (lambda: (head.integrated_gradients_ascii(d_win, 2, a.steps, "zero"), sync()),
                    lambda: (head.integrated_gradients_novelty_ascii(d_win, tg, a.steps, "zero"), sync()))}
    for name, (fh, fn) in calls.items():
        th, tn = alternate(fh, fn, a.reps)
        res[name] = {"head_windows_per_s": a.windows / th, "novelty_windows_per_s": a.windows / tn, "time_ratio": tn / th}
        print(f"{name}: head {a.windows / th:,.0f} windows/s, novelty {a.windows / tn:,.0f} windows/s ({tn / th:.3f}x)",
              flush=True)
    clf.check_status()
    hp_arrays = {k: np.asarray(v) for k, v in W.initial_head(a.classes, 0).items()}
    head.close()
    clf.close()
    nnc.release_classifiers()
    torch.cuda.empty_cache()
    seq, offs = make_contigs(a.contigs, 0)
    res["contigs"], res["gbp"] = a.contigs, float(offs[-1]) / 1e9
    novelty = {"novelty_center": fit.center, "novelty_whitening": fit.whitening, "novelty_means": fit.means,
               "novelty_calibration": np.sort(rng.uniform(0.5, 3, 99)).astype(np.float32)}
    with tempfile.TemporaryDirectory() as d:
        d = Path(d)
        fa = d / "c.fna"
        write_fasta(fa, seq, offs)
        hfile = d / "h.npz"
        W.save_head(hfile, hp_arrays, tuple(f"k{i}" for i in range(a.classes)), W.load_weights(), novelty=novelty)
        pairs = {"attributions": ({"write_head_attributions": "k2"}, {"write_novelty_attributions": True}),
                 "window_novelty": ({"window_stride": 1000}, {"window_stride": 1000, "write_window_novelty": True})}
        nnc.main(fa, d / "warm", False, 128, False, 8, False, False, head=hfile)
        n, mod = 0, {}
        for name, (kb, kn) in pairs.items():
            times = {"base": [], "novelty": []}
            for _ in range(a.reps):
                for key, kw in (("base", kb), ("novelty", kn)):
                    n += 1
                    t0 = time.perf_counter()
                    nnc.main(fa, d / f"run{n}", False, 128, False, 8, False, False, head=hfile, **kw)
                    times[key].append(time.perf_counter() - t0)
            med = {k: statistics.median(v) for k, v in times.items()}
            mod[name] = {"s_all": times, "s": med, "time_ratio": med["novelty"] / med["base"]}
            print(f"module {name}: {med['base']:.2f} s vs {med['novelty']:.2f} s ({med['novelty'] / med['base']:.3f}x)",
                  flush=True)
        res["module"] = mod
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm,power.draw,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    res["clocks_after"] = q.stdout.strip().splitlines()[:1]
    out = Path(a.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "head_novelty_attributions_h100.json").write_text(json.dumps(res, indent=1, default=str))
    c = res["card"]
    md = ["# Novelty attributions and window novelty on one H100", "",
          f"Card: {json.dumps(c)}; clocks / power after the run: {res['clocks_after']}.", "",
          f"## API: {a.windows:,} seeded windows, a C = {a.classes} head (median of {a.reps} alternating runs)", "",
          "| call | Head.attribute_* windows/s | novelty windows/s | time ratio |", "|---|---|---|---|"]
    for name in ("gxi", "ig"):
        r = res[name]
        md.append(f"| {'gradient x input' if name == 'gxi' else f'IG m = {a.steps}'} | {r['head_windows_per_s']:,.0f} | "
                  f"{r['novelty_windows_per_s']:,.0f} | {r['time_ratio']:.3f} |")
    md += ["", f"## Module: the first {a.contigs:,} seeded contigs of tools/contig_throughput.py ({res['gbp']:.3f} Gbp)", "",
           "| pair | base s | with the option s | ratio |", "|---|---|---|---|"]
    for name, label in (("attributions", "--write-head-attributions k2 vs --write-novelty-attributions"),
                        ("window_novelty", "--window-stride 1000 vs + --write-window-novelty")):
        r = res["module"][name]
        md.append(f"| {label} | {r['s']['base']:.2f} | {r['s']['novelty']:.2f} | {r['time_ratio']:.3f} |")
    md += ["", "Measured by tools/novelty_attribution_throughput.py in one process; the card name and power limit above were "
           "read in the same run."]
    (out / "head_novelty_attributions_h100.md").write_text("\n".join(md) + "\n")


if __name__ == "__main__":
    main()
