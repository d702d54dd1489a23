"""
What attributions through a trained head cost on one H100 (a study, not part of bench.py), in one run, on the same seeded
device-resident windows, each pair run alternately after a warm-up:

  gxi  Head.attribute_ascii (a seeded C-class head) vs Classifier.attribute_ascii                         windows/s
  ig   Head.integrated_gradients_ascii vs Classifier.integrated_gradients_ascii, m = --steps (8)          windows/s

A head attribution chunk adds one TF32 dense_1 GEMM and one softmax to the classifier's.  The card's name, power limit and
clocks are read in the same call.

    python tools/head_attribution_throughput.py [--windows 4096] [--classes 7] [--steps 8] [--reps 3] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path
from types import SimpleNamespace

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
sys.path.insert(0, str(ROOT / "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=4096)
    ap.add_argument("--classes", type=int, default=7)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", type=str, default="")
    a = ap.parse_args()

    import torch
    from attribution_throughput import alternate
    from contig_throughput import card
    from head_ref import random_head
    from genomad_b200 import engine, synth
    if not torch.cuda.is_available():
        raise SystemExit("needs an H100")
    info = card()
    win = synth.windows_numpy(synth.subsample_indices(a.windows, 1_000_000, seed=a.seed), seed=a.seed)
    d_win = torch.from_numpy(win).cuda()
    sync = torch.cuda.synchronize
    clf = engine.Classifier(None, device=0, max_batch=1024)
    clf._attr_ctx(engine.ATTR_MAX_BATCH)
    head = engine.Head(clf, SimpleNamespace(arrays=random_head(a.classes, a.seed),
                                            class_names=tuple(f"k{i}" for i in range(a.classes))))
    res = {"card": info, "windows": a.windows, "classes": a.classes, "ig_steps": a.steps,
           "attr_max_batch": clf.attr_max_batch}
    out = {}

    def clf_gxi():
        out["p"], _ = clf.attribute_ascii(d_win, 2); sync()

    def head_gxi():
        out["hp"], out["hhp"], _ = head.attribute_ascii(d_win, 2); sync()

    def clf_ig():
        clf.integrated_gradients_ascii(d_win, 2, a.steps, "zero"); sync()

    def head_ig():
        head.integrated_gradients_ascii(d_win, 2, a.steps, "zero"); sync()

    tc, th = alternate(clf_gxi, head_gxi, a.reps)
    assert torch.equal(out["p"], out["hp"]), "the head call's shipped probabilities differ from the classifier call's"
    res["gxi"] = {"classifier_windows_per_s": a.windows / tc, "head_windows_per_s": a.windows / th, "time_ratio": th / tc}
    print(f"gradient x input: classifier {a.windows / tc:,.0f} windows/s, head (C = {a.classes}) {a.windows / th:,.0f} "
          f"windows/s ({th / tc:.3f}x the time)", flush=True)
    tc, th = alternate(clf_ig, head_ig, a.reps)
    res["ig"] = {"classifier_windows_per_s": a.windows / tc, "head_windows_per_s": a.windows / th, "time_ratio": th / tc}
    print(f"integrated gradients, m = {a.steps}: classifier {a.windows / tc:,.0f} windows/s, head {a.windows / th:,.0f} "
          f"windows/s ({th / tc:.3f}x the time)", flush=True)
    clf.check_status()
    head.close()
    clf.close()
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm,power.draw,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    res["clocks_after"] = q.stdout.strip().splitlines()[:1]
    print(json.dumps(res["card"]), res["clocks_after"])
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
