#!/usr/bin/env python
"""
Same-card A/B of two builds of the library: the fused IGLOO kernel's stage times, the step time and the outputs.

    python tools/wvg_ab.py prepare REV DIR                # export commit REV into DIR and build it there (git + nvcc, no GPU)
    python tools/wvg_ab.py run --base DIR [--new DIR] --out OUT [--runs 3] [--steps 50] [--warmup 5]

`run` (GPU) compares two built trees; --new defaults to this repository.  It first dumps from each build q0, q1, mpi0, mpi1
and the probabilities of seeded batches of 1024 and 7 windows (shipped weights) and of every crowded patch set of
tests/test_gpu_igloo_patches.py at 9 and 24 windows, and reports whether the two builds agree bitwise.  Then it alternates
`bench.py --gpus 1 --steps K --warmup W --no-module --cpu-sample 0 --dump-outputs` between the builds, --runs times each, and
prints value, ms_per_step, stage_ms wvg0 / wvg1 and the sampled SM clock of every run, the per-build means and spreads, and
whether every run's probs.npy is bitwise the first run's.  The card's name, power limit and clocks are read in the same call.
What it keeps goes under OUT.
"""
import argparse
import json
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
DUMP_KEYS = ("q0", "mpi0", "q1", "mpi1", "probs")


def prepare(rev, out):
    out = Path(out).resolve()
    out.mkdir(parents=True, exist_ok=False)
    archive = subprocess.run(["git", "-C", str(ROOT), "archive", rev], check=True, capture_output=True).stdout
    subprocess.run(["tar", "-x", "-C", str(out)], input=archive, check=True)
    subprocess.run([sys.executable, "-m", "genomad_b200.build", "--force"], cwd=out, check=True, stdout=subprocess.DEVNULL)
    print(f"{rev} built in {out}")


def dump(tree, out):
    """(runs inside a subprocess with `tree` first on sys.path) the IGLOO stages and probabilities of the fixed cases"""
    import torch
    tree = Path(tree)
    sys.path[:0] = [str(tree), str(tree / "tests"), str(tree / "tools")]
    import test_gpu_igloo_patches as P
    import test_gpu_stages as S
    from oracle import igloo_model as M
    shipped = M.load_npz_weights(tree / "genomad_b200" / "data" / "nn_classifier.npz")
    synthetic = M.synthetic_igloo_weights(shipped)
    cases = [("shipped n=1024", shipped, S._windows(1024, seed=11), 1024), ("shipped n=7", shipped, S._windows(7, seed=12), 8)]
    for name in P.SETS:
        w, _ = P._crowded(name, synthetic)
        cases += [(f"{name} n=9", w, S._windows(9, seed=61), 9), (f"{name} n=24", w, S._windows(24, seed=67), 24)]
    res = {}
    for label, w, a, mb in cases:
        got = S._fetch(w, a, mb, {}, stops=(2, 0))
        for k in DUMP_KEYS:
            res[f"{label}/{k}"] = got[k].float().numpy()
    torch.cuda.synchronize()
    np.savez(out, **res)


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem,temperature.gpu"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return f"{q}: {r.stdout.strip()}"


def bench(tree, out_dir, args):
    cmd = [sys.executable, str(Path(tree) / "bench.py"), "--gpus", "1", "--steps", str(args.steps), "--warmup", str(args.warmup),
           "--no-module", "--cpu-sample", "0", "--dump-outputs", str(out_dir)]
    r = subprocess.run(cmd, cwd=tree, capture_output=True, text=True)
    if r.returncode != 0:
        sys.exit(f"bench.py failed in {tree}:\n{r.stderr[-3000:]}")
    line = json.loads(r.stdout.strip().splitlines()[-1])
    (Path(out_dir) / "bench.json").write_text(json.dumps(line) + "\n")
    return line


def run(args):
    out = Path(args.out).resolve()
    out.mkdir(parents=True, exist_ok=True)
    trees = {"base": Path(args.base).resolve(), "new": Path(args.new).resolve()}
    print(card(), flush=True)

    with tempfile.TemporaryDirectory() as tmp:                   # q0 / q1 of 1024 windows are ~0.4 GB each: not kept
        dumps = {}
        for label, tree in trees.items():
            f = Path(tmp) / f"stages_{label}.npz"
            subprocess.run([sys.executable, __file__, "dump", str(tree), str(f)], check=True, stdout=subprocess.DEVNULL)
            dumps[label] = np.load(f)
        keys = dumps["base"].files
        differ = [k for k in keys if not np.array_equal(dumps["base"][k], dumps["new"][k])]
    print(f"stage outputs: {len(keys)} arrays ({', '.join(DUMP_KEYS)} of {len(keys) // len(DUMP_KEYS)} cases), bitwise equal: "
          f"{not differ}" + (f"; differ: {differ}" if differ else ""), flush=True)

    rows = {label: [] for label in trees}
    for i in range(args.runs):
        for label, tree in trees.items():
            d = out / f"bench_{label}_{i}"
            line = bench(tree, d, args)
            r = dict(value=line["value"], ms=line["ms_per_step"], wvg0=line["stage_ms"].get("wvg0"), wvg1=line["stage_ms"].get("wvg1"),
                     mhz=(line.get("clocks") or {}).get("sm_mhz"), reasons=(line.get("clocks") or {}).get("reasons"),
                     probs=np.load(d / "probs.npy"))
            rows[label].append(r)
            print(f"run {i} {label:4s}: value {r['value']:,.0f} windows/s  ms/step {r['ms']:.3f}  wvg0 {r['wvg0']:.3f}  "
                  f"wvg1 {r['wvg1']:.3f}  sm MHz {r['mhz']}  {r['reasons']}", flush=True)
    print(card())

    first = rows["base"][0]["probs"]
    same = all(np.array_equal(r["probs"], first) for rs in rows.values() for r in rs)
    print(f"probs.npy of all {sum(len(v) for v in rows.values())} runs bitwise equal: {same}")
    print("| build | value (windows/s) | ms per step | wvg0 `stage_ms` | wvg1 `stage_ms` | sm MHz |")
    print("|---|---|---|---|---|---|")
    for label, rs in rows.items():
        cell = lambda k, f: " / ".join(f.format(r[k]) for r in rs)                 # noqa: E731
        print(f"| {label} | {cell('value', '{:,.0f}')} | {cell('ms', '{:.2f}')} | {cell('wvg0', '{:.2f}')} | {cell('wvg1', '{:.2f}')} "
              f"| {cell('mhz', '{:.0f}')} |")
    mean = {label: {k: float(np.mean([r[k] for r in rs])) for k in ("value", "ms", "wvg0", "wvg1")} for label, rs in rows.items()}
    spread = {label: float(np.ptp([r["value"] for r in rs])) for label, rs in rows.items()}
    b, n = mean["base"], mean["new"]
    print(f"mean value: base {b['value']:,.0f}, new {n['value']:,.0f} ({n['value'] / b['value']:.3f}x, gap {n['value'] - b['value']:,.0f}); "
          f"largest within-build spread {max(spread.values()):,.0f} (base {spread['base']:,.0f}, new {spread['new']:,.0f})")
    for k in ("wvg0", "wvg1", "ms"):
        print(f"mean {k}: base {b[k]:.3f} ms, new {n[k]:.3f} ms ({(n[k] / b[k] - 1) * 100:+.1f} %)")


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    p = sub.add_parser("prepare")
    p.add_argument("rev")
    p.add_argument("dir")
    r = sub.add_parser("run")
    r.add_argument("--base", required=True, help="built tree of the base build (see `prepare`)")
    r.add_argument("--new", default=str(ROOT), help="built tree of the new build (default: this repository)")
    r.add_argument("--out", required=True)
    r.add_argument("--runs", type=int, default=3)
    r.add_argument("--steps", type=int, default=50)
    r.add_argument("--warmup", type=int, default=5)
    d = sub.add_parser("dump")
    d.add_argument("tree")
    d.add_argument("out")
    args = ap.parse_args()
    if args.cmd == "prepare":
        prepare(args.rev, args.dir)
    elif args.cmd == "dump":
        dump(args.tree, args.out)
    else:
        run(args)


if __name__ == "__main__":
    main()
