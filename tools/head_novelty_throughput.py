"""
Cost of head novelty on one GPU.

    python tools/head_novelty_throughput.py [--contigs 10000] [--reps 3] [--fit-rows 1000000] [--out profiles]

  * the fit (gnm_novelty_fit) on --fit-rows post-ReLU-like rows at C = 3 and 32: the whole call (host clock around a call that
    ends in a device synchronise, median of --reps) and, from a torch.profiler run of its own, the kernel time of the means
    (nv_class_sums + nv_means), the scatter (nv_scatter + nv_scatter_reduce) and the factor (nv_factor + nv_inverse +
    nv_whiten_means);
  * gnm_head_novelty rows/s against Head.predict (gnm_head_forward) on the same 262,144 rows, CUDA events over 20 calls;
  * nn-classification --head with a novelty head against the same head without the keys, on the seeded contigs of
    tools/contig_throughput.py, medians of --reps alternating runs (module wall clock);
  * train-head --novelty against plain train-head (3 classes, contig i labelled i mod 3, 3 epochs), medians of alternating runs.
Writes <out>/head_novelty_h100.{md,json} with the card's name and power limit, read in the same run.
"""
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

from head_outputs_throughput import card, write_fasta  # noqa: E402

PHASES = {"means": ("nv_class_sums", "nv_means"), "scatter": ("nv_scatter",), "factor": ("nv_factor", "nv_inverse", "nv_whiten")}


def fit_rows(torch, n, C, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = torch.randint(0, C, (n,), generator=g, device="cuda", dtype=torch.int32)
    centers = torch.randn((C, 512), generator=g, device="cuda")
    X = torch.relu(centers[y.long()] + torch.randn((n, 512), generator=g, device="cuda"))
    X[:, :40] = 0                                          # dead columns, as after the encoder's ReLU
    return X.contiguous(), y


def time_fit(torch, clf, C, n, reps):
    from genomad_b200 import engine
    X, y = fit_rows(torch, n, C)
    rows = torch.arange(n, dtype=torch.int64, device="cuda")
    engine.novelty_fit(clf, X, rows, y, C)                 # warm-up
    wall = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fit = engine.novelty_fit(clf, X, rows, y, C)
        wall.append(time.perf_counter() - t0)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        engine.novelty_fit(clf, X, rows, y, C)
    phase = {k: 0.0 for k in PHASES}
    for ev in prof.key_averages():
        for k, names in PHASES.items():
            if any(nm in ev.key for nm in names):
                phase[k] += ev.device_time_total / 1e6 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e6
    del X, y, rows
    torch.cuda.empty_cache()
    return {"wall_s": statistics.median(wall), "wall_s_all": wall, "kernel_s": phase, "min_pivot": fit.min_pivot}, fit


def time_score(torch, clf, fit, C, n=262144, calls=20):
    from genomad_b200 import engine, weights as W
    h = engine.Head(clf, W.HeadFile(W.initial_head(C, 0), tuple(f"c{i}" for i in range(C)), ""))
    h.set_novelty(fit.center, fit.whitening, fit.means)
    X, _ = fit_rows(torch, n, C, seed=1)
    out = {}
    for name, fn in (("novelty", h.novelty), ("predict", h.predict)):
        fn(X)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(calls):
            fn(X)
        b.record()
        b.synchronize()
        out[name] = n * calls / (a.elapsed_time(b) / 1e3)
    h.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--contigs", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--fit-rows", type=int, default=1_000_000)
    ap.add_argument("--out", default=str(ROOT / "profiles"))
    args = ap.parse_args()
    import torch
    from contig_throughput import make_contigs
    from genomad_b200 import engine, nn_classification as nnc, sequence, train_head, weights as W
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"card": card(), "contigs": args.contigs, "reps": args.reps, "fit_rows": args.fit_rows}
    clf = engine.Classifier(None, device=0, max_batch=1024)
    res["fit"], res["score_rows_per_s"] = {}, {}
    for C in (3, 32):
        r, fit = time_fit(torch, clf, C, args.fit_rows, args.reps)
        res["fit"][C] = r
        res["score_rows_per_s"][C] = time_score(torch, clf, fit, C)
    clf.close()
    torch.cuda.empty_cache()
    seq, offs = make_contigs(args.contigs, 0)
    res["gbp"] = float(offs[-1]) / 1e9
    with tempfile.TemporaryDirectory() as d:
        d = Path(d)
        fa = d / "c.fna"
        write_fasta(fa, seq, offs)
        del seq
        pf = sequence.ParsedFasta(fa)
        res["windows"] = int(pf.n_windows)
        pf.close()
        labels = d / "labels.tsv"
        labels.write_text("seq_name\tclass\n" + "".join(f"c{i}\t{'abc'[i % 3]}\n" for i in range(args.contigs)))
        train = {}
        for rep in range(args.reps):
            for name, nov in (("plain", False), ("novelty", True)):
                t0 = time.perf_counter()
                train_head.main(fa, labels, d / f"train_{name}{rep}", epochs=3, batch_size=256, seed=0, verbose=False,
                                novelty=nov)
                train.setdefault(name, []).append(time.perf_counter() - t0)
        res["train_head_s_all"] = train
        res["train_head_s"] = {k: statistics.median(v) for k, v in train.items()}
        hn = d / "train_novelty0" / "c_head.npz"
        hp = d / "train_plain0" / "c_head.npz"
        res["calibration_size"] = int(len(W.load_head(hn, W.load_weights()).novelty["novelty_calibration"]))
        nnc.main(fa, d / "warm", False, 128, False, 8, False, False, head=hn)
        times, n = {}, 0
        for rep in range(args.reps):
            for name, h in (("plain", hp), ("novelty", hn)):
                n += 1
                t0 = time.perf_counter()
                nnc.main(fa, d / f"run{n}", False, 128, False, 8, False, False, head=h)
                times.setdefault(name, []).append(time.perf_counter() - t0)
        res["module_s_all"] = times
        res["module_s"] = {k: statistics.median(v) for k, v in times.items()}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "head_novelty_h100.json").write_text(json.dumps(res, indent=1, default=str) + "\n")
    f, s, m, t = res["fit"], res["score_rows_per_s"], res["module_s"], res["train_head_s"]
    md = [f"# Head novelty on {res['card']}", "",
          "Measured by tools/head_novelty_throughput.py in one process; the card name and power limit above were read in the "
          "same run.", "",
          f"## Fit, {args.fit_rows:,} post-ReLU-like rows (median of {args.reps}; kernel times from a profiled run of its own)", "",
          "| C | whole call (s) | means (ms) | scatter (ms) | factor (ms) |", "|---|---|---|---|---|"]
    for C in (3, 32):
        k = f[C]["kernel_s"]
        md.append(f"| {C} | {f[C]['wall_s']:.3f} | {k['means'] * 1e3:.1f} | {k['scatter'] * 1e3:.1f} | {k['factor'] * 1e3:.1f} |")
    md += ["", "## Scoring, 262,144 rows, CUDA events over 20 calls", "",
           "| C | gnm_head_novelty (rows/s) | Head.predict (rows/s) |", "|---|---|---|"]
    for C in (3, 32):
        md.append(f"| {C} | {s[C]['novelty']:,.0f} | {s[C]['predict']:,.0f} |")
    md += ["", f"## End to end, the {args.contigs:,} seeded contigs of tools/contig_throughput.py ({res['gbp']:.2f} Gbp, "
           f"{res['windows']:,} windows), medians of {args.reps} alternating runs", "",
           "| run | without the model (s) | with it (s) | ratio |", "|---|---|---|---|",
           f"| nn-classification --head | {m['plain']:.2f} | {m['novelty']:.2f} | {m['novelty'] / m['plain']:.3f} |",
           f"| train-head (3 epochs, batch 256) | {t['plain']:.2f} | {t['novelty']:.2f} | {t['novelty'] / t['plain']:.3f} |",
           "", f"The novelty head's calibration set holds {res['calibration_size']} validation sequences.", ""]
    (out / "head_novelty_h100.md").write_text("\n".join(md))
    print("\n".join(md))


if __name__ == "__main__":
    main()
