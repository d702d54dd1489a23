"""
Cost of the head's strand and window outputs and of train-head --both-strands on one GPU.

    python tools/head_outputs_throughput.py [--contigs 10000] [--reps 3] [--out profiles]

On the seeded contigs of tools/contig_throughput.py (10,000 contigs, ~0.8 Gbp), in one process, alternating the two runs of each
pair and reporting medians:
  * nn-classification --head --both-strands against --both-strands (module wall clock);
  * nn-classification --head --window-stride 1000 against --window-stride 1000 (module wall clock);
  * train-head --both-strands against train-head (3 classes, contig i labelled i mod 3, 3 epochs): the embedding time (the
    chunk-loop passes, ended by a device synchronise) and the time per epoch (training steps plus validation).
The head is the shipped classifier's tail saved as a head file (C = 3).  Writes <out>/head_outputs_h100.{md,json} with the
card's name and power limit, read in the same run.
"""
import argparse
import json
import statistics
import subprocess
import sys
import tempfile
import time
from pathlib import Path


ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def write_fasta(path, seq, offs):
    with open(path, "wb") as f:
        for i in range(len(offs) - 1):
            f.write(f">c{i}\n".encode() + seq[offs[i]: offs[i + 1]].tobytes() + b"\n")


def timed_train(torch, train_head, nnc, fa, labels, out, both):
    """(embedding s, [epoch s]) of one train-head run: the chunk-loop passes, each ended by a device synchronise, and the time
    from one epoch's weight read (after its last step) to the next, which covers a validation and an epoch's steps."""
    marks = {"embed": 0.0, "epochs": []}
    classify = nnc._chunk_pass

    def classify_timed(*a, **k):
        t0 = time.perf_counter()
        r = classify(*a, **k)
        torch.cuda.synchronize()
        marks["embed"] += time.perf_counter() - t0
        marks["last"] = time.perf_counter()
        return r

    nnc._chunk_pass = classify_timed
    trainer_make = train_head._make_trainer

    def trainer_timed(*a, **k):
        tr = trainer_make(*a, **k)
        w = tr.weights

        def weights():                             # read at the end of each epoch's steps
            r = w()
            now = time.perf_counter()
            marks["epochs"].append(now - marks["last"])
            marks["last"] = now
            return r
        tr.weights = weights
        return tr
    train_head._make_trainer = trainer_timed
    try:
        train_head.main(fa, labels, out, epochs=3, batch_size=256, seed=0, verbose=False, both_strands=both)
    finally:
        nnc._chunk_pass, train_head._make_trainer = classify, trainer_make
    return marks["embed"], marks["epochs"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--contigs", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=str(ROOT / "profiles"))
    args = ap.parse_args()
    import torch
    from contig_throughput import make_contigs
    from genomad_b200 import nn_classification as nnc, sequence, train_head, weights as W
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"card": card(), "contigs": args.contigs, "reps": args.reps}
    seq, offs = make_contigs(args.contigs, 0)
    res["gbp"] = float(offs[-1]) / 1e9
    with tempfile.TemporaryDirectory() as d:
        d = Path(d)
        fa = d / "c.fna"
        write_fasta(fa, seq, offs)
        del seq
        pf = sequence.ParsedFasta(fa)
        res["windows"] = int(pf.n_windows)
        wl = pf.windows(1000)
        res["profile_windows_1000"] = int(wl.n_windows)
        wl.close()
        pf.close()
        w = W.load_weights()
        h = W.shipped_head(w)
        W.save_head(d / "h.npz", h.arrays, h.class_names, w)
        pairs = {"both_strands": ({"both_strands": True}, {"both_strands": True, "head": d / "h.npz"}),
                 "window_stride_1000": ({"window_stride": 1000}, {"window_stride": 1000, "head": d / "h.npz"})}
        nnc.main(fa, d / "warm", False, 128, False, 8, False, False, both_strands=True, head=d / "h.npz")
        times = {}
        n = 0
        for rep in range(args.reps):
            for pair, (plain, with_head) in pairs.items():
                for name, kw in (("plain", plain), ("head", with_head)):
                    n += 1
                    t0 = time.perf_counter()
                    nnc.main(fa, d / f"run{n}", False, 128, False, 8, False, False, **kw)
                    times.setdefault(pair, {}).setdefault(name, []).append(time.perf_counter() - t0)
        res["module_s"] = {p: {k: statistics.median(v) for k, v in t.items()} for p, t in times.items()}
        res["module_s_all"] = times
        labels = d / "labels.tsv"
        labels.write_text("seq_name\tclass\n" + "".join(f"c{i}\t{'abc'[i % 3]}\n" for i in range(args.contigs)))
        train = {}
        for rep in range(args.reps):
            for name, both in (("forward", False), ("both_strands", True)):
                emb, epochs = timed_train(torch, train_head, nnc, fa, labels, d / f"train_{name}{rep}", both)
                train.setdefault(name, {"embed_s": [], "epoch_s": []})
                train[name]["embed_s"].append(emb)
                train[name]["epoch_s"].append(statistics.median(epochs))
        res["train_head_all"] = train
        res["train_head"] = {k: {m: statistics.median(v) for m, v in t.items()} for k, t in train.items()}
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "head_outputs_h100.json").write_text(json.dumps(res, indent=1, default=str) + "\n")
    m, t = res["module_s"], res["train_head"]
    md = [f"# Head strand and window outputs, and train-head --both-strands, on {res['card']}", "",
          "Measured by tools/head_outputs_throughput.py in one process; the card name and power limit above were read in the "
          f"same run.  Input: the {args.contigs:,} seeded contigs of tools/contig_throughput.py ({res['gbp']:.2f} Gbp, "
          f"{res['windows']:,} windows; {res['profile_windows_1000']:,} windows at stride 1000).  Medians of {args.reps} "
          "alternating runs; the head is the shipped classifier's tail saved as a head file (C = 3).", "",
          "| nn-classification | without --head (s) | with --head (s) | ratio |", "|---|---|---|---|"]
    for p, label in (("both_strands", "--both-strands"), ("window_stride_1000", "--window-stride 1000")):
        md.append(f"| {label} | {m[p]['plain']:.2f} | {m[p]['head']:.2f} | {m[p]['head'] / m[p]['plain']:.3f} |")
    md += ["", "| train-head (3 epochs, batch 256) | forward (s) | --both-strands (s) | ratio |", "|---|---|---|---|"]
    for k, label in (("embed_s", "embedding"), ("epoch_s", "per epoch")):
        md.append(f"| {label} | {t['forward'][k]:.2f} | {t['both_strands'][k]:.2f} | "
                  f"{t['both_strands'][k] / t['forward'][k]:.3f} |")
    md.append("")
    (out / "head_outputs_h100.md").write_text("\n".join(md))
    print("\n".join(md))


if __name__ == "__main__":
    main()
