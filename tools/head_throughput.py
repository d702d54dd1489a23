"""
Cost of classifier-head training and of nn-classification --head on one GPU.

    python tools/head_throughput.py [--out profiles]

Writes <out>/head_training_h100.{md,json} with the card's name and power limit read in the same run:
  * training step time (CUDA events over 200 steps after 20 warm-up steps) at B = 256 and 1024, C = 3 and 32;
  * one epoch over 1 M cached windows (synthetic non-negative embeddings) at the defaults (B = 256, C = 3), and 10 epochs;
  * the encoder's embedding rate over 65,536 synthetic windows (synth.windows_torch), and the time that rate gives for 1 M;
  * nn-classification --head against --write-embeddings on the same seeded contigs: 2,000 contigs of 300 kb (100,000 windows),
    enough for the GPU work to outweigh the fixed costs of a call (wall clock, one process, best of two).
"""
import argparse
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


N_CONTIGS, CONTIG_NT = 2000, 300_000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def step_ms(torch, engine, W, X, labels, B, C, steps=200, warm=20):
    tr = engine.HeadTrainer(W.initial_head(C, 0), device=0, max_batch=B, seed=0)
    cw = torch.ones(C, dtype=torch.float32, device="cuda")
    lab = (labels % C).contiguous()
    idx = torch.randint(0, X.shape[0], (steps + warm, B), device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    for i in range(warm):
        tr.step(X, idx[i], lab, cw)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(steps):
        tr.step(X, idx[warm + i], lab, cw)
    b.record()
    b.synchronize()
    tr.close()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(ROOT / "profiles"))
    args = ap.parse_args()
    import torch
    from genomad_b200 import engine, nn_classification as nnc, synth, weights as W
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"card": card()}
    N = 1_000_000
    g = torch.Generator("cuda").manual_seed(1)
    X = torch.relu(torch.randn((N, 512), device="cuda", generator=g))
    labels = torch.randint(0, 32, (N,), device="cuda", generator=g, dtype=torch.int32)
    res["step_ms"] = {f"B={B},C={C}": step_ms(torch, engine, W, X, labels, B, C) for B in (256, 1024) for C in (3, 32)}
    tr = engine.HeadTrainer(W.initial_head(3, 0), device=0, max_batch=256, seed=0)
    lab3 = (labels % 3).contiguous()
    cw = torch.ones(3, dtype=torch.float32, device="cuda")
    order = torch.randperm(N, device="cuda", generator=g)
    tr.step(X, order[:256], lab3, cw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for s in range(0, N, 256):
        tr.step(X, order[s: s + 256], lab3, cw)
    tr.weights()
    res["epoch_1M_s"] = time.perf_counter() - t0
    res["ten_epochs_1M_s"] = 10 * res["epoch_1M_s"]
    tr.close()
    del X
    clf = engine.Classifier(None, device=0, max_batch=1024)
    n_emb = 65536
    win = synth.windows_torch(0, n_emb, 1, torch.device("cuda"))
    clf.embed_ascii(win[:1024])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for a in range(0, n_emb, 8192):
        clf.embed_ascii(win[a: a + 8192])
    torch.cuda.synchronize()
    rate = n_emb / (time.perf_counter() - t0)
    res["embed_windows_per_s"] = rate
    res["embed_1M_s_at_measured_rate"] = N / rate
    del win
    clf.close()
    # nn-classification --head against --write-embeddings on the same seeded contigs
    with tempfile.TemporaryDirectory() as d:
        d = Path(d)
        rng = np.random.default_rng(0)
        with open(d / "c.fna", "w") as f:
            for i in range(N_CONTIGS):
                f.write(f">c{i}\n" + np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, CONTIG_NT)].tobytes().decode() + "\n")
        w = W.load_weights()
        h = W.shipped_head(w)
        W.save_head(d / "h.npz", h.arrays, h.class_names, w)
        nnc.main(d / "c.fna", d / "warm", False, 128, False, 8, False, False, write_embeddings=True)
        times = {}
        for rep in range(2):
            for name, kw in (("write_embeddings", {"write_embeddings": True}), ("head", {"head": d / "h.npz"})):
                t0 = time.perf_counter()
                nnc.main(d / "c.fna", d / f"{name}{rep}", False, 128, False, 8, False, False, **kw)
                times.setdefault(name, []).append(time.perf_counter() - t0)
        res["module_s"] = {k: min(v) for k, v in times.items()}
        res["module_windows"] = N_CONTIGS * CONTIG_NT // 6000
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "head_training_h100.json").write_text(json.dumps(res, indent=1) + "\n")
    sm = res["step_ms"]
    md = [f"# Classifier-head training on {res['card']}", "",
          "Measured by tools/head_throughput.py in one run; the card name and power limit above were read in the same run.", "",
          "| training step | time (ms) |", "|---|---|"]
    md += [f"| {k} | {v:.4f} |" for k, v in sm.items()]
    md += ["", f"One epoch over 1,000,000 cached windows at the defaults (B = 256, C = 3): {res['epoch_1M_s']:.2f} s; "
               f"10 epochs: {res['ten_epochs_1M_s']:.1f} s.",
           f"Embedding rate of the encoder over 65,536 windows: {res['embed_windows_per_s']:.0f} windows/s, so 1,000,000 windows "
           f"take {res['embed_1M_s_at_measured_rate']:.1f} s (extrapolated from that rate, not timed at 1 M).",
           f"10 epochs cost {res['ten_epochs_1M_s'] / res['embed_1M_s_at_measured_rate']:.2f} x embedding the windows they train on.",
           "",
           f"nn-classification on {N_CONTIGS} seeded {CONTIG_NT // 1000} kb contigs ({res['module_windows']} windows), best of "
           f"two: --write-embeddings {res['module_s']['write_embeddings']:.2f} s, --head {res['module_s']['head']:.2f} s "
           f"({res['module_s']['head'] / res['module_s']['write_embeddings']:.2f}x).", ""]
    (out / "head_training_h100.md").write_text("\n".join(md))
    print("\n".join(md))


if __name__ == "__main__":
    main()
