#!/usr/bin/env python
"""
Parity sweep on the GPU box: N windows (default 10,240) from the 8 worst-case families of tools/precision_study.py plus the
counter-based config-2 stream, CUDA path (batch-1024 handle, through the C ABI) against the CPU oracle in fp32 -- with the
shipped weights and, on a smaller sample, with synthetic O(1) IGLOO weights (live patch gather / logits / softmax).
The oracle runs in a process pool (PyTorch's CPU conv does not scale past ~8-16 threads per process).

    python tools/parity_sweep.py [--n 10240] [--n-syn 2048] [--procs 16] [--out gpurun_out/r02_parity_sweep.md]

Writes a markdown report (histogram of |dp|, worst windows per family, argmax agreement).  The SURVEY (Appendix C) asked for
>= 10 k windows before freezing the numeric recipe; VERDICT r1 item 1(b).
"""
import argparse
import os
import sys
import time
from concurrent.futures import ProcessPoolExecutor
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

FAMILIES = ["iid uniform (window 0: all A)", "GC-skewed (window 1: all N)", "short tandem repeat", "N-padded tail", "Markov chain",
            "homopolymer runs", "N islands", "iid uniform (b)", "config-2 counter stream"]


def _oracle_chunk(args):
    a, synthetic, threads = args
    import torch
    torch.set_num_threads(threads)
    from oracle import igloo_model as M, tokenizer as T
    w = M.load_npz_weights(ROOT / "genomad_b200" / "data" / "nn_classifier.npz")
    if synthetic:
        w = M.synthetic_igloo_weights(w)
    tok = T.tokenize_windows(a)
    return np.concatenate([M.forward(tok[i:i + 16], w, torch.float32) for i in range(0, len(tok), 16)])


def oracle(a, synthetic, procs, threads):
    chunks = [a[i:i + 64] for i in range(0, len(a), 64)]
    with ProcessPoolExecutor(max_workers=procs) as ex:
        parts = list(ex.map(_oracle_chunk, [(c, synthetic, threads) for c in chunks]))
    return np.concatenate(parts)


def family_windows(n, seed):
    """The 8 families of tools/precision_study.py::make_windows, vectorised (its Markov family draws one symbol per Python
    call: minutes for thousands of windows).  Window i belongs to family i % 8."""
    rng = np.random.default_rng(seed)
    out = np.empty((n, 6000), np.uint8)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    for i in range(n):
        kind = i % 8
        if kind in (0, 3, 6, 7):
            s = rng.integers(0, 4, 6000)
        elif kind == 1:
            s = rng.choice(4, 6000, p=rng.dirichlet([2, 2, 2, 2]))
        elif kind == 2:
            s = np.resize(rng.integers(0, 4, rng.integers(1, 12)), 6000)
        elif kind == 4:                                    # first-order Markov chain by inverse-CDF lookup
            cdf = np.cumsum(rng.dirichlet([0.5] * 4, size=4), axis=1)
            u = rng.random(6000)
            s = np.zeros(6000, np.int64)
            for t in range(1, 6000):
                s[t] = min(3, int(np.searchsorted(cdf[s[t - 1]], u[t])))
        else:
            s = np.resize(np.repeat(rng.integers(0, 4, 600), rng.integers(1, 30, 600))[:6000], 6000)
        b = acgt[s].copy()
        if kind == 3:
            b[rng.integers(2500, 6000):] = ord("N")
        if kind == 6:
            for _ in range(rng.integers(1, 8)):
                a0 = rng.integers(0, 5990)
                b[a0:a0 + rng.integers(1, 400)] = ord("N")
        out[i] = b
    out[0] = ord("A")
    out[1] = ord("N")
    return out


def make_inputs(n, seed):
    from genomad_b200 import synth
    n_fam = n * 8 // 9 // 8 * 8
    fam = family_windows(n_fam, seed)
    fam_id = np.arange(n_fam) % 8
    idx = synth.subsample_indices(n - n_fam, 1_000_000, seed=seed + 1)
    cfg2 = synth.windows_numpy(idx, seed=1)
    return np.concatenate([fam, cfg2]), np.concatenate([fam_id, np.full(len(cfg2), 8)])


def report(title, p, ref, fam_id, lines):
    d = np.abs(p - ref).max(1)
    flips = int((p.argmax(1) != ref.argmax(1)).sum())
    edges = [0, 1e-7, 3e-7, 1e-6, 3e-6, 1e-5, 3e-5, 1e-4, 1]
    hist, _ = np.histogram(d, bins=edges)
    lines.append(f"## {title}\n")
    lines.append(f"windows: {len(d)}; max |dp| = **{d.max():.3e}** (bar 1e-4); mean {d.mean():.2e}; p99 {np.quantile(d, 0.99):.2e}; "
                 f"p99.9 {np.quantile(d, 0.999):.2e}; argmax flips: **{flips}**; rows summing to 1 within 1e-6: "
                 f"{int((np.abs(p.sum(1) - 1) < 1e-6).sum())}/{len(d)}\n")
    lines.append("| max abs dp per window in | " + " | ".join(f"[{a:g}, {b:g})" for a, b in zip(edges[:-1], edges[1:])) + " |")
    lines.append("|---|" + "---|" * (len(edges) - 1))
    lines.append("| windows | " + " | ".join(str(int(h)) for h in hist) + " |\n")
    lines.append("| family | windows | max abs dp | mean |")
    lines.append("|---|---|---|---|")
    for f, name in enumerate(FAMILIES):
        m = fam_id == f
        if m.any():
            lines.append(f"| {name} | {int(m.sum())} | {d[m].max():.2e} | {d[m].mean():.2e} |")
    lines.append("")
    return float(d.max()), flips


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10240)
    ap.add_argument("--n-syn", type=int, default=2048)
    ap.add_argument("--procs", type=int, default=0)
    ap.add_argument("--out", default=str(ROOT / "gpurun_out" / "r02_parity_sweep.md"))
    args = ap.parse_args()
    from oracle import igloo_model as M
    cores = len(os.sched_getaffinity(0))
    procs = args.procs or max(1, min(24, cores // 8))
    threads = max(1, min(8, cores // procs))
    lines = [f"# Parity sweep (round 2): CUDA path vs the fp32 CPU oracle\n",
             f"`python tools/parity_sweep.py --n {args.n} --n-syn {args.n_syn}` on 1 x H100; oracle on {procs} processes x {threads} torch "
             f"threads ({cores} host cores); CUDA path through `gnm_forward_ascii` with a max_batch = 1024 handle.  "
             "|dp| = max over the 3 classes of |p_cuda - p_oracle| per window.\n"]
    worst = 0.0
    shipped = M.load_npz_weights(ROOT / "genomad_b200" / "data" / "nn_classifier.npz")
    cases = ((f"Shipped weights, {args.n} windows", args.n, False, 2024),
             (f"Synthetic O(1) IGLOO weights (live gather / logits / softmax), {args.n_syn} windows", args.n_syn, True, 4048))
    prepared = []
    for title, n, synthetic, seed in cases:                 # all CPU work first: the pool forks before CUDA is initialised
        a, fam_id = make_inputs(n, seed)
        t0 = time.time()
        ref = oracle(a, synthetic, procs, threads)
        prepared.append((title, synthetic, a, fam_id, ref, time.time() - t0))
        print(f"oracle done: {title} in {prepared[-1][-1]:.1f} s", flush=True)
    import torch
    from genomad_b200 import engine
    for title, synthetic, a, fam_id, ref, t_cpu in prepared:
        w = M.synthetic_igloo_weights(shipped) if synthetic else shipped
        clf = engine.Classifier(w, device=0, max_batch=1024)
        t0 = time.time()
        p = clf.predict_ascii(torch.from_numpy(a).cuda()).cpu().numpy()
        clf.check_status()
        t_gpu = time.time() - t0
        clf.close()
        m, flips = report(title, p, ref, fam_id, lines)
        lines.append(f"(oracle: {t_cpu:.1f} s = {len(a) / t_cpu:.0f} windows/s on the host; CUDA path incl. H2D/D2H: {t_gpu:.2f} s)\n")
        worst = max(worst, m)
        print(f"{title}: max |dp| {m:.3e}, flips {flips}", flush=True)
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text("\n".join(lines))
    print("wrote", args.out)
    if worst > 1e-4:
        raise SystemExit(f"parity sweep FAILED: max |dp| = {worst:.3e} > 1e-4")


if __name__ == "__main__":
    main()
