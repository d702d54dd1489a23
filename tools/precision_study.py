#!/usr/bin/env python
"""
Operand-precision study for the tensor-core stages (CPU emulation, fp64 accumulation).

Question: which operand formats can conv2/conv3 (K=768) and the w_v projection (K=128)
use on the tensor cores and still keep per-window |dp| <= 1e-4 against the fp32/fp64 oracle?
Each recipe rounds the MMA operands the way the kernel would and evaluates the rest of
the network in fp64.  Output: a markdown table on stdout.

    python tools/precision_study.py [n_windows]
"""
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import igloo_model as M, tokenizer as T  # noqa: E402


def tf32_rn(x):
    b = x.float().view(torch.int32)
    b = (b + 0x0FFF + ((b >> 13) & 1)) & ~0x1FFF
    return b.view(torch.float32).to(x.dtype)


def tf32_trunc(x):
    b = x.float().view(torch.int32) & ~0x1FFF
    return b.view(torch.float32).to(x.dtype)


def f16(x):
    return x.half().to(x.dtype)


def bf16(x):
    return x.bfloat16().to(x.dtype)


def split3(rnd):
    def fn(y, Wv):
        yh = rnd(y); yl = rnd(y - yh)
        wh = rnd(Wv); wl = rnd(Wv - wh)
        return yh @ wh + yl @ wh + yh @ wl
    return fn


def split2a(rnd):
    def fn(y, Wv):
        yh = rnd(y); yl = rnd(y - yh)
        wh = rnd(Wv)
        return yh @ wh + yl @ wh
    return fn


def single(rnd):
    return lambda y, Wv: rnd(y) @ rnd(Wv)


def make_windows(n, seed=0):
    rng = np.random.default_rng(seed)
    wins = []
    for i in range(n):
        kind = i % 8
        if kind == 0:   # iid uniform
            s = rng.integers(0, 4, 6000)
        elif kind == 1:  # GC-skewed
            p = rng.dirichlet([2, 2, 2, 2]); s = rng.choice(4, 6000, p=p)
        elif kind == 2:  # short tandem repeat
            u = rng.integers(0, 4, rng.integers(1, 12)); s = np.resize(u, 6000)
        elif kind == 3:  # N-padded tail
            s = rng.integers(0, 4, 6000)
        elif kind == 4:  # markov chain
            Tm = rng.dirichlet([0.5] * 4, size=4); s = np.zeros(6000, int)
            for t in range(1, 6000):
                s[t] = rng.choice(4, p=Tm[s[t - 1]])
        elif kind == 5:  # homopolymer runs
            s = np.repeat(rng.integers(0, 4, 600), rng.integers(1, 30, 600))[:6000]
            s = np.resize(s, 6000)
        elif kind == 6:  # N islands
            s = rng.integers(0, 4, 6000)
        else:
            s = rng.integers(0, 4, 6000)
        b = np.frombuffer(b"ACGT", np.uint8)[s].copy()
        if kind == 3:
            b[rng.integers(2500, 6000):] = ord("N")
        if kind == 6:
            for _ in range(rng.integers(1, 8)):
                a = rng.integers(0, 5990); b[a:a + rng.integers(1, 400)] = ord("N")
        wins.append(b)
    wins[0][:] = ord("A"); wins[1][:] = ord("N")
    return np.stack(wins)


RECIPES = {
    "fp32 everywhere":                 dict(dtype=torch.float32),
    "conv tf32-RN | wv fp64":          dict(round_a=tf32_rn, round_w=tf32_rn),
    "conv tf32-trunc | wv fp64":       dict(round_a=tf32_trunc, round_w=tf32_trunc),
    "conv f16 | wv fp64":              dict(round_a=f16, round_w=f16),
    "conv bf16 | wv fp64":             dict(round_a=bf16, round_w=bf16),
    "conv fp64 | wv tf32-RN 1pass":    dict(wv_fn=single(tf32_rn)),
    "conv fp64 | wv f16 1pass":        dict(wv_fn=single(f16)),
    "conv fp64 | wv f16 2pass(a)":     dict(wv_fn=split2a(f16)),
    "conv fp64 | wv f16 3pass":        dict(wv_fn=split3(f16)),
    "conv fp64 | wv bf16 3pass":       dict(wv_fn=split3(bf16)),
    "conv f16 | wv f16 3pass":         dict(round_a=f16, round_w=f16, wv_fn=split3(f16)),
    "conv f16 | wv f16 2pass(a)":      dict(round_a=f16, round_w=f16, wv_fn=split2a(f16)),
    "conv f16 | wv f16 1pass":         dict(round_a=f16, round_w=f16, wv_fn=single(f16)),
    "conv tf32-RN | wv tf32 3pass":    dict(round_a=tf32_rn, round_w=tf32_rn, wv_fn=split3(tf32_rn)),
    "conv bf16 | wv bf16 3pass":       dict(round_a=bf16, round_w=bf16, wv_fn=split3(bf16)),
}


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 256
    torch.set_num_threads(8)
    w = M.load_npz_weights(Path(__file__).resolve().parents[1] / "genomad_b200/data/nn_classifier.npz")
    wsyn = M.synthetic_igloo_weights(w)
    tok = T.tokenize_windows(make_windows(n))
    print(f"# precision study: {n} windows (8 families), errors are max |dp| over windows x 3 classes\n")
    for label, ww in (("shipped weights", w), ("synthetic O(1) IGLOO weights", wsyn)):
        ref = np.concatenate([M.forward(tok[i:i + 32], ww, torch.float64) for i in range(0, n, 32)])
        print(f"## {label}\n\n| recipe | max abs dp vs fp64 | p99.9 | argmax flips |\n|---|---|---|---|")
        for name, kw in RECIPES.items():
            kw = dict(kw); dt = kw.pop("dtype", torch.float64)
            t0 = time.time()
            out = np.concatenate([M.forward(tok[i:i + 32], ww, dt, **kw) for i in range(0, n, 32)])
            err = np.abs(out - ref)
            flips = int((out.argmax(1) != ref.argmax(1)).sum())
            print(f"| {name} | {err.max():.2e} | {np.quantile(err, 0.999):.2e} | {flips} |", flush=True)
        print()


if __name__ == "__main__":
    main()
