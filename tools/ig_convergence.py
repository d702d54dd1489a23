"""
Convergence of integrated gradients in fp64, on the CPU (no GPU): the completeness gap

    gap = | sum_t IG[t] - (log p_c(x) - log p_c(x')) |

of the midpoint rule at m in {4, 8, 16, 32, 64, 128}, for both baselines, every target, on golden windows, with the shipped
weights, the synthetic IGLOO weights and the head-sharpened sets of tests/test_gpu_attr_confidence.py (d2w, d2b times k).  The
gap is the quadrature error alone: the reference is exact up to fp64 rounding.  Each row's three logit gradients are taken once
(tests/ig_ref.py) and combined per target and head scale.

    python tools/ig_convergence.py [--rows 0,1,16,21] [--weights shipped,synthetic] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

STEPS = (4, 8, 16, 32, 64, 128)
SHARPENED = {"shipped": (1, 2, 4, 16), "synthetic": (1, 8)}       # head scales k per weight set (k = 1: the set itself)


def main():
    import ig_ref as I
    from oracle import igloo_model as M, tokenizer as T
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="0,1,16,21", help="golden windows (tests/golden/reference_graph_golden.npz)")
    ap.add_argument("--weights", default="shipped,synthetic", help="weight sets (each with its head-sharpened variants)")
    ap.add_argument("--out", type=Path, default=None)
    args = ap.parse_args()
    rows = [int(r) for r in args.rows.split(",")]
    asc = np.load(ROOT / "tests" / "golden" / "reference_graph_golden.npz")["windows"][rows]
    tok = T.tokenize_windows(asc)
    base = M.load_npz_weights(ROOT / "genomad_b200" / "data" / "nn_classifier.npz")
    sets = {"shipped": base, "synthetic": M.synthetic_igloo_weights(base)}
    out = {"rows": rows, "steps": list(STEPS), "cases": []}
    t0 = time.time()
    for name, w in ((k, sets[k]) for k in args.weights.split(",")):
        for baseline in I.BASELINES:
            lx, lb = I.endpoint_logits(tok, w, baseline)
            for m in STEPS:
                B = len(tok)
                lg, J = I.logit_jacobian(np.repeat(tok, m, axis=0), w, np.tile(I.alphas(m), B), baseline)
                for k in SHARPENED[name]:
                    for c in range(3):
                        rws = I.rows_from_jacobian(lg, J, c, scale=k).reshape(B, m, -1)
                        ig_sum = rws.mean(axis=1).sum(axis=1)
                        delta = I.log_p(lx, c, k) - I.log_p(lb[None], c, k)[0]
                        mu = k * (lx[:, c] - np.delete(lx, c, axis=1).max(axis=1))
                        for i, r in enumerate(rows):
                            out["cases"].append({"weights": name, "k": k, "baseline": baseline, "steps": m, "row": r,
                                                 "target": c, "mu": float(mu[i]), "delta": float(delta[i]),
                                                 "ig_sum": float(ig_sum[i]), "gap": float(abs(ig_sum[i] - delta[i])),
                                                 "mean_row_max": float(np.abs(rws[i]).max(axis=1).mean())})
                print(f"{name} {baseline} m={m}: {time.time() - t0:.0f} s", flush=True)
    # summary: worst gap per (set, baseline, m), absolute and relative to |delta|
    summ = {}
    for cs in out["cases"]:
        key = f"{cs['weights']} x{cs['k']} {cs['baseline']}"
        s = summ.setdefault(key, {})
        e = s.setdefault(str(cs["steps"]), {"gap": 0.0, "rel": 0.0})
        e["gap"] = max(e["gap"], cs["gap"])
        e["rel"] = max(e["rel"], cs["gap"] / max(abs(cs["delta"]), 1e-300))
    out["worst"] = summ
    print("worst |sum IG - delta log p| (relative to |delta|) per m:")
    for key, s in summ.items():
        print(f"  {key:24s} " + "  ".join(f"m={m}: {s[str(m)]['gap']:.1e} ({s[str(m)]['rel']:.1e})" for m in STEPS))
    if args.out:
        args.out.write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
