"""
How much the classifier's answers depend on the strand: seeded synthetic 6 kb windows, each scored and embedded on both strands.

Windows: `--uniform` of uniform base composition at GC evenly spread over 0.3-0.7, and `--skewed` with a G/C strand skew
(G - C) / (G + C) evenly spread over 0.1-0.3 at GC 0.5.  For each window and its reverse complement (the reference's rc()) it
reports max |p_f - p_r| over the three classes, whether the called class flips, and cos(e_f, e_r) of the encoder embeddings;
and, for scale, the cosine of pairs of unrelated forward windows.

    python tools/strand_agreement.py --device gpu [--uniform 8] [--skewed 4] [--seed 0] [--out FILE.json]   # the library, H100
    python tools/strand_agreement.py --device cpu ...                                                       # the fp64 oracle
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def make_windows(n_uniform: int, n_skewed: int, seed: int):
    rng = np.random.default_rng(seed)
    wins, kinds = [], []
    for gc in np.linspace(0.3, 0.7, n_uniform):
        p = np.array([(1 - gc) / 2, gc / 2, gc / 2, (1 - gc) / 2])          # A C G T
        wins.append(np.frombuffer(b"ACGT", np.uint8)[rng.choice(4, 6000, p=p)])
        kinds.append(f"uniform GC {gc:.2f}")
    for skew in np.linspace(0.1, 0.3, n_skewed):
        g, c = 0.25 * (1 + skew), 0.25 * (1 - skew)
        wins.append(np.frombuffer(b"ACGT", np.uint8)[rng.choice(4, 6000, p=[0.25, c, g, 0.25])])
        kinds.append(f"G/C skew {skew:.2f}")
    return np.stack(wins), kinds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--device", choices=("gpu", "cpu"), required=True)
    ap.add_argument("--uniform", type=int, default=8)
    ap.add_argument("--skewed", type=int, default=4)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", type=str, default="")
    a = ap.parse_args()

    import torch
    from genomad_b200 import sequence
    fwd, kinds = make_windows(a.uniform, a.skewed, a.seed)
    rev = np.stack([np.frombuffer(sequence.reverse_complement(w.tobytes()), np.uint8) for w in fwd])
    both = np.concatenate([fwd, rev])
    if a.device == "gpu":
        from genomad_b200 import engine
        clf = engine.Classifier(None, device=0, max_batch=64)
        p, e = clf.embed_ascii(torch.from_numpy(both).cuda())
        p, e = p.cpu().numpy().astype(np.float64), e.cpu().numpy().astype(np.float64)
        clf.close()
    else:
        import encoder_ref
        from oracle import igloo_model as M, tokenizer as T
        w = M.load_npz_weights(ROOT / "genomad_b200" / "data" / "nn_classifier.npz")
        tok = T.tokenize_windows(both)
        p = M.forward(tok, w, torch.float64)
        e = encoder_ref.encoder(tok, w, torch.float64)
    n = len(fwd)
    pf, pr, ef, er = p[:n], p[n:], e[:n], e[n:]

    def cos(x, y):
        return float(x @ y / max(np.linalg.norm(x) * np.linalg.norm(y), 1e-300))
    rows = [{"window": k, "max_abs_dp": round(float(np.abs(pf[i] - pr[i]).max()), 4),
             "call_forward": int(pf[i].argmax()), "call_reverse": int(pr[i].argmax()),
             "cos_fr": round(cos(ef[i], er[i]), 4)} for i, k in enumerate(kinds)]
    unrelated = [cos(ef[i], ef[j]) for i in range(n) for j in range(i + 1, n)]
    out = {"device": a.device, "seed": a.seed, "windows": rows,
           "median_max_abs_dp": round(float(np.median([r["max_abs_dp"] for r in rows])), 4),
           "largest_max_abs_dp": max(r["max_abs_dp"] for r in rows),
           "call_flips": sum(r["call_forward"] != r["call_reverse"] for r in rows),
           "median_cos_unrelated_forward": round(float(np.median(unrelated)), 4) if unrelated else None}
    if a.device == "gpu":
        sys.path.insert(0, str(ROOT / "tools"))
        from contig_throughput import card
        out["card"] = card()
    for r in rows:
        print(f"{r['window']:>18}  max|dp| {r['max_abs_dp']:.4f}  call {r['call_forward']}->{r['call_reverse']}  "
              f"cos {r['cos_fr']:.4f}")
    print(json.dumps({k: v for k, v in out.items() if k != "windows"}))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
