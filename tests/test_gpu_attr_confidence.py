"""
Attributions across the confidence range on the H100 (run with `-m gpu -s` for the per-bin precision): every golden window,
every target, shipped and synthetic IGLOO weights, and head-sharpened weight sets, binned by the fp64 log-odds margin of the
target, mu = log p_c - max_{i != c} log p_i, against the fp64 autograd reference (tests/attr_ref.py) along the GPU forward's
routing, LeakyReLU branches and logits.  A window classified confidently as the target is the case attributions are most
wanted for, and the one where the head's gradient e_c - p would cancel (1 - p_c) in fp32.

    A  mu < 0         the target is not the argmax (p_c down to below fp32's range)     within 1e-4 of max |attr|
    B  0 <= mu < 9                                                                       within 1e-4
    C  9 <= mu < 17   p_c < 1.0f, 1 - p_c < 1e-4                                         within 1e-4
    D  17.5 <= mu < 40  p_c == 1.0f                                                      within 1e-4
    -  40 <= mu < 110  off-target p and the head's gradient leave fp32's normal range     finite, status clean
    E  mu >= 110      every off-target p is 0.0f                                         exactly 0, status clean

Why the logits too: in bins C and D the attributions scale as the off-target p_i ~ e^-mu, so an error d in the forward's
log-odds l_i - l_c moves all of them by the relative d.  The golden windows have logits up to ~176, where an fp32 forward
(the GPU's, or PyTorch's on the CPU) is off by ~1e-4, and by k times that with head-sharpened weights; that is the forward's
precision, not the backward's.  So the reference evaluates log p_c at the forward's logits (from its h2, in fp64), as it
follows the forward's max-pool and LeakyReLU branches; the error against fp64's own logits is printed and bounded by
1e-4 + 2 d, d the forward's log-odds error weighted by the off-target probabilities.

Head-sharpened sets multiply d2w and d2b by a power of two k: every logit is multiplied by k exactly, in fp32 as in fp64, and
h2, the routing and the LeakyReLU branches do not change.  They run on all windows on the GPU; the fp64 reference runs on
the rows listed for them, the ones that cover bins C, D and E.
"""
import time
from pathlib import Path

import numpy as np
import pytest
import torch

from genomad_b200 import engine
from oracle import igloo_model as M
from oracle import tokenizer as T
import attr_ref as A

pytestmark = pytest.mark.gpu

BAR = 1e-4
REF_ROWS = 8                # windows per fp64 autograd call
# (weights, k) -> golden rows checked against fp64; shipped row 16 / virus has mu 9.1, row 21 / plasmid 12.1, synthetic
# row 21 / plasmid 20.3: k = 2 puts the shipped ones in bin D, k = 4 takes row 21 to 48, k = 16 and k = 8 past 110
SHARPENED = {("shipped", 2): [16, 21], ("shipped", 4): [16, 21], ("shipped", 16): [], ("synthetic", 8): []}


@pytest.fixture(scope="module", autouse=True)
def _report_cost():
    t0 = time.time()
    yield
    print(f"\n{Path(__file__).name}: {time.time() - t0:.0f} s; peak torch allocation {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


@pytest.fixture(scope="module")
def weights(weights_npz):
    w = M.load_npz_weights(weights_npz)
    return {"shipped": w, "synthetic": M.synthetic_igloo_weights(w)}


@pytest.fixture(scope="module")
def golden(golden_dir):
    asc = np.load(golden_dir / "reference_graph_golden.npz")["windows"]
    return asc, T.tokenize_windows(asc)


def _sharpen(w, k):
    out = dict(w)
    out["d2w"] = w["d2w"] * np.float32(k)
    out["d2b"] = w["d2b"] * np.float32(k)
    return out


def _bin(mu):
    if mu < 0:
        return "A"
    if mu < 9:
        return "B"
    if mu < 17:
        return "C"
    if mu < 17.5:
        return "C/D"
    if mu < 40:
        return "D"
    return "-" if mu < 110 else "E"


def _margins(tok, w):
    """fp64 logits [n, 3] of the unchanged model and mu [n, 3] for every target"""
    with torch.no_grad():
        _, it = M.forward(tok, w, torch.float64, return_intermediates=True)
        lg = M.head(it["h0"], w, torch.float64, return_logits=True).numpy()
    mu = np.stack([lg[:, c] - np.delete(lg, c, axis=1).max(axis=1) for c in range(3)], axis=1)
    return lg, mu


def _gpu(w, asc):
    """probabilities, attributions per target, predict_ascii, and the forward's routing and LeakyReLU branches (all rows:
    the attribution chunk holds every window, so the debug buffers do too)"""
    n = len(asc)
    c = engine.Classifier(w, device=0, max_batch=n)
    try:
        c._attr_ctx(n)
        assert c.attr_max_batch >= n
        a = torch.from_numpy(asc).cuda()
        out = {}
        for target in range(3):
            probs, attr = c.attribute_ascii(a, target)
            c.check_status()
            out[target] = (probs.cpu().numpy(), attr.cpu().numpy())
        pred = c.predict_ascii(a).cpu().numpy()
        routes = [c.debug_fetch(f"route{s}", n).cpu().numpy() for s in (0, 1)]
        masks = [(c.debug_fetch(b, n) > 0).cpu().numpy() for b in ("attr_y1", "buf1", "buf0")]
        h2 = c.debug_fetch("h2", n).cpu().numpy().astype(np.float64)
        c.check_status()
    finally:
        c.close()
    logits = h2 @ w["d2w"].astype(np.float64) + w["d2b"].astype(np.float64)      # the forward's logits, from its h2
    return out, pred, routes, masks, logits


def _reference(tok, w, target, rows, routes, masks, logits=None):
    ref = []
    for i in range(0, len(rows), REF_ROWS):
        r = rows[i: i + REF_ROWS]
        ref.append(A.attribution(tok[r], w, target, routes=[x[r] for x in routes], masks=[m[r] for m in masks],
                                 logits_at=None if logits is None else logits[r]))
    return np.concatenate(ref)


def _error(got, ref):
    """per window max_t |got - ref| / max_t |ref|"""
    return np.abs(got.astype(np.float64) - ref).max(axis=1) / np.maximum(np.abs(ref).max(axis=1), 1e-300)


def test_attributions_across_the_confidence_range(weights, golden):
    asc, tok = golden
    n = len(asc)
    base = {v: _margins(tok, w) for v, w in weights.items()}
    sets = [(v, 1, list(range(n))) for v in weights] + [(v, k, rows) for (v, k), rows in SHARPENED.items()]
    cases = []                                   # (bin, set, row, target, mu, error or None)
    failures = []
    for variant, k, ref_rows in sets:
        w = weights[variant] if k == 1 else _sharpen(weights[variant], k)
        name = variant if k == 1 else f"{variant} x{k}"
        lg64, mu = base[variant][0] * k, base[variant][1] * k
        out, pred, routes, masks, logits = _gpu(w, asc)
        for target in range(3):
            probs, attr = out[target]
            assert np.array_equal(probs, pred), (name, target, "probabilities are not predict_ascii's")
            assert np.all(np.isfinite(attr)), (name, target)
            bins = [_bin(m) for m in mu[:, target]]
            # rows without a reference: the 40..110 gap (finite, checked above) and bin E
            for r in range(n):
                if bins[r] == "E":
                    assert np.all(np.delete(probs[r], target) == 0), (name, r, target, probs[r])
                    cases.append(("E", name, r, target, mu[r, target], None))
                    if not np.all(attr[r] == 0):
                        failures.append(f"{name} row {r} target {target}: bin E attributions not 0 "
                                        f"(max |attr| {np.abs(attr[r]).max():.2e})")
                elif bins[r] == "-":
                    cases.append(("-", name, r, target, mu[r, target], None))
            rows = [r for r in ref_rows if bins[r] not in ("-", "E")]
            if not rows:
                continue
            err = _error(attr[rows], _reference(tok, w, target, rows, routes, masks, logits))
            confident = [r for r in rows if bins[r] in ("C", "C/D", "D")]
            if confident:                                    # for the record: against fp64 at fp64's own logits
                err64 = dict(zip(confident, _error(attr[confident], _reference(tok, w, target, confident, routes, masks))))
            for r, e in zip(rows, err):
                b = bins[r]
                if b == "C":
                    assert probs[r, target] < 1.0, (name, r, target)
                if b == "D":
                    assert probs[r, target] == 1.0, (name, r, target)
                cases.append((b, name, r, target, mu[r, target], e))
                if r in confident:
                    # the forward's error in the log-odds l_i - l_c moves p_i, and its share of the attributions, by as
                    # much: weighted by the off-target p_i (a class at mu -248 does not count)
                    d = np.delete((logits[r] - logits[r, target]) - (lg64[r] - lg64[r, target]), target)
                    p_off = np.delete(np.exp(lg64[r] - lg64[r].max()), target)
                    d = float(np.abs(d) @ p_off / p_off.sum())
                    print(f"\n{name} row {r} target {target}: mu {mu[r, target]:.1f}, p_c {probs[r, target]!r}: "
                          f"{e:.2e} of max |attr| at the forward's logits; {err64[r]:.2e} at fp64's, the forward's "
                          f"log-odds off by {d:.1e}", end="")
                    if not err64[r] <= BAR + 2 * d:
                        failures.append(f"{name} row {r} target {target}: {err64[r]:.2e} at fp64's logits")
                if not e <= BAR:
                    failures.append(f"{name} row {r} target {target} (bin {b}, mu {mu[r, target]:.1f}): {e:.2e}")
    print()
    for b in ("A", "B", "C", "C/D", "D", "-", "E"):
        cs = [c for c in cases if c[0] == b]
        errs = [c for c in cs if c[5] is not None]
        if not cs:
            print(f"bin {b}: empty")
            continue
        worst = max(errs, key=lambda c: c[5]) if errs else None
        print(f"bin {b}: {len(cs)} cases, mu {min(c[4] for c in cs):.1f} .. {max(c[4] for c in cs):.1f}"
              + (f", worst {worst[5]:.2e} ({worst[1]} row {worst[2]} target {worst[3]})" if worst else ""))
    for b in ("A", "B", "C", "D", "-", "E"):
        assert any(c[0] == b for c in cases), f"bin {b} is empty"
    # bin A reaches p_c below fp32's range (shipped row 16, chromosome: p = 1.5e-108)
    assert any(c[0] == "A" and c[1] == "shipped" and c[2] == 16 and c[3] == 0 for c in cases)
    assert not failures, "\n".join(failures)
