"""
fp64 NumPy oracle of the head novelty model (include/gnm.h, DESIGN.md "Head novelty"), stated independently of the kernels:
class means and center, the two-pass tied within-class scatter S, shrinkage, Cholesky whitening, whitened class means, window
distances and the conformal p-value.  Also the error bars the H100 tests hold the kernels to.
"""
import numpy as np

DIM = 512
ALPHA = 0.01
U = 2.0 ** -53                     # fp64 unit roundoff


def fit(X, labels, C):
    """X float32 [N, 512] (the fit rows), labels int [N] in [0, C) -> dict of fp64 arrays: mu [C, 512], center [512], S, Sigma,
    L, P [512, 512], m [C, 512] (= P (mu_c - center)), counts [C]."""
    x = np.asarray(X, np.float64)
    y = np.asarray(labels, np.int64)
    counts = np.bincount(y, minlength=C)
    if (counts == 0).any():
        raise ValueError(f"class {int(np.flatnonzero(counts == 0)[0])} has no fit row")
    mu = np.stack([x[y == c].sum(0) / counts[c] for c in range(C)])
    center = np.stack([x[y == c].sum(0) for c in range(C)]).sum(0) / len(x)
    d = x - mu[y]
    S = d.T @ d / len(x)
    tr = np.trace(S)
    if not tr > 0:
        raise ValueError("the training windows have no within-class variation")
    Sigma = (1 - ALPHA) * S + ALPHA * (tr / DIM) * np.eye(DIM)
    L = np.linalg.cholesky(Sigma)
    P = np.linalg.solve(L, np.eye(DIM))
    P = np.tril(P)
    m = (mu - center) @ P.T
    return {"mu": mu, "center": center, "S": S, "Sigma": Sigma, "L": L, "P": P, "m": m, "counts": counts, "d": d}


def distances(x, center, P, m):
    """Window distances D [n, C] = || P (x - center) - m_c ||^2 / 512 in fp64."""
    y = (np.asarray(x, np.float64) - center) @ np.asarray(P).T
    return ((y[:, None, :] - np.asarray(m)[None]) ** 2).sum(-1) / DIM


def p_value(novelty, calibration):
    """(1 + #{v in calibration : v >= novelty}) / (1 + |calibration|), one value at a time; NaN stays NaN."""
    if np.isnan(novelty):
        return np.nan
    cal = np.asarray(calibration, np.float32)
    return (1.0 + float(np.sum(cal >= np.float32(novelty)))) / (1.0 + len(cal))


# ---------------------------------------------------------------------------------------------------------------------- bars
def sum_bar(X, labels, C):
    """Per (class, column) bound on a fixed-order fp64 class mean against the oracle's: both are sums of N_c terms, each within
    N_c u sum |x| of the exact sum, so |mu_gpu - mu_ref| <= 2 N_c u sum|x| / N_c (+ the division's rounding).  The center's
    bar is the same with N."""
    x = np.abs(np.asarray(X, np.float64))
    y = np.asarray(labels)
    mu = np.stack([2 * (np.sum(y == c) + 2) * U * x[y == c].sum(0) / max(1, np.sum(y == c)) for c in range(C)])
    center = 2 * (len(x) + C + 2) * U * x.sum(0) / len(x)
    return mu, center


def scatter_bar(ref, mu_err):
    """Bound on |S_gpu - S_ref|: the sums of N products d_i d_j in two fixed orders, 2 (N + 1) u (|d|^T |d|) / N, plus the
    centering difference from the class means' bar (|d_i| |dmu_j| + |dmu_i| |d_j|, summed, / N)."""
    d = np.abs(ref["d"])
    N = len(d)
    base = 2 * (N + 2) * U * (d.T @ d) / N
    e = np.abs(mu_err)
    return base + 2 * (d.T @ np.ones((N, 1))) / N * e.max(0)[None, :] + 2 * e.max(0)[:, None] * (np.ones((1, N)) @ d) / N


def whitening_bar(ref, N):
    """Elementwise bound on P and m from the condition number of Sigma: a backward-stable Cholesky and triangular inverse give
    a relative error of order kappa(Sigma) n u in P, and S itself carries (N + n) u relative; the constant 64 covers the
    growth factors of both steps.  Returns (P bar, m bar)."""
    kappa = np.linalg.cond(ref["Sigma"])
    rel = 64 * kappa * (DIM + N) * U
    P = rel * np.abs(ref["P"]).max()
    m = rel * (np.abs(ref["P"]) @ np.abs(ref["mu"] - ref["center"]).T).T.max() + rel * np.abs(ref["m"]).max()
    return P, m
