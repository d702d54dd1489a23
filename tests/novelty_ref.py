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


# ------------------------------------------------------------------------------------------------- derived per-step bounds
# Each step of the fit is checked elementwise against its own computed inputs (the GPU's S, L, P, mu, center), with the
# standard a-priori bounds of Higham, "Accuracy and Stability of Numerical Algorithms" (2nd ed.).  They do not depend on
# kappa(Sigma), so a wrong small entry fails where a bar scaled by the largest entry would not.  |.| is elementwise.
U32 = 2.0 ** -24                   # fp32 unit roundoff
TINY32 = 2.0 ** -150               # half the smallest fp32 subnormal: the absolute rounding error of an fp32 store


def gamma(k, u=U):
    """gamma_k = k u / (1 - k u)."""
    return k * u / (1 - k * u)


def shrink(S):
    """(A, tr) as nv_factor_kernel forms them from S: tr S summed over k = 0..511 in that order (bitwise the kernel's), then
    A = (1 - alpha) S + alpha (tr / 512) I.  The kernel may contract the diagonal into an fma: A is within 2 u |A| of it."""
    S = np.asarray(S, np.float64)
    tr = 0.0
    for k in range(DIM):
        tr += float(S[k, k])
    A = (1.0 - ALPHA) * S
    A[np.diag_indices(DIM)] += ALPHA * (tr / DIM)
    return A, tr


def cholesky_ratio(L, A):
    """max |L L^T - A| / bound over the lower triangle, bound = 2 gamma_513 |L| |L^T| + 2 u |A| (Thm 10.3, gamma_{n+1} for the
    factorization, doubled for the host's own product; 2 u |A| for the shrinkage's fma)."""
    L = np.tril(np.asarray(L, np.float64))
    res = np.abs(L @ L.T - A)
    bound = 2 * gamma(DIM + 1) * (np.abs(L) @ np.abs(L).T) + 2 * U * np.abs(A)
    return _ratio(np.tril(res), np.tril(bound))


def pivot_ratio(min_pivot, L):
    """|min_pivot - min diag(L)^2| / (4 u min_pivot): the pivot is what the kernel took the square root of."""
    d2 = np.diagonal(np.asarray(L, np.float64)) ** 2
    return abs(min_pivot - d2.min()) / (4 * U * min_pivot)


def inverse_ratio(L, P):
    """max |L P - I| / (2 gamma_512 |L| |P|) (Thm 8.5 per column, doubled for the host's product)."""
    L, P = np.tril(np.asarray(L, np.float64)), np.asarray(P, np.float64)
    res = np.abs(L @ P - np.eye(DIM))
    return _ratio(res, 2 * gamma(DIM) * (np.abs(L) @ np.abs(P)))


def whiten_ratio(P, mu, center, m):
    """max |m_c - P (mu_c - center)| / (2 gamma_513 |P| |mu_c - center|): the device's and the host's fp64 products."""
    dm = np.asarray(mu, np.float64) - np.asarray(center, np.float64)
    P = np.asarray(P, np.float64)
    res = np.abs(np.asarray(m) - dm @ P.T)
    return _ratio(res, 2 * gamma(DIM + 1) * (np.abs(dm) @ np.abs(P).T))


def distance_bound(x, center, P, m):
    """(D [n, C], bound [n, C]) for the window distances of the stored model (center, P, m): D from the fp64 oracle, and a bound
    on |D_device - D| for a device that computes in fp64 and stores fp32.  With a = |x - center|, dY = gamma_514 |P| a (the
    error of one fp64 Y = P (x - center)), r = |Y - m_c|:
      fp64 = [sum_j (2 r_j dY_j + dY_j^2) + gamma_513 sum_j (r_j + dY_j)^2] / 512 + u D,
    doubled because the oracle is an fp64 computation too, then 2^-24 of the value for the fp32 store and 2^-150 absolute."""
    x = np.asarray(x, np.float64)
    center, P, m = np.asarray(center, np.float64), np.asarray(P, np.float64), np.asarray(m, np.float64)
    a = x - center
    Y = a @ P.T
    dY = gamma(DIM + 2) * (np.abs(a) @ np.abs(P).T)
    D = np.empty((len(x), len(m)))
    bound = np.empty_like(D)
    for c in range(len(m)):
        r = np.abs(Y - m[c])
        D[:, c] = (r * r).sum(1) / DIM
        b64 = ((2 * r * dY + dY * dY).sum(1) + gamma(DIM + 1) * ((r + dY) ** 2).sum(1)) / DIM + U * D[:, c]
        bound[:, c] = 2 * b64 + U32 * (D[:, c] + 2 * b64) + TINY32
    return D, bound


def contig_bound(D, bound, offsets):
    """Per-contig (mean [k, C], bound [k, C]) of window distances D with window bounds `bound` over the windows
    offsets[i]:offsets[i+1], for the head reducer (one fp32 running sum in window order, then / n in fp32): the windows'
    bounds, gamma_n (fp32) of the summed magnitudes for the running sum (n rather than n - 1 also covers this fp64 mean), and
    2^-24 of the mean for the division."""
    offsets = np.asarray(offsets)
    k = len(offsets) - 1
    mean, out = np.full((k, D.shape[1]), np.nan), np.full((k, D.shape[1]), np.nan)
    for i in range(k):
        b, e = int(offsets[i]), int(offsets[i + 1])
        if e == b:
            continue
        n = e - b
        mean[i] = D[b:e].sum(0) / n
        tot = bound[b:e].sum(0) + gamma(n, U32) * np.abs(D[b:e]).sum(0) + bound[b:e].sum(0) * gamma(n, U32)
        out[i] = tot / n + U32 * (np.abs(mean[i]) + tot / n) + TINY32
    return mean, out


def _ratio(err, bound):
    """max err / bound, with 0 / 0 read as 0."""
    err, bound = np.asarray(err), np.asarray(bound)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(r.max())
