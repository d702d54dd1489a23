"""
CPU checks of the derived per-step bounds of tests/novelty_ref.py, the bars the H100 tests (tests/test_gpu_novelty_steps.py)
hold the novelty fit and the window distances to.  Run with -s for the ratios.
  * Honest arithmetic stays within every bound: a NumPy fit in an order unlike the kernels' (pairwise class sums, a BLAS
    scatter, a column-oriented Cholesky, forward substitution and whitened means with the k order reversed, einsum distances)
    on rank-1, -8 and -64 rows, rows offset by 1e2 and 1e4, columns scaled from 1e-3 to 1e3, imbalanced classes, tiny N and the
    encoder's own embeddings of the golden windows.
  * Each bound catches the error it exists for: x - center in fp32 (which the older 1e-6 D + 1e-9 distance bar lets through),
    fp32 class sums, whitened means from fp32 class means, a distance accumulated in fp32, one skipped Cholesky update, an fp32
    Cholesky, a forward substitution without its k = j term, and a one-pass scatter E[xx^T] - mu mu^T on offset rows.
  * engine.novelty_scores on NaN and infinite distances, ties and novelty equal to a calibration value.
"""
from pathlib import Path

import numpy as np
import pytest

import novelty_ref as R
from genomad_b200 import engine

DIM = R.DIM


# --------------------------------------------------------------------------------------------------------------- inputs
def family(kind, seed=0):
    """(X float32 [N, 512], labels int32 [N], C) of one input family; every class has a row."""
    rng = np.random.default_rng(seed)

    def labels(N, C):
        y = np.concatenate([np.arange(C), rng.integers(0, C, N - C)]).astype(np.int32)
        rng.shuffle(y)
        return y

    if kind.startswith("rank"):                            # within-class scatter of rank k, class offsets
        k, N, C = int(kind[4:]), 2000, 3
        y = labels(N, C)
        X = rng.normal(0, 3, (C, DIM))[y] + rng.normal(0, 1, (N, k)) @ rng.normal(0, 1, (k, DIM))
    elif kind.startswith("offset"):                        # a common offset far above the unit spread
        off, N, C = float(kind[6:]), 3000, 3
        y = labels(N, C)
        X = off + rng.normal(0, 1, (C, DIM))[y] + rng.normal(0, 1, (N, DIM))
    elif kind == "spread20":                               # offset 20, per-column spreads 0.05 .. 2
        N, C = 4000, 3
        y = rng.integers(0, C, N).astype(np.int32)
        X = rng.normal(0, 1, (C, DIM))[y] + rng.normal(0, 1, (N, DIM)) * rng.uniform(0.05, 2, DIM) + 20.0
    elif kind == "colscale":                               # columns scaled from 1e-3 to 1e3
        N, C = 3000, 3
        y = labels(N, C)
        X = (rng.normal(0, 1, (C, DIM))[y] + rng.normal(0, 0.5, (N, DIM))) * 10.0 ** rng.uniform(-3, 3, DIM)
    elif kind == "imbalance":                              # one class at 99.9 %
        N, C = 4000, 3
        y = np.zeros(N, np.int32)
        y[rng.choice(N, 4, replace=False)] = [1, 1, 2, 2]
        X = rng.normal(0, 2, (C, DIM))[y] + rng.normal(0, 1, (N, DIM)) * rng.uniform(0.2, 2, DIM)
    elif kind == "onerow32":                               # C = 32, classes 24..31 with one row each
        N, C = 1500, 32
        y = rng.integers(0, 24, N).astype(np.int32)
        y[rng.choice(N, 8, replace=False)] = np.arange(24, 32)
        X = np.maximum(rng.normal(0, 1, (C, DIM))[y] + rng.normal(0, 1, (N, DIM)), 0)
    elif kind == "tiny":                                   # N = C + 1
        N, C = 6, 5
        y = labels(N, C)
        X = rng.normal(0, 1, (N, DIM))
    elif kind == "golden":                                 # the encoder's own embeddings of the 40 golden windows
        z = np.load(Path(__file__).parent / "golden" / "reference_encoder_golden.npz")
        X = np.concatenate([z["graph_shipped"], z["tokens_shipped"]])
        y = np.repeat(np.arange(2, dtype=np.int32), [len(z["graph_shipped"]), len(z["tokens_shipped"])])
        C = 2
    else:
        raise ValueError(kind)
    return np.asarray(X, np.float32), y, C


FAMILIES = ["rank1", "rank8", "rank64", "offset1e2", "offset1e4", "colscale", "imbalance", "onerow32", "tiny", "golden"]


# ---------------------------------------------------------------------------------------------- honest NumPy arithmetic
def honest_means(X, y, C):
    """Class means by pairwise sums (NumPy's reduction along a contiguous axis), the center from those class sums."""
    x = np.asarray(X, np.float64)
    sums = np.stack([np.ascontiguousarray(x[y == c].T).sum(1) for c in range(C)])
    counts = np.bincount(y, minlength=C)
    return sums / counts[:, None], sums.sum(0) / len(x)


def chol_columns(A):
    """Left-looking (column-oriented) Cholesky of the lower triangle of A -> (L, pivots before their square roots)."""
    L = np.zeros_like(A)
    piv = np.empty(DIM)
    for j in range(DIM):
        v = A[j:, j] - L[j:, :j] @ L[j, :j]
        piv[j] = v[0]
        L[j, j] = np.sqrt(v[0])
        L[j + 1:, j] = v[1:] / L[j, j]
    return L, piv


def inverse_reversed(L, drop_diag_term=False):
    """P = L^-1 by forward substitution row by row, each sum over k taken from k = i - 1 down to j.  drop_diag_term: the mutant
    that leaves out the k = j term."""
    P = np.zeros_like(L)
    for i in range(DIM):
        P[i, i] = 1.0 / L[i, i]
        if i:
            s = L[i, :i][::-1] @ P[:i, :i][::-1]
            if drop_diag_term:
                s = s - L[i, :i] * np.diagonal(P)[:i]
            P[i, :i] = -s / L[i, i]
    return P


def honest_fit(X, y, C):
    mu, center = honest_means(X, y, C)
    d = np.asarray(X, np.float64) - mu[y]
    S = d.T @ d / len(d)
    A, tr = R.shrink(S)
    L, piv = chol_columns(A)
    P = inverse_reversed(L)
    m = (mu - center)[:, ::-1] @ P.T[::-1]             # k descending
    return {"mu": mu, "center": center, "S": S, "A": A, "L": L, "min_pivot": piv.min(), "P": P, "m": m}


def honest_distances(x, center, P, m):
    """fp64 distances in einsum's own k order, stored as float32."""
    Y = np.einsum("nk,jk->nj", np.asarray(x, np.float64) - center, P, optimize=False)
    return np.stack([((Y - mc) ** 2)[:, ::-1].sum(1) / DIM for mc in m], 1).astype(np.float32)


def score_rows(X, y, C, fit, rng):
    """Rows to score: fit rows, rows equal to fp32(mu_c), the center, zeros, rows 1e3 times the scale, rows with one huge
    column."""
    scale = np.abs(X).max()
    huge = X[:C].astype(np.float64).copy()
    huge[np.arange(C), rng.integers(0, DIM, C)] = 1e6 * max(scale, 1)
    rows = [X[:500], fit["mu"].astype(np.float32), fit["center"][None].astype(np.float32), np.zeros((2, DIM), np.float32),
            (1e3 * X[rng.integers(0, len(X), 3)]).astype(np.float32), huge.astype(np.float32)]
    return np.concatenate(rows)


def kappa(A):
    return float(np.linalg.cond(A))


@pytest.fixture(scope="module")
def honest():
    cache = {}

    def get(kind):
        if kind not in cache:
            X, y, C = family(kind)
            cache[kind] = (X, y, C, honest_fit(X, y, C))
        return cache[kind]
    return get


# ------------------------------------------------------------------------------------------------ bounds hold for honest fits
@pytest.mark.parametrize("kind", FAMILIES)
def test_bounds_hold_for_honest_arithmetic(honest, kind):
    X, y, C, f = honest(kind)
    ref = R.fit(X, y, C)
    mu_bar, c_bar = R.sum_bar(X, y, C)
    assert (np.abs(f["mu"] - ref["mu"]) <= mu_bar).all() and (np.abs(f["center"] - ref["center"]) <= c_bar).all()
    assert (np.abs(f["S"] - ref["S"]) <= R.scatter_bar(ref, mu_bar)).all()
    ratios = {"chol": R.cholesky_ratio(f["L"], f["A"]), "pivot": R.pivot_ratio(f["min_pivot"], f["L"]),
              "inverse": R.inverse_ratio(f["L"], f["P"]), "means": R.whiten_ratio(f["P"], f["mu"], f["center"], f["m"])}
    rng = np.random.default_rng(1)
    x = score_rows(X, y, C, f, rng)
    D, bound = R.distance_bound(x, f["center"], f["P"], f["m"])
    got = honest_distances(x, f["center"], f["P"], f["m"])
    ratios["distance"] = R._ratio(np.abs(got - D), bound)
    # per-contig: consecutive runs of 1, 7 and 100 windows, one fp32 running sum each
    offsets = np.unique(np.minimum([0, 1, 8, 108, len(x)], len(x)))
    mean, cbound = R.contig_bound(D, bound, offsets)
    run = np.stack([np.cumsum(got[b:e], 0, dtype=np.float32)[-1] / np.float32(e - b) for b, e in zip(offsets[:-1], offsets[1:])])
    ratios["contig"] = R._ratio(np.abs(run - mean), cbound)
    k = kappa(f["A"])
    print(f"\n{kind}: N={len(X)} C={C} kappa(Sigma) {k:.4g}; error / bound " + ", ".join(f"{n} {v:.2g}" for n, v in ratios.items()))
    for name, v in ratios.items():
        assert v <= 1.0, f"{kind}: {name} at {v:.3g} of its bound"
    if kind == "rank1":
        assert abs(k / (1 + DIM * (1 - R.ALPHA) / R.ALPHA) - 1) < 0.01, f"rank 1: kappa {k:.5g} is not at the shrinkage's ceiling"


# ----------------------------------------------------------------------------------------------- bounds catch the mutants
def _report(name, ratio):
    print(f"\nmutant {name}: {ratio:.3g} x its bound")
    assert ratio > 1.0, f"the bound does not catch {name} ({ratio:.3g} of it)"


def test_fp32_subtraction_is_caught_and_passes_the_old_bar():
    X, y, C = family("spread20")
    f = R.fit(X, y, C)
    x = X[:500]
    D, bound = R.distance_bound(x, f["center"], f["P"], f["m"])
    a32 = (x - f["center"].astype(np.float32)).astype(np.float64)
    Y = a32 @ f["P"].T
    got = np.stack([((Y - mc) ** 2).sum(1) / DIM for mc in f["m"]], 1).astype(np.float32)
    err = np.abs(got - D)
    old = 1e-6 * D + 1e-9
    print(f"\nx - center in fp32 (kappa {kappa(f['Sigma']):.3g}): {(err / old).max():.3g} of the old 1e-6 D + 1e-9 bar")
    assert (err <= old).all(), "the old distance bar was expected to let this mutant through"
    _report("x - center in fp32", R._ratio(err, bound))


def test_fp32_class_sums_are_caught():
    X, y, C = family("offset1e2")
    mu_bar, _ = R.sum_bar(X, y, C)
    ref = R.fit(X, y, C)
    mu32 = np.stack([np.cumsum(X[y == c], 0, dtype=np.float32)[-1] / np.float32((y == c).sum()) for c in range(C)])
    _report("class sums in fp32", R._ratio(np.abs(mu32.astype(np.float64) - ref["mu"]), mu_bar))


def test_means_from_fp32_mu_are_caught(honest):
    X, y, C, f = honest("offset1e2")
    m = (f["mu"].astype(np.float32).astype(np.float64) - f["center"]) @ f["P"].T
    _report("m_c from fp32 mu", R.whiten_ratio(f["P"], f["mu"], f["center"], m))


def test_fp32_distance_accumulation_is_caught(honest):
    X, y, C, f = honest("rank64")
    x = X[:500]
    D, bound = R.distance_bound(x, f["center"], f["P"], f["m"])
    Y = (np.asarray(x, np.float64) - f["center"]) @ f["P"].T
    got = np.stack([np.cumsum(((Y - mc) ** 2).astype(np.float32), 1, dtype=np.float32)[:, -1] / np.float32(DIM)
                    for mc in f["m"]], 1)
    _report("distance accumulated in fp32", R._ratio(np.abs(got - D), bound))


def test_skipped_cholesky_update_is_caught(honest):
    X, y, C, f = honest("offset1e2")
    L, A = f["L"], f["A"]
    # skipping step 0's update of (i, j) factors A plus l_i0 l_j0 at (i, j): take the largest such term with i > j >= 1
    prod = np.tril(np.outer(L[:, 0], L[:, 0]), -1)
    prod[:, 0] = 0
    i, j = np.unravel_index(np.argmax(np.abs(prod)), prod.shape)
    E = np.zeros_like(A)
    E[i, j] = E[j, i] = prod[i, j]
    Lm = np.linalg.cholesky(A + E)
    _report(f"Cholesky update of ({i}, {j}) at k = 0 skipped", R.cholesky_ratio(Lm, A))


def test_fp32_cholesky_is_caught(honest):
    X, y, C, f = honest("golden")
    L32 = np.linalg.cholesky(f["A"].astype(np.float32)).astype(np.float64)
    _report("Cholesky in fp32", R.cholesky_ratio(L32, f["A"]))


def test_forward_substitution_without_the_diagonal_term_is_caught(honest):
    X, y, C, f = honest("colscale")
    _report("forward substitution without k = j", R.inverse_ratio(f["L"], inverse_reversed(f["L"], drop_diag_term=True)))


def test_one_pass_scatter_is_caught():
    X, y, C = family("offset1e4")
    ref = R.fit(X, y, C)
    mu_bar, _ = R.sum_bar(X, y, C)
    x = np.asarray(X, np.float64)
    S1 = sum(x[y == c].T @ x[y == c] - (y == c).sum() * np.outer(ref["mu"][c], ref["mu"][c]) for c in range(C)) / len(x)
    _report("one-pass scatter E[xx^T] - mu mu^T", R._ratio(np.abs(S1 - ref["S"]), R.scatter_bar(ref, mu_bar)))


# ------------------------------------------------------------------------------------------------ novelty_scores edges
def test_novelty_scores_follow_the_oracle_on_non_finite_distances_and_ties():
    cal = np.array([0.5, 1.0, 1.0, 2.0, 4.0], np.float32)
    inf, nan = np.inf, np.nan
    dist = np.array([[nan, 0.7], [0.7, nan], [inf, 0.3], [0.3, -inf], [inf, inf], [nan, nan],    # non-finite: NaN, -1, NaN
                     [1.0, 1.0], [2.0, 3.0], [4.0, 4.0], [4.5, 5.0], [0.2, 0.1], [1.0, 0.5]],     # ties, calibration values
                    np.float32)
    counts = np.array([2, 1, 3, 1, 4, 2, 1, 1, 2, 1, 1, 0])
    nov, nearest, p = engine.novelty_scores(dist, counts, cal)
    bad = ~np.isfinite(dist).all(1) | (counts == 0)
    assert np.isnan(nov[bad]).all() and (nearest[bad] == -1).all() and np.isnan(p[bad]).all()
    assert nearest[~bad].tolist() == [0, 0, 0, 0, 1]                     # ties: the lowest index
    assert np.array_equal(nov[~bad], np.array([1.0, 2.0, 4.0, 4.5, 0.1], np.float32))
    for i in range(len(dist)):
        r = R.p_value(nov[i], cal)
        assert (np.isnan(r) and np.isnan(p[i])) or r == p[i], (i, r, p[i])
    assert p[6] == 5 / 6 and p[7] == 3 / 6 and p[8] == 2 / 6 and p[9] == 1 / 6   # equal to a calibration value counts as >=


def test_non_finite_distances_are_written_as_na(tmp_path):
    from genomad_b200 import nn_classification as nnc
    dist = np.array([[np.nan, 1.0], [1.0, 2.0], [np.inf, 0.5], [1.0, 1.0]], np.float32)
    names = np.array(["a", "b", "c", "d"])
    nnc._write_head_novelty(tmp_path / "n.npz", tmp_path / "n.tsv", "contig_names", names, dist, np.array([3, 1, 2, 0]),
                            np.array([0.5, 2.0], np.float32), ("x", "y"), "0" * 64)
    lines = (tmp_path / "n.tsv").read_text().split("\n")
    assert lines[1:5] == ["a\tNA\tNA\tNA", "b\tx\t1\t0.666667", "c\tNA\tNA\tNA", "d\tNA\tNA\tNA"]
    z = np.load(tmp_path / "n.npz")
    assert z["nearest_class"].tolist() == [-1, 0, -1, -1] and np.isnan(z["p_value"][[0, 2, 3]]).all()
    assert z["distances"].tobytes() == dist.tobytes()
