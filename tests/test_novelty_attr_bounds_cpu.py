"""
CPU checks of the seed bound of tests/novelty_attr_ref.py, the bar the H100 tests (tests/test_gpu_novelty_attr.py) hold the
GPU's g_h1 = dD_c / dh1 to.  Run with -s for the ratios.
  * Honest arithmetic stays within the bound: a NumPy gradient with every sum in another order, rounded to fp32 once, on
    models fitted to low-rank, offset, column-scaled and one-row-class rows and to the encoder's own embeddings of the golden
    windows, at typical rows (D ~ 1) and novel ones (D >> 1), for every target.
  * The bound catches the errors it exists for: r formed in fp32, and the i = j term dropped from P^T r.
"""
from pathlib import Path

import numpy as np
import pytest

import novelty_attr_ref as NA
import novelty_ref as R

DIM = R.DIM


def model(kind, seed=0):
    """(fit dict of novelty_ref.fit, rows float32 [n, 512] to score, C): typical rows from the fit's distribution and novel
    rows far from every class."""
    rng = np.random.default_rng(seed)
    if kind == "rank8":
        C, N = 3, 2000
        y = rng.integers(0, C, N)
        X = rng.normal(0, 3, (C, DIM))[y] + rng.normal(0, 1, (N, 8)) @ rng.normal(0, 1, (8, DIM))
    elif kind == "offset1e2":
        C, N = 3, 3000
        y = rng.integers(0, C, N)
        X = 100.0 + rng.normal(0, 1, (C, DIM))[y] + rng.normal(0, 1, (N, DIM))
    elif kind == "colscale":
        C, N = 7, 3000
        y = rng.integers(0, C, N)
        X = (rng.normal(0, 1, (C, DIM))[y] + rng.normal(0, 0.5, (N, DIM))) * 10.0 ** rng.uniform(-3, 3, DIM)
    elif kind == "onerow32":
        C, N = 32, 1500
        y = rng.integers(0, 24, N)
        y[rng.choice(N, 8, replace=False)] = np.arange(24, 32)
        X = np.maximum(rng.normal(0, 1, (C, DIM))[y] + rng.normal(0, 1, (N, DIM)), 0)
    elif kind == "golden":
        z = np.load(Path(__file__).parent / "golden" / "reference_encoder_golden.npz")
        X = np.concatenate([z["graph_shipped"], z["tokens_shipped"]])
        y = np.repeat(np.arange(2), [len(z["graph_shipped"]), len(z["tokens_shipped"])])
        C = 2
    else:
        raise ValueError(kind)
    X = np.asarray(X, np.float32)
    f = R.fit(X, y, C)
    typical = X[rng.choice(len(X), 12, replace=False)]
    spread = X.std(0) + 1e-3
    novel = (X.mean(0) + spread * rng.normal(0, 30, (12, DIM))).astype(np.float32)
    return f, np.concatenate([typical, novel]), C


KINDS = ["rank8", "offset1e2", "colscale", "onerow32", "golden"]


@pytest.fixture(scope="module")
def models():
    return {k: model(k) for k in KINDS}


@pytest.mark.parametrize("kind", KINDS)
def test_bound_holds_for_honest_arithmetic(models, kind):
    f, x, C = models[kind]
    D = R.distances(x, f["center"], f["P"], f["m"])
    assert np.median(D[:12].min(1)) < 10 and np.median(D[12:].min(1)) > 50, "typical and novel rows"
    worst = 0.0
    for c in range(C):
        tg = np.full(len(x), c)
        g, bound = NA.grad_bound(x, f["center"], f["P"], f["m"], tg)
        mine = NA.grad_other_order(x, f["center"], f["P"], f["m"], tg)
        worst = max(worst, NA.grad_ratio(mine, g, bound))
        # D_c is ||r||^2 / 512 and g its gradient: a central difference along g agrees
        r = NA.residual(x, f["center"], f["P"], f["m"], tg)
        assert np.allclose((r * r).sum(1) / DIM, D[:, c], rtol=1e-12, atol=0)
    print(f"\n{kind}: honest / bound {worst:.3f}", end="")
    assert worst <= 1.0


def test_gradient_is_the_derivative_of_the_distance(models):
    f, x, C = models["golden"]
    tg = np.arange(len(x)) % C
    g = NA.grad(x, f["center"], f["P"], f["m"], tg)
    rng = np.random.default_rng(3)
    v = rng.normal(0, 1, x.shape)
    h = 1e-4

    def D(z):
        r = NA.residual(z, f["center"], f["P"], f["m"], tg)
        return (r * r).sum(1) / DIM
    num = (D(x.astype(np.float64) + h * v) - D(x.astype(np.float64) - h * v)) / (2 * h)
    assert np.allclose(num, (g * v).sum(1), rtol=1e-6, atol=1e-9)


@pytest.mark.parametrize("kind", ["golden", "rank8", "colscale"])
def test_fp32_residual_is_caught(models, kind):
    f, x, C = models[kind]
    tg = np.zeros(len(x), int)
    g, bound = NA.grad_bound(x, f["center"], f["P"], f["m"], tg)
    ratio = NA.grad_ratio(NA.grad_fp32_residual(x, f["center"], f["P"], f["m"], tg), g, bound)
    print(f"\n{kind}: fp32 r / bound {ratio:.1f}", end="")
    assert ratio > 1.0


@pytest.mark.parametrize("kind", KINDS)
def test_dropped_diagonal_term_is_caught(models, kind):
    f, x, C = models[kind]
    tg = np.zeros(len(x), int)
    g, bound = NA.grad_bound(x, f["center"], f["P"], f["m"], tg)
    ratio = NA.grad_ratio(NA.grad_no_diagonal(x, f["center"], f["P"], f["m"], tg), g, bound)
    assert ratio > 1e3
