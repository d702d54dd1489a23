"""
CPU check of the training step's softmax cross-entropy as head_softmax_xent_kernel computes it in float32 (restated by
head_ref.xent_fp32) against the fp64 statement head_ref.xent, over log-odds margins from -120 to 120.  Once a row is
classified confidently, p_y - 1 cancels in float32 (values just below 1 are 2^-24 apart) and log(sum e^(l - max)) rounds to
log(1 + a few ulps); the kernel takes the target component of dZ2 as -sum_{c != y} p_c and the loss from log1p of the sum
without the argmax, so both keep their relative precision.
"""
import numpy as np
import pytest

import head_ref as R

ULP = 2.0 ** -24
B = 256


def _sweep(C, n=4001, seed=0):
    """float32 logits [n, C] and labels: margin mu = l_y - max_{c != y} l_c from -120 to 120, the other classes 0..30 below
    the largest of them (two of them tied at it on every fifth row), a common shift.  All values are multiples of 2^-12
    below 2^9, so every difference the softmax forms is exact in float32 and the sweep measures the formula, not the rounding
    of its input."""
    rng = np.random.default_rng(seed + C)
    q = lambda v: np.round(v * 4096.0) / 4096.0                     # noqa: E731
    mu = q(np.linspace(-120.0, 120.0, n))
    y = rng.integers(0, C, n)
    shift = q(rng.uniform(-20.0, 20.0, n))
    lg = shift[:, None] - q(rng.uniform(0.0, 30.0, (n, C)))
    r = np.arange(n)
    top = (y + 1 + rng.integers(0, C - 1, n)) % C                    # the largest other class
    lg[r, top] = shift
    if C > 2:
        for i in r[::5]:
            lg[i, rng.choice([c for c in range(C) if c not in (y[i], top[i])])] = shift[i]
    lg[r, y] = shift + mu
    lg32 = lg.astype(np.float32)
    assert np.array_equal(lg32.astype(np.float64), lg)
    return lg32, y, mu


@pytest.mark.parametrize("C", [2, 7, 32])
def test_softmax_xent_fp32_over_the_margin_sweep(C):
    lg32, y, mu = _sweep(C)
    cw = np.random.default_rng(C).uniform(0.5, 25.0, C).astype(np.float32)
    nll, g = R.xent(lg32.astype(np.float64), y)
    w = cw.astype(np.float64)[y]
    ref_loss, ref_dz2 = w * nll, w[:, None] * g / B
    loss, dz2 = R.xent_fp32(lg32, y, cw, B)
    assert np.all(np.isfinite(loss)) and np.all(np.isfinite(dz2))
    # rows whose gradient is far enough above fp32's normal range that every term near its max is normal
    scale = np.abs(ref_dz2).max(axis=1)
    normal = np.abs(g).max(axis=1) >= 2.0 ** -100
    assert (mu[normal] > 60).any() and (mu[normal] < -60).any()
    err = np.abs(dz2 - ref_dz2).max(axis=1) / scale
    err_loss = np.abs(loss - ref_loss) / ref_loss
    print(f"\nC {C}: fixed formula: dZ2 {err[normal].max() / ULP:.2f} ulp of the row's max |g|, loss {err_loss[normal].max() / ULP:.2f}"
          f" ulp over {normal.sum()} rows (mu {mu[normal].min():.0f} .. {mu[normal].max():.0f})")
    # a component is exp, up to five butterfly additions, a quotient, the weight's product and the division by B (exact):
    # each rounds by at most an ulp of its value, which is at most the row's max |g|
    assert err[normal].max() <= 8 * ULP
    assert err_loss[normal].max() <= 8 * ULP
    # the formula before the fix, from the same float32 logits: cancels, so the sweep reaches the regime the fix is for
    old_loss, old_dz2 = R.xent_fp32_cancelling(lg32, y, cw, B)
    err_old = np.abs(old_dz2 - ref_dz2).max(axis=1) / scale
    err_old_loss = np.abs(old_loss - ref_loss) / ref_loss
    print(f"C {C}: p - onehot: worst {err_old[normal].max():.2e}, first mu above 1e-4: "
          f"{mu[normal & (err_old > 1e-4)].min():.1f}; loss worst {err_old_loss[normal].max():.2e}")
    assert err_old[normal].max() > 1e-4 and err_old_loss[normal].max() > 1e-4
    # from mu ~ 104 on every other e underflows: the row's loss and gradient are exactly 0, not NaN
    dead = mu >= 110
    assert dead.any() and np.all(loss[dead] == 0) and np.all(dz2[dead] == 0)


def test_fp64_reference_keeps_precision_past_p_equal_one():
    """head_ref.xent against closed forms at margins where p_y is exactly 1.0 in fp64: the loss and the target component
    are the sum of the other probabilities to fp64 relative precision, not 0."""
    mu = np.array([40.0, 80.0, 300.0, 700.0])
    lg = np.stack([mu, np.zeros_like(mu), -np.ones_like(mu)], axis=1)
    nll, g = R.xent(lg, np.zeros(4, int))
    other = np.exp(-mu) + np.exp(-mu - 1)                 # sum of the other e; p_y == 1.0 in fp64 on every row
    assert np.all(np.exp(-mu) / (1 + other) > 0)
    assert np.allclose(nll, np.log1p(other), rtol=1e-15, atol=0) and np.all(nll > 0)
    assert np.allclose(g[:, 0], -other / (1 + other), rtol=1e-15, atol=0)
    # a wrong label: nll = margin + log1p(...) and the gradient is p_y off the argmax, -sum of the others at the label
    nll, g = R.xent(lg, np.ones(4, int))
    assert np.allclose(nll, mu + np.log1p(other), rtol=1e-15)
    assert np.allclose(g[:, 1], -(1 + np.exp(-mu - 1)) / (1 + other), rtol=1e-15)
