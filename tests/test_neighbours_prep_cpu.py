"""
nb_prep_kernel's recipe on the CPU (tests/nb_prep_ref.py, an exact statement of the kernel's fp32 arithmetic): with the
power-of-two prescale, a row's TF32 halves are bitwise invariant under x -> x * 2^e while every entry stays a normal float, the
halves' dot product stays within 1e-6 of the fp64 cosine at every scale from 2^-140 to 2^100, and on rows of ordinary scale the
halves are bitwise those of the recipe without the prescale.  The recipe without it is kept on record: its sum of squares
overflows (the row becomes the zero row) or goes subnormal (the norm loses digits) at the scales asserted below.
"""
from fractions import Fraction

import numpy as np

import nb_prep_ref as P

F32 = np.float32
E_RANGE = range(-140, 101)
TINY = np.finfo(F32).tiny                       # 2^-126, the smallest normal float


def sparse_rows(n, seed):
    rng = np.random.default_rng(seed)
    return (np.maximum(rng.standard_normal((n, 512)), 0) * (rng.random((n, 512)) < 0.3)).astype(F32)


def signed_rows(n, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((n, 512)) * (rng.random((n, 512)) < 0.5)).astype(F32)


def one_hot_rows(n, seed):
    rng = np.random.default_rng(seed)
    x = np.zeros((n, 512), F32)
    x[np.arange(n), rng.integers(0, 512, n)] = rng.choice([-3.0, -1.0, 0.75, 1.0, 5.5], n)
    return x


def mixed_rows():
    return np.concatenate([sparse_rows(6, 1), signed_rows(6, 2), one_hot_rows(4, 3)])


def scaled(x, e):
    """x * 2^e rounded once to float32 per entry (the rows a user with data at that scale would pass); None if not finite."""
    y = x.astype(np.float64) * 2.0 ** e
    if np.abs(y).max() >= float(np.finfo(F32).max):
        return None
    return y.astype(F32)


def all_normal(x):
    a = np.abs(x)
    return bool(np.all((a == 0) | (a >= TINY)))


def cos64(a, b):
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    na, nb = np.linalg.norm(a64), np.linalg.norm(b64)
    return 0.0 if na == 0 or nb == 0 else float(a64 @ b64 / (na * nb))


def test_fma32_is_rounded_once():
    """fma32 against the exact rational a*b + c rounded once, on random operands and on float32 midpoints that a float64
    sum rounds onto (where rounding the float64 sum to float32 would be wrong)."""
    rng = np.random.default_rng(0)
    a = (rng.standard_normal(3000) * 2.0 ** rng.integers(-80, 60, 3000)).astype(F32)
    b = (rng.standard_normal(3000) * 2.0 ** rng.integers(-80, 60, 3000)).astype(F32)
    c = (rng.standard_normal(3000) * 2.0 ** rng.integers(-150, 120, 3000)).astype(F32)
    # midpoints: 2^60 + 2^37 + (2^36 - 2^-10) rounds down, 2^60 + (2^36 + 1) rounds up (2^36 + 1 = 4097 * 16773121)
    a = np.concatenate([a, [2.0 ** 18 * (1 + 2.0 ** -23), 4097.0, 2.0 ** -12]]).astype(F32)
    b = np.concatenate([b, [2.0 ** 18 * (1 - 2.0 ** -23), 16773121.0, 2.0 ** -12]]).astype(F32)
    c = np.concatenate([c, [2.0 ** 60 + 2.0 ** 37, 2.0 ** 60, 1.0]]).astype(F32)
    got = P.fma32(a, b, c)
    want = np.array([P.round32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)], F32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert got[-3] == F32(2.0 ** 60 + 2.0 ** 37) and got[-2] == F32(2.0 ** 60 + 2.0 ** 37) and got[-1] == F32(1.0)


def test_prescale_keeps_ordinary_rows_bitwise():
    """Rows of the scale of the encoder's embeddings: the prescale changes no bit of the halves."""
    x = np.concatenate([mixed_rows(), sparse_rows(64, 4) * F32(7.5), signed_rows(64, 5) * F32(0.01), np.zeros((2, 512), F32)])
    for h_new, h_old in zip(P.prep(x), P.prep(x, prescale_rows=False)):
        assert np.array_equal(h_new.view(np.uint32), h_old.view(np.uint32))


def test_halves_invariant_under_power_of_two_scaling():
    x = mixed_rows()
    base = P.prep(x)
    checked = 0
    for e in E_RANGE:
        xs = scaled(x, e)
        if xs is None:
            continue
        keep = [i for i in range(len(x)) if all_normal(xs[i])]
        if not keep:
            continue
        hi, lo = P.prep(xs[keep])
        assert np.array_equal(hi.view(np.uint32), base[0][keep].view(np.uint32)), f"e = {e}: hi"
        assert np.array_equal(lo.view(np.uint32), base[1][keep].view(np.uint32)), f"e = {e}: lo"
        checked += len(keep)
    assert checked > 200 * len(x)


def pairs():
    """Row pairs with cosines from -1 to 1: near-copies, a row and its negation, unrelated and signed rows."""
    rng = np.random.default_rng(8)
    a = np.concatenate([sparse_rows(4, 9), signed_rows(4, 10)])
    out = []
    for r in a:
        for rel in (1e-2, 1e-4):
            out.append((r, (r * (1 + rel * rng.standard_normal(512))).astype(F32)))
        out.append((r, -r))
    out += list(zip(sparse_rows(4, 11), sparse_rows(4, 12))) + list(zip(signed_rows(4, 13), signed_rows(4, 14)))
    return out


def test_similarity_against_fp64_at_every_scale():
    worst = 0.0
    for a, b in pairs():
        for e in E_RANGE:
            sa, sb = scaled(a, e), scaled(b, -e // 3)              # the two rows at different scales
            if sa is None or sb is None:
                continue
            hi, lo = P.prep(np.stack([sa, sb]))
            err = abs(P.similarity((hi[0], lo[0]), (hi[1], lo[1])) - cos64(sa, sb))
            worst = max(worst, err)
            assert err <= 1e-6, f"e = {e}: |s - cos64| = {err:.3e}"
    print(f"\nworst |(hi + lo) . (hi + lo) - cos64| over 2^-140 .. 2^100: {worst:.2e}")


def old_similarity(a, b, e):
    hi, lo = P.prep(np.stack([scaled(a, e), scaled(b, e)]), prescale_rows=False)
    return P.similarity((hi[0], lo[0]), (hi[1], lo[1]))


def test_unscaled_recipe_fails_at_extreme_scales():
    """What the recipe without the prescale returned on near-duplicate sparse rows (cos64 ~ 0.9999): the row squares overflow
    past 2^62 (norm inf, the zero row) and underflow below 2^-79 (norm 0, the zero row); in between the norm of subnormal
    squares is off by up to ~4x at 2^-76 and by 1e-5 at 2^-70.  Between 2^-62 and 2^60 it is bitwise the unscaled result."""
    rng = np.random.default_rng(15)
    rows = sparse_rows(8, 16)
    near = (rows * (1 + 1e-2 * rng.standard_normal(rows.shape))).astype(F32)
    at = {e: [] for e in (-80, -76, -72, -70, 62)}
    for a, b in zip(rows, near):
        c = cos64(a, b)
        s0 = old_similarity(a, b, 0)
        for e in (-62, -30, 30, 60):
            assert old_similarity(a, b, e) == s0
        for e in at:
            at[e].append(old_similarity(a, b, e) - c)
            hi, lo = P.prep(np.stack([scaled(a, e), scaled(b, e)]))   # the prescaled recipe at the same scale: no failure
            assert abs(P.similarity((hi[0], lo[0]), (hi[1], lo[1])) - c) <= 1e-6
    for e in (62, -80):                                             # the zero row: similarity 0
        assert all(abs(d + cos64(a, b)) < 1e-12 for d, a, b in zip(at[e], rows, near)), f"2^{e}"
    assert max(at[-76]) > 1.0                                       # s far above 1
    assert max(abs(d) for d in at[-72]) > 1e-4
    assert max(abs(d) for d in at[-70]) > 1e-5
