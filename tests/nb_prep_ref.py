"""
An exact CPU statement of nb_prep_kernel (csrc/neighbours.cuh), bit for bit, with and without its power-of-two prescale.

One warp per 512-wide row; lane l holds the float4s l, l + 32, l + 64, l + 96, i.e. the entries 128 i + 4 l + c (i, c in 0..3):
  * prescale (the kernel's recipe): the row's max |x| m (a max butterfly: exact), E = ilogb(m), the row times 2^-E as one exact
    float factor, or 2^64 and then 2^(-E - 64) for a subnormal max (E < -127);
  * lane l sums the squares of its 16 entries in that order with fmaf, each rounded once to fp32;
  * xor butterfly 16, 8, 4, 2, 1 (ss += shfl_xor(ss, o): every lane ends with the same bits);
  * nrm = sqrtf(ss), y = x / nrm (IEEE fp32, round to nearest), or 0 when nrm == 0;
  * split_tf32 (logits_tc.cuh): hi = y with the low 13 mantissa bits cleared, lo = (y - hi) likewise.
prescale=False is the recipe before the prescale, kept to state what it got wrong on rows of extreme scale.
"""
from fractions import Fraction

import numpy as np

F32 = np.float32
_MASK = np.uint32(0xFFFFE000)


def fma32(a, b, c):
    """fmaf(a, b, c) elementwise on float32 arrays: a*b + c rounded once to float32.  a*b is exact in float64 (48 bits) and
    TwoSum makes p + c = s + err exactly; float32(s) is the correct rounding unless s is a float32 midpoint, where the sign of
    err breaks the tie."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    err = (p - (s - bb)) + (c64 - bb)
    with np.errstate(over="ignore"):
        r = s.astype(F32)
    r64 = r.astype(np.float64)
    other = np.where(s > r64, np.nextafter(r, F32(np.inf)), np.nextafter(r, F32(-np.inf)))
    with np.errstate(over="ignore", invalid="ignore"):
        mid = (r64 + other.astype(np.float64)) / 2
    tie = (s == mid) & (err != 0)
    return np.where(tie, np.where(err > 0, np.maximum(r, other), np.minimum(r, other)), r).astype(F32)


def round32(v: Fraction) -> F32:
    """A rational rounded once to float32 (nearest, ties to even): the plain statement fma32 is tested against."""
    r = F32(float(v))                                   # within one float32 step of the answer (double rounding)
    cands = {r, np.nextafter(r, F32(np.inf)), np.nextafter(r, F32(-np.inf))}
    best = None
    for c in sorted(cands, key=float):
        if not np.isfinite(c):
            continue
        d = abs(Fraction(float(c)) - v)
        even = int(np.array(c, F32).view(np.uint32)) & 1 == 0
        if best is None or d < best[0] or (d == best[0] and even):
            best = (d, c)
    return best[1]


def pow2(e):
    """2^e as float32, exactly, for integer arrays e in [-149, 127]."""
    return np.ldexp(F32(1), np.asarray(e, np.int32)).astype(F32)


def prescale(x):
    """The rows times 2^-E, E = ilogb(max |x|) per row (E = 0 for a zero row), as the kernel computes them."""
    x = np.asarray(x, F32)
    m = np.abs(x).max(axis=1)
    E = np.where(m > 0, np.frexp(m)[1] - 1, 0)           # frexp: m = f 2^e with f in [0.5, 1), also for subnormal m
    two = E < -127
    f0 = np.where(two, pow2(64), F32(1))[:, None]
    f1 = pow2(np.where(two, -E - 64, -E))[:, None]
    return (x * f0) * f1, E


def norms(y):
    """The kernel's fp32 norm of each row: per-lane fmaf sums in order, then the xor butterfly, then sqrtf."""
    n = y.shape[0]
    v = y.reshape(n, 4, 32, 4)
    ss = np.zeros((n, 32), F32)
    for i in range(4):
        for c in range(4):
            ss = fma32(v[:, i, :, c], v[:, i, :, c], ss)
    lane = np.arange(32)
    with np.errstate(over="ignore"):
        for o in (16, 8, 4, 2, 1):
            ss = (ss + ss[:, lane ^ o]).astype(F32)
    assert np.all(ss == ss[:, :1]) or np.all(np.isnan(ss))
    return np.sqrt(ss[:, 0]).astype(F32)


def split_tf32(y):
    y = np.ascontiguousarray(y, F32)
    hi = (y.view(np.uint32) & _MASK).view(F32)
    lo = (np.ascontiguousarray(y - hi).view(np.uint32) & _MASK).view(F32)
    return hi, lo


def prep(x, prescale_rows: bool = True):
    """(hi, lo) float32 [n, 512]: the halves nb_prep_kernel writes for the rows x (float32 [n, 512], finite)."""
    x = np.asarray(x, F32)
    assert x.ndim == 2 and x.shape[1] == 512
    y = prescale(x)[0] if prescale_rows else x
    nrm = norms(y)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(nrm[:, None] > 0, y / nrm[:, None], F32(0)).astype(F32)
    return split_tf32(q)


def similarity(a, b):
    """fp64 sum of (hi + lo)_a (hi + lo)_b over the halves of two rows: what the split-TF32 dot product approximates."""
    return float(np.dot(a[0].astype(np.float64) + a[1], b[0].astype(np.float64) + b[1]))
