"""
CPU checks of the references that tests/test_gpu_head_inference.py holds gnm_head_forward to (tests/head_ref.py):
  * fold_bound covers the gap between the folded head (fold_bn's float32 scale / shift) and the exact head across BN regimes:
    moving mean / moving std up to 10^3, moving variance 0 .. 10^4, gamma 2^-10 .. 2^10;
  * kernel_bound covers a NumPy emulation of both routes (the TF32 three-pass product with bit masks on float32 views, and the
    FFMA chain) on embedding-like rows and on arbitrary rows (signs, zeros, 2^+-20 scales, TF32-exact values, subnormal lo
    halves), is not loose by more than 100x at dense_1 on typical rows of the tensor-core route, and fails an emulation that
    drops the xl wh pass;
  * the head weight checks of weights._check_head_arrays and of the C API (gnm_head_train_create shares gnm_head_create's).
Run with -s for the ratios.
"""
import ctypes as C
import re

import numpy as np
import pytest

import head_ref as R
from genomad_b200 import weights as W

LN = np.log


def embedding_rows(n, seed):
    """Non-negative rows with a large common component, like the encoder's ReLU outputs."""
    rng = np.random.default_rng(seed)
    common = rng.uniform(0.2, 1.5, 512)
    return np.maximum(common * rng.uniform(0.5, 1.5, (n, 1)) + rng.normal(0, 0.6, (n, 512)), 0).astype(np.float32)


def arbitrary_rows(seed):
    """Rows Head.predict accepts but the encoder never writes."""
    rng = np.random.default_rng(seed)
    g = rng.normal(0, 1, (6, 512)).astype(np.float32)
    rows = [g[0], np.zeros(512, np.float32), np.where(rng.random(512) < 0.5, 0, g[1]).astype(np.float32),
            g[2] * np.float32(2.0 ** 20), g[3] * np.float32(2.0 ** -20)]
    rows.append(R.split_tf32(g[4])[0])                                  # TF32-exact: lo == 0
    k = rng.integers(1, 1024, 512).astype(np.float64)
    sub = (2.0 ** -115 + k * 2.0 ** -135).astype(np.float32)             # hi = 2^-115, lo = k 2^-135: subnormal
    rows.append(np.where(rng.random(512) < 0.5, sub, g[5]).astype(np.float32))
    rows.append(-np.abs(g[5]))
    return np.stack(rows)


def test_split_tf32_halves():
    x = np.concatenate([embedding_rows(4, 0).ravel(), arbitrary_rows(1).ravel()])
    hi, lo = R.split_tf32(x)
    for v in (hi, lo):
        assert not (v.view(np.uint32) & np.uint32(0x1FFF)).any()
    r = x.astype(np.float64) - hi - lo
    assert (np.abs(r) <= np.abs(x.astype(np.float64)) * 2.0 ** -21).all()
    _, lo_sub = R.split_tf32(arbitrary_rows(1)[6])
    assert ((lo_sub != 0) & (np.abs(lo_sub) < 2.0 ** -126)).any(), "the subnormal-lo row has no subnormal lo half"
    assert not R.split_tf32(arbitrary_rows(1)[5])[1].any()


REGIMES = [dict(ratio=r) for r in (0, 10, 100, 1000)] + [dict(var=v, ratio=10) for v in (0, 1e-6, 1, 1e4)] + \
          [dict(gamma_log2=(-10, 10))]


@pytest.mark.parametrize("regime", REGIMES, ids=lambda r: ",".join(f"{k}={v}" for k, v in r.items()))
def test_fold_error_is_within_its_derived_bound(regime):
    X = embedding_rows(256, 2)
    a = R.bn_regime_head(X, 6, 3, **regime)
    gap = np.abs(R.folded(a, X)["logits"] - R.logits_exact(a, X))
    bound = R.fold_bound(a, X)
    l = np.abs(R.logits_exact(a, X))
    print(f"{regime}: fold gap max {gap.max():.3e} (|logit| median {np.median(l):.2f}), gap / bound max {(gap / bound).max():.3f}")
    assert (gap <= bound).all()


def _looseness(err, bound):
    """median over rows of bound / err at each row's worst element"""
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.nan_to_num(err / bound).max(1)
    return float(np.median(1 / q[q > 0])) if (q > 0).any() else np.inf


@pytest.mark.parametrize("route", ["tc", "ffma"])
@pytest.mark.parametrize("C", [2, 7, 32])
def test_emulated_kernels_are_within_the_kernel_bound(route, C):
    X = np.concatenate([embedding_rows(48, C), arbitrary_rows(C)])
    for name, a in (("random", R.random_head(C, 10 + C)), ("ratio=100", R.bn_regime_head(X[:48], C, C, ratio=100))):
        b = R.kernel_bound(a, X, route)
        e = R.emulate_forward(a, X, route)
        ref = b["ref"]
        out = []
        for k, bk in (("z", "dz"), ("y", "dy"), ("logits", "dl")):
            err = np.abs(e[k].astype(np.float64) - ref[k])
            assert (err <= b[bk]).all(), (name, k, float((err / b[bk]).max()))
            out.append(f"{k} max err/bound {(err / b[bk]).max():.3f} looseness {_looseness(err, b[bk]):.0f}x")
        logp = R.log_softmax(e["logits"].astype(np.float64))
        normal = ref["logp"] >= LN(2.0 ** -126)
        q = np.abs(logp - ref["logp"])[normal] / b["dlogp"][normal]
        assert (q <= 1).all()
        print(f"{route} C={C} {name}: " + "; ".join(out) + f"; log p max err/bound {q.max():.2e}")
        if route == "tc":
            typical = _looseness(np.abs(e["z"].astype(np.float64) - ref["z"])[:48], b["dz"][:48])
            assert typical <= 100, f"dense_1 bound {typical:.0f}x looser than the emulated error on typical rows"


def test_bound_catches_a_dropped_correction_pass():
    X = embedding_rows(32, 5)
    a = R.random_head(7, 17)
    b = R.kernel_bound(a, X, "tc")
    m = R.emulate_forward(a, X, "tc", drop_pass=True)
    q = (np.abs(m["z"].astype(np.float64) - b["ref"]["z"]) / b["dz"]).max()
    print(f"without the xl wh pass: dense_1 err / bound {q:.1f}")
    assert q > 2


# ------------------------------------------------------------------------------------------------ head weight checks
def _arrays(C=4):
    return {k: v.copy() for k, v in R.random_head(C, 1).items()}


@pytest.mark.parametrize("key,value,message", [
    ("d1w", np.nan, "not all finite"), ("bn1m", np.inf, "not all finite"), ("d2b", -np.inf, "not all finite"),
    ("bn1v", -1e-3, "moving variance \\+ 1e-3 must be > 0 \\(unit 7\\)"),
    ("bn1v", -2.0, "moving variance \\+ 1e-3 must be > 0 \\(unit 7\\)")])
def test_check_head_arrays_refuses_unusable_weights(key, value, message):
    a = _arrays()
    a[key].reshape(-1)[3 if key == "d2b" else 7] = value
    path = W.KEYS[key][0]
    with pytest.raises(ValueError, match=f"^{path}: {message}"):
        W._check_head_arrays(a, 4)


def test_check_head_arrays_accepts_zero_variance():
    a = _arrays()
    a["bn1v"][:] = 0
    a["bn1v"][3] = -9.0e-4                       # var + 1e-3 > 0: a usable, if odd, statistic
    W._check_head_arrays(a, 4)


@pytest.mark.parametrize("key,value,message", [
    ("d1w", np.nan, "dense1_kernel not finite at index 7"),
    ("d1b", np.inf, "dense1_bias not finite at index 7"),
    ("bn1g", np.nan, "bn1.gamma not finite at index 7"),
    ("bn1b", -np.inf, "bn1.beta not finite at index 7"),
    ("bn1m", np.nan, "bn1.moving_mean not finite at index 7"),
    ("bn1v", np.inf, "bn1.moving_variance not finite at index 7"),
    ("bn1v", -1e-3, "bn1.moving_variance \\+ 1e-3 is not > 0 at unit 7"),
    ("d2w", np.nan, "dense2_kernel not finite at index 7"),
    ("d2b", np.nan, "dense2_bias not finite at index 3")])
def test_c_api_refuses_unusable_head_weights(key, value, message):
    """gnm_head_create and gnm_head_train_create share the check; the trainer's runs before it looks for a device."""
    from genomad_b200 import engine
    lib = engine.load_library()
    a = _arrays()
    a[key].reshape(-1)[3 if key == "d2b" else 7] = value
    hw = W.head_c_struct(a, engine._HeadW, engine._BnW)
    tr = C.c_void_p()
    rc = lib.gnm_head_train_create(0, C.byref(hw), 8, 0, C.c_float(1e-3), C.byref(tr))
    assert rc != 0 and not tr.value
    assert re.fullmatch(f"gnm_head_train_create: {message}", lib.gnm_last_error().decode())
