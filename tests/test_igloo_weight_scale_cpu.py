"""
The fp16 operand split of the fused IGLOO kernel's folded patch weights (csrc/api.cu pack_patches) across fp32's whole range of
weight scales, on the host (no GPU).

pack_patches folds w = w_mult * w_summer / 32, multiplies it by 2^k with max |w| * 2^k in [2^13, 2^14), splits the product into
fp16 hi / lo halves (the B fragments of the gather's mma) and gives the kernel unscale = 2^-k.  k is clamped to [-126, 121], where
2^k, 2^-k and the q epilogues' 2^-k / 32 are normal fp32.  So scaling w_mult by 2^j changes nothing but unscale, by exactly
2^-j, for every j whose k lies inside the clamp and whose folded weights stay normal fp32; past the clamp's top (weights below
2^-107) the halves still carry the weights to the gather's precision while they are normal fp32; folded weights that are not
finite cannot be carried and are refused.  (The clamp's bottom, k = -126, needs max |w| >= 2^139: no finite fp32 weight gets
there, so the halves of every finite weight set are finite.)  With the earlier clamp [-24, 40] the synthetic weights broke at
j = -20 (k = 41: the lo halves of the smallest weights left fp16's normal range) and at j = +46 (k = -25: the largest hi halves
reached 2^15, and 2^16 = inf at j = +48).
"""
import numpy as np
import pytest

from genomad_b200 import engine, weights
from oracle import igloo_model as M
from test_host_cpu import _frag_halves, _pack_patches

K_MIN, K_MAX = -126, 121
J_SWEEP = sorted(set(range(-100, 101)) | {-101, -105, -110, -112, -116, -119, -120, -125, -130, -140, 110, 120, 127}, key=abs)


@pytest.fixture(scope="module")
def layer0():
    w = M.synthetic_igloo_weights(weights.load_weights())
    return (np.ascontiguousarray(w["ig0_random_patches"].reshape(2100, 4), np.int32),
            w["ig0_w_mult"].reshape(2100, 4, 128).astype(np.float32), w["ig0_w_summer"].reshape(512).astype(np.float32))


def _scaled(x, j):
    """x * 2^j rounded once to fp32 (exact while the result is a normal fp32 number)"""
    return (x.astype(np.float64) * 2.0 ** j).astype(np.float32)


def _reconstruct(o):
    """the folded weights the fragments carry: (hi + lo) * unscale in fp64, [8400][128], with the kernel's channel mapping"""
    halves = _frag_halves(o["frag"][:8400]).astype(np.float64)             # [e][kh][ks][tig][word 4][half 2]
    w = np.zeros((8400, 128))
    for kh in range(2):
        for ks in range(4):
            for tig in range(4):
                k0 = 64 * kh + 16 * ks + 2 * tig
                w[:, [k0, k0 + 1]] = halves[:, kh, ks, tig, 0] + halves[:, kh, ks, tig, 2]
                w[:, [k0 + 8, k0 + 9]] = halves[:, kh, ks, tig, 1] + halves[:, kh, ks, tig, 3]
    return w * o["unscale"]


def test_patch_weight_scale_sweep(layer0):
    """w_mult x 2^j, j = -140 .. +127.  Where the folded weights are exactly the unscaled ones x 2^j (all of them normal fp32)
    and k = k0 - j is inside the clamp: fragments bitwise those of j = 0, unscale exactly 2^-j times j = 0's.  Wherever the
    largest folded weight is normal fp32: every weight reconstructed within 2^-20 of the largest (2^-24 measured at k's exact
    value; at the clamped k = 121 the error grows as the weights shrink, to 2^-20 where the largest is fp32's smallest normal
    number).  The halves are finite at every j."""
    patches, w_mult, w_summer = layer0
    o0 = _pack_patches(patches, w_mult, w_summer)
    w0 = o0["ent_w"][:8400].astype(np.float64)
    k0 = -int(np.log2(o0["unscale"]))
    assert o0["unscale"] == 2.0 ** -k0 and 2.0 ** 13 <= np.abs(w0).max() * 2.0 ** k0 < 2.0 ** 14
    nz = np.abs(w0[w0 != 0])
    rows = []
    for j in J_SWEEP:
        o = _pack_patches(patches, _scaled(w_mult, j), w_summer)
        ent = o["ent_w"][:8400].astype(np.float64)
        k = int(np.clip(k0 - j, K_MIN, K_MAX))
        halves = _frag_halves(o["frag"][:8400])
        assert np.all(np.isfinite(halves)), j
        assert o["unscale"] == 2.0 ** -k, (j, o["unscale"])
        exact = nz.min() * 2.0 ** j >= 2.0 ** -126 and np.array_equal(ent, w0 * 2.0 ** j)
        if exact and k == k0 - j:
            assert np.array_equal(o["frag"], o0["frag"]), j
        scale = np.abs(ent).max()
        err = np.abs(_reconstruct(o) - ent).max() / scale if scale > 0 else 0.0
        if scale >= 2.0 ** -126:
            assert err <= 2.0 ** -20, (j, err)
        rows.append((j, k, exact, err))
    assert {j for j, _, exact, _ in rows if exact} >= set(range(-90, 101))       # the sweep reaches the bitwise cases it claims
    print("\n| j | k | bitwise | max err / max w |\n|---|---|---|---|")
    for j, k, exact, err in sorted(rows):
        if j % 20 == 0 or j < -95 or abs(k0 - j - 40.5) < 1 or abs(k0 - j + 24.5) < 1:
            print(f"| {j} | {k} | {'yes' if exact and k == k0 - j else 'no'} | {err:.1e} |")


@pytest.mark.parametrize("case", ["product overflows", "inf in w_mult", "nan in w_mult", "nan in w_summer"])
def test_patch_weights_that_cannot_be_carried_are_refused(layer0, case):
    """Folded weights w_mult * w_summer / 32 that are not finite (here: finite factors whose product overflows fp32, or an inf /
    NaN factor) have no fp16 split; the packing refuses them instead of handing the gather inf or NaN fragments."""
    patches, w_mult, w_summer = layer0
    w_mult, w_summer = w_mult.copy(), w_summer.copy()
    if case == "product overflows":
        w_mult, w_summer = _scaled(w_mult, 100), _scaled(w_summer, 40)
        assert np.all(np.isfinite(w_mult)) and np.all(np.isfinite(w_summer))
    elif case == "inf in w_mult":
        w_mult[17, 2, 5] = np.inf
    elif case == "nan in w_mult":
        w_mult[2099, 3, 127] = np.nan
    else:
        w_summer[300] = np.nan
    with pytest.raises(AssertionError, match="not finite"):
        _pack_patches(patches, w_mult, w_summer)
    lib = engine.load_library()
    assert b"gnm_pack_patches" in lib.gnm_last_error()
