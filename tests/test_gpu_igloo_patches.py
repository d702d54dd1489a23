"""
The IGLOO kernels on crowded patch sets and across fp32's range of w_v and patch-weight scales, against fp64 at stage precision
(run with `-m gpu -s` on an H100 for the tables).

Crowded patch sets.  The fused IGLOO kernel's gather (csrc/wv_gather.cuh) takes a fast path for a band of 24 positions with at
most 28 position groups (7 gather warps x 4 groups; a group is <= 4 patch entries on one position) and a generic path, which
parks the pass-0 halves in part_t, for bands with more; a CTA's unit range spans several bands and the path is chosen again
at every band.  The shipped and synthetic patch sets never exceed 27 groups per band, so the stage tests never reach the
generic path.  The sets below do, for both IGLOO layers: bands with exactly 27 / 28 groups (fast, every gather warp full) next
to 29 and ~35 (generic), among them band 0 (causal padding) and the short last band; every other band generic (at n = 24 most
CTAs change path inside one launch); all 8,400 entries on one band, on the two ends of the window or on one position; and
duplicate entries inside a patch, an all-zero patch and empty bands.  Each set's group counts are checked with the host
packing hook before the GPU runs it; then mpi, the logits of layer 1, h0-h2 and the probabilities meet their bars of
tests/stage_ref.py, and mpi's error is reported separately for patches that touch a generic band and patches that do not.

Weight scales.  gnm_create splits w_v * 2^e and the folded patch weights * 2^k into fp16 halves, max |w| moved to
[2^13, 2^14), e and k clamped to [-126, 121].  Two rescalings leave the model unchanged in exact arithmetic: (w_mult, w_bias)
x 2^j with w_qk x 2^-j, and w_v of both layers x 2^j with dense0's kernel x 2^-j.  While e and k stay inside the clamp the
fragments are the same bits and every later step scales by an exact power of two, so the library reproduces the rescaling
bit for bit wherever the rescaled fp32 inputs themselves are exact (no value near fp32's subnormal range); at every j the
fused path meets the fp64 bar wherever the fp32 path does.  The sweeps include both ends of the old clamp [-24, 40] (past its
bottom the fp16 halves overflowed: inf at j = +48) and the new clamp's top with the first j past it.
"""
import numpy as np
import pytest
import torch

import stage_ref as R
from oracle import igloo_model as M
from test_gpu_attr import _check_against_fp64
from test_gpu_stages import HEADER, PATHS, _fetch, _scaled, _windows
from test_host_cpu import _pack_patches

pytestmark = pytest.mark.gpu

BAND, N_BANDS, FAST_CAP = 24, 250, 28          # positions per band, bands, position groups the fast path takes (7 warps x 4)
LAST_ROWS = 5997 - (N_BANDS - 1) * BAND          # 21 valid positions in the last band
TRIO = ("tc fused (default)", "tc fuse_gather=0", "tc fuse_l1")
SAME_ALL_PATHS = ("y1", "y2", "y3_0", "q0", "q1")


@pytest.fixture(scope="module")
def synthetic(weights_npz):
    return M.synthetic_igloo_weights(M.load_npz_weights(weights_npz))


# ------------------------------------------------------------------------------------------ crowded patch sets
def _band_counts(groups, rows, rng, fixed=(), top_up=True):
    """entry counts of a band's `rows` positions giving exactly `groups` position groups (ceil(count / 4) each); `fixed`: the
    counts of the first positions; top_up: random extra entries that do not open a group"""
    c = np.zeros(rows, np.int64)
    c[:len(fixed)] = fixed
    free = np.arange(len(fixed), rows)
    while int(((c + 3) // 4).sum()) < groups:
        empty = free[c[free] == 0]
        i = empty[0] if len(empty) else rng.choice(free)
        c[i] = 4 * ((c[i] + 3) // 4) + 1
    assert int(((c + 3) // 4).sum()) == groups
    if top_up:
        c[free] = rng.integers(c[free], 4 * ((c[free] + 3) // 4) + 1)
    return c


def _positions(bands, rng):
    """{band: entry counts} -> the 8,400 entries' positions: the listed bands exactly, the rest spread at random over the other
    bands (a handful of groups each), dealt to the 2100 patches at random"""
    pos = [b * BAND + np.repeat(np.arange(len(c)), c) for b, c in bands.items()]
    pos = np.concatenate(pos) if pos else np.zeros(0, np.int64)
    assert len(pos) <= 8400
    others = np.concatenate([np.arange(b * BAND, min(5997, (b + 1) * BAND)) for b in range(N_BANDS) if b not in bands])
    pos = np.concatenate([pos, rng.choice(others, 8400 - len(pos))])
    return rng.permutation(pos).reshape(2100, 4).astype(np.int32)


def _set_threshold(rng):
    rows = lambda b: LAST_ROWS if b == N_BANDS - 1 else BAND                                      # noqa: E731
    plan = {0: (35, (9, 8, 5, 4)), 1: (27, (4, 5)), 2: (28, (8, 9)), 3: (29, ()), 60: (28, ()), 61: (29, (9,)),
            62: (27, ()), 63: (35, (5, 5, 5)), 124: (29, ()), 125: (28, (4, 4, 4, 4)), 126: (36, ()), 247: (27, ()),
            248: (28, ()), 249: (29, (8,))}
    bands = {b: _band_counts(g, rows(b), rng, fixed) for b, (g, fixed) in plan.items()}
    return _positions(bands, rng), {b: g for b, (g, _) in plan.items()}


def _set_alternating(rng):
    bands = {b: _band_counts(int(rng.integers(29, 37)), BAND, rng, top_up=False) for b in range(0, N_BANDS, 2)}
    return _positions(bands, rng), None


def _patch_set(name, s, w):
    """(patches [2100][4], {band: group count} to assert or None, w_mult of layer s) of one crowded set"""
    rng = np.random.default_rng(100 + s)
    w_mult = w[f"ig{s}_w_mult"]
    expect = None
    if name == "threshold":
        p, expect = _set_threshold(rng)
    elif name == "alternating":
        p, _ = _set_alternating(rng)
    elif name == "one_band":
        p = (3000 + rng.permutation(np.repeat(np.arange(BAND), 350))).reshape(2100, 4)
    elif name == "ends":
        p = np.tile(np.asarray([0, 1, 5995, 5996]), (2100, 1))
    elif name == "one position x4":
        p = np.full((2100, 4), 3001)
    else:                                       # "odd": duplicates inside patches, an all-zero patch, empty bands 10-40 and 249
        p = w[f"ig{s}_random_patches"].reshape(2100, 4).copy()
        moved = ((p >= 10 * BAND) & (p < 41 * BAND)) | (p >= (N_BANDS - 1) * BAND)
        p[moved] = rng.integers(41 * BAND, (N_BANDS - 1) * BAND, int(moved.sum()))
        p[100:200, 1], p[100:200, 3] = p[100:200, 0], p[100:200, 2]
        p[200:210] = p[200:210, :1]
        w_mult = w_mult.copy()
        w_mult[0, 300] = 0.0
    return np.ascontiguousarray(p, np.int32), expect, w_mult


SETS = ["threshold", "alternating", "one_band", "ends", "one position x4", "odd"]


def _crowded(name, w):
    """the weights with set `name` in both IGLOO layers, and per layer the patches that touch a generic-path band; asserts the
    group counts per band with the host packing hook"""
    w = dict(w)
    generic = []
    for s in (0, 1):
        p, expect, w_mult = _patch_set(name, s, w)
        w[f"ig{s}_random_patches"] = p.reshape(2100, 4, 1)
        w[f"ig{s}_w_mult"] = w_mult
        o = _pack_patches(p, w_mult.reshape(2100, 4, 128), w[f"ig{s}_w_summer"].reshape(512))
        assert (o["band_rows"], o["n_bands"]) == (BAND, N_BANDS)
        g = np.diff(o["band_first"])
        counts = np.bincount(p.reshape(-1), minlength=5997)
        if name == "threshold":
            assert {b: int(g[b]) for b in expect} == expect
            assert g[[b for b in range(N_BANDS) if b not in expect]].max() <= 24
            assert {4, 5, 8, 9} <= set(counts[:BAND].tolist()) | set(counts[2 * BAND:3 * BAND].tolist())
        elif name == "alternating":
            assert np.all(g[0::2] > FAST_CAP) and np.all(g[1::2] <= FAST_CAP)
        elif name == "one_band":
            assert g[125] == 24 * 88 and g.sum() == g[125]
        elif name == "odd":
            assert np.all(g[10:41] == 0) and g[N_BANDS - 1] == 0
            assert np.all(p[200:210] == p[200:210, :1]) and not w_mult[0, 300].any()
        gen_band = g > FAST_CAP
        generic.append(gen_band[p // BAND].any(axis=1))
        print(f"\n{name}, layer {s}: groups per band max {g.max()}, {int(gen_band.sum())} generic bands, "
              f"{int(generic[-1].sum())} of 2100 patches touch one")
    return w, generic


class _Refs:
    """fp64 references of the stages that depend only on y1 / y3 (the same bits on every path), computed once per input"""

    def __init__(self, w):
        self.w, self.key, self.val = w, None, None

    def get(self, got):
        if self.key is None or not (torch.equal(self.key[0], got["y1"]) and torch.equal(self.key[1], got["y3_0"])):
            w = self.w
            self.key = (got["y1"], got["y3_0"])
            self.val = {"q0": R.wv_pool(got["y1"], w["ig0_w_v"]), "mpi0": R.gather(got["y1"], w, 0),
                        "q1": R.wv_pool(got["y3_0"], w["ig1_w_v"]), "mpi1": R.gather(got["y3_0"], w, 1)}
        return self.val


def _check_igloo(label, w, got, refs, generic=None):
    """IGLOO stages of `got` (a _fetch with stops (2, 0)) against their bars; mpi's max error also split by `generic` (per layer:
    patches touching a generic-path band).  Prints one table row per stage, returns the misses."""
    n = got["q0"].shape[0]
    preg = R.position_regions(n, pooled=True)
    ref = refs.get(got)
    logits0 = got["mpi0"] @ torch.as_tensor(w["ig0_w_qk"], dtype=R.D)
    checks = [("q0 (w_v#0)", "wv", got["q0"], ref["q0"], preg), ("mpi0", "gather", got["mpi0"], ref["mpi0"], 0),
              ("q1 (w_v#1)", "wv", got["q1"], ref["q1"], preg), ("mpi1", "gather", got["mpi1"], ref["mpi1"], 1),
              ("logits1", "tf32x3", got["logits"], R.matmul(got["mpi1"], w["ig1_w_qk"]), {}),
              ("h0[:128]", "attention", got["h0"][:, :128], R.attention(logits0, got["q0"]), {}),
              ("h0[128:]", "attention", got["h0"][:, 128:], R.attention(got["logits"], got["q1"]), {}),
              ("h1 (dense0)", "tf32x3", got["h1"], R.dense_bn_relu(got["h0"], w, 0), {}),
              ("h2 (dense1)", "tf32x3", got["h2"], R.dense_bn_relu(got["h1"], w, 1), {}),
              ("probs", "probs", got["probs"], R.head_softmax(got["h2"], w), {})]
    bad = []
    for stage, key, g, r, regions in checks:
        rms_bar, max_bar = R.BARS[key]
        if isinstance(regions, int):                       # mpi of layer `regions`: generic-band patches vs the others
            m = R.metrics(g, r)
            cols = {}
            if generic is not None:
                gen = torch.from_numpy(generic[regions])
                for part, idx in (("generic", gen), ("fast", ~gen)):
                    if idx.any():
                        cols[part] = R.metrics(g[:, idx], R.Ref(*(t[:, idx] for t in r)))["max"]
                        m["max " + part] = cols[part]
            per_region = ", ".join(f"{k} {v:.1e}" for k, v in cols.items()) or "-"
        else:
            m = R.metrics(g, r, regions)
            per_region = ", ".join(f"{k[4:]} {v:.1e}" for k, v in m.items() if k.startswith("max ")) or "-"
        ok = m["rms"] <= rms_bar and all(v <= max_bar for k, v in m.items() if k.startswith("max"))
        print(f"| {label} | {stage} | {m['rms']:.2e} | {rms_bar:.0e} | {m['max']:.2e} | {max_bar:.1e} | {per_region} | "
              f"{'ok' if ok else 'MISS'} |")
        if not ok:
            bad.append((label, stage, m))
    return bad


def _three_paths(w, a, max_batch):
    """_fetch through the default path, fuse_gather = 0 and fuse_l1; asserts what the paths share bitwise (y, q everywhere;
    fuse_l1 = 1 runs the separate gather of fuse_gather = 0, so those two agree in everything)"""
    runs = {p: _fetch(w, a, max_batch, PATHS[p][0], stops=(2, 0)) for p in TRIO}
    base, sep, l1 = (runs[p] for p in TRIO)
    for k in SAME_ALL_PATHS:
        assert torch.equal(base[k], sep[k]) and torch.equal(base[k], l1[k]), k
    for k in sep:
        assert torch.equal(sep[k], l1[k]), f"fuse_l1 vs fuse_gather=0: {k}"
    return runs


@pytest.mark.parametrize("name", SETS)
def test_crowded_patch_sets_every_igloo_stage(synthetic, name):
    w, generic = _crowded(name, synthetic)
    refs = _Refs(w)
    print(HEADER)
    bad = []
    for n, mb in ((1, 9), (9, 9), (24, 24)):
        a = _windows(9, seed=61)[:n] if n < 24 else _windows(24, seed=67)
        runs = _three_paths(w, a, mb)
        for p in TRIO[:2]:                             # fuse_l1: bitwise fuse_gather = 0 (asserted)
            bad += _check_igloo(f"{name}, n={n}, max_batch={mb}, {p}", w, runs[p], refs, generic)
    assert not bad


def test_crowded_patch_set_attributions(synthetic, golden_dir):
    """The attribution backward pass walks the same patch packing (slot_of, ent_w): the threshold set through
    gnm_attribute_ascii against the fp64 reference at the 1e-4 bar of tests/test_gpu_attr.py."""
    from genomad_b200 import engine
    w, _ = _crowded("threshold", synthetic)
    g = np.load(golden_dir / "reference_graph_golden.npz")["windows"][:4]
    acgt = np.frombuffer(b"ACGT", np.uint8)
    a = np.concatenate([g, acgt[np.random.default_rng(71).integers(0, 4, (3, 6000))]])
    c = engine.Classifier(w, device=0, max_batch=16)
    try:
        c._attr_ctx(16)
        for target in (0, 1, 2):
            probs, _, err = _check_against_fp64(c, a, w, target)
            print(f"\nthreshold set, target {target}: per-window max|d attr| / max|attr| vs fp64: " + " ".join(f"{e:.1e}" for e in err))
            assert err.max() <= 1e-4, (target, err)
            assert torch.equal(probs, c.predict_ascii(torch.from_numpy(a).cuda()))
    finally:
        c.close()


# ------------------------------------------------------------------------------------------ weight scales
def _safe(x, j):
    """x * 2^j is exact in fp32 and far from its subnormal range and its overflow (margin 2^26, enough for the TF32 / fp16 lo
    halves taken of it)"""
    a = np.abs(np.asarray(x, np.float64))
    a = a[a > 0]
    return a.min() * 2.0 ** j >= 2.0 ** -100 and a.max() * 2.0 ** j <= 2.0 ** 100


def _sweep(w0, scale, js, paths, stage_keys, bitwise_keys, scaled_keys, exact):
    """Runs the rescaled weights scale(j) through `paths`; asserts (1) bitwise: where exact(j, run at j = 0), the stages
    `scaled_keys` are the j = 0 values x 2^j and `bitwise_keys` the j = 0 values, on every path; (2) precision: at every j the
    stages `stage_keys` of every path meet their bar wherever the last path (the fp32 yardstick) does.  Prints a table."""
    a = _windows(8, seed=53)
    runs0 = {p: _fetch(w0, a, 8, PATHS[p][0], stops=(2, 0)) for p in paths}
    print("\n| j | path | " + " | ".join(f"{k} rms / max" for k in stage_keys) + " | bitwise |\n|---|---|" + "---|" * (len(stage_keys) + 1))
    bad = []
    for j in js:
        w = scale(j)
        refs = _Refs(w)
        ok = {}
        bit = exact(j, runs0[paths[0]])
        for p in paths:
            got = runs0[p] if j == 0 else _fetch(w, a, 8, PATHS[p][0], stops=(2, 0))
            for k in ("q0", "q1", "mpi0", "mpi1", "logits", "h0", "h1", "h2", "probs"):
                assert torch.isfinite(got[k]).all(), (j, p, k)
            if bit:
                for k in scaled_keys:
                    assert torch.equal(got[k], runs0[p][k] * 2.0 ** j), (j, p, k)
                for k in bitwise_keys:
                    assert torch.equal(got[k], runs0[p][k]), (j, p, k)
            ref = refs.get(got)
            ms = {k: R.metrics(got[k], ref[k]) for k in stage_keys}
            ok[p] = {k: ms[k]["rms"] <= R.BARS[b][0] and ms[k]["max"] <= R.BARS[b][1] for k, b in stage_keys.items()}
            print(f"| {j} | {p} | " + " | ".join(f"{ms[k]['rms']:.1e} / {ms[k]['max']:.1e}" for k in stage_keys)
                  + f" | {'yes' if bit else '-'} |")
        for p in paths[:-1]:
            for k in stage_keys:
                if ok[paths[-1]][k] and not ok[p][k]:
                    bad.append((j, p, k))
    assert not bad, bad


PATCH_J = [-101, -100, -64, -20, -19, 0, 24, 45, 46, 48, 64, 100]


def test_patch_weight_scale_sweep(synthetic):
    """(w_mult, w_bias) of both layers x 2^j, w_qk x 2^-j.  The synthetic folded weights have k = 21, so the clamp's top
    (k = 121) is j = -100; the old clamp [-24, 40] ended at j = -19 and j = +45."""
    w0 = synthetic

    def scale(j):
        f = {f"ig{s}_{n}": 2.0 ** j for s in (0, 1) for n in ("w_mult", "w_bias")}
        f.update({f"ig{s}_w_qk": 2.0 ** -j for s in (0, 1)})
        return _scaled(w0, **f)

    def exact(j, run0):
        folded = [np.asarray(w0[f"ig{s}_w_mult"], np.float64).reshape(2100, 4, 128) * w0[f"ig{s}_w_summer"].reshape(1, 4, 128) / 32
                  for s in (0, 1)]
        return all(_safe(x, j) for x in folded + [w0[f"ig{s}_{n}"] for s in (0, 1) for n in ("w_mult", "w_bias")]
                   + [run0["mpi0"].numpy(), run0["mpi1"].numpy()]) and all(_safe(w0[f"ig{s}_w_qk"], -j) for s in (0, 1))

    _sweep(w0, scale, PATCH_J, ["tc fused (default)", "tc fuse_gather=0"], {"mpi0": "gather", "mpi1": "gather"},
           ("y1", "y3_0", "q0", "q1", "logits", "h0", "h1", "h2", "probs"), ("mpi0", "mpi1"), exact)


WV_J = [-105, -104, -103, -64, -23, -22, 0, 41, 42, 48, 100]


def test_wv_weight_scale_sweep_full_range(synthetic):
    """w_v of both layers x 2^j, dense0's kernel x 2^-j, through the three w_v paths and the fp32 validation kernels
    (conv_impl = 1, the yardstick).  max |w_v| gives e = 17 (layer 0) and 18 (layer 1): the clamp's top (e = 121) is j = -104
    and -103; the old clamp [-24, 40] ended at j = -23 / -22 and j = +41 / +42."""
    w0 = synthetic

    def scale(j):
        return _scaled(w0, ig0_w_v=2.0 ** j, ig1_w_v=2.0 ** j, d0w=2.0 ** -j)

    def exact(j, run0):
        return (all(_safe(x, j) for x in (w0["ig0_w_v"], w0["ig1_w_v"], run0["q0"].numpy(), run0["q1"].numpy(), run0["h0"].numpy()))
                and _safe(w0["d0w"], -j))

    _sweep(w0, scale, WV_J, ["tc fused (default)", "tc fuse_l1", "tc fuse_gather=0", "fp32 validation (conv_impl=1)"],
           {"q0": "wv", "q1": "wv"}, ("y1", "y3_0", "mpi0", "mpi1", "logits", "h1", "h2", "probs"), ("q0", "q1", "h0"), exact)


@pytest.mark.parametrize("case", ["w_v inf", "w_v nan", "folded patch weights overflow"])
def test_weights_without_an_fp16_split_are_refused(synthetic, case):
    """gnm_create refuses, naming the layer, w_v or folded patch weights that are not finite (no fp16 split carries them)
    instead of building a classifier that returns inf or NaN."""
    from genomad_b200 import engine
    w = dict(synthetic)
    if case == "w_v inf":
        w["ig1_w_v"] = w["ig1_w_v"].copy()
        w["ig1_w_v"].reshape(-1)[4321] = np.inf
        match = "IGLOO layer 1: w_v not finite"
    elif case == "w_v nan":
        w["ig0_w_v"] = w["ig0_w_v"].copy()
        w["ig0_w_v"].reshape(-1)[7] = np.nan
        match = "IGLOO layer 0: w_v not finite"
    else:
        w = _scaled(w, ig1_w_mult=2.0 ** 100, ig1_w_summer=2.0 ** 40)       # both finite, the product overflows fp32
        match = "IGLOO layer 1: folded patch weights .* not finite"
    with pytest.raises(engine.GnmError, match=match):
        engine.Classifier(w, device=0, max_batch=8)
