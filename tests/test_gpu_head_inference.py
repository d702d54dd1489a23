"""
Classifier-head inference on an H100 against fp64 (run with `-m gpu -s` for the tables), and the per-contig reductions on
chromosome-length contigs.

Every case runs on both routes of gnm_head_forward, conv_impl 0 (3 x TF32 on the tensor cores, what --head uses) and 1 (FFMA),
and is checked against head_ref.folded -- the head evaluated in fp64 from fold_bn's own float32 scale and shift -- with the
derived per-row bounds of head_ref.kernel_bound:
  * the hidden rows h2 (the handle's last step) within the per-unit bound of dense_1 + BN + ReLU;
  * log p within the bound wherever fp64's p is a normal fp32, p == 0 only below fp32's subnormal range, no NaN, and fp64's
    argmax wherever its margin exceeds the bound (head_ref.check_probs).
The fold's own error (folded against the exact head) is printed per case and held to head_ref.fold_bound.

Cases: every class count 2..32; batch shapes at the 64- and 128-row tile edges and max_batch steps (with each row's bits
independent of the call it is in); encoder embeddings of unusual windows and arbitrary float32 rows; BN regimes (moving
mean / std up to 10^3, moving variance 0 .. 10^4, gamma 2^-10 .. 2^10) and a head trained by engine.HeadTrainer; heads
sharpened by 2^k, k = 0..8, binned by the log-odds margin of the top class.
"""
import numpy as np
import pytest

import head_ref as R
from test_head_inference_cpu import arbitrary_rows

pytestmark = pytest.mark.gpu

ROUTES = {0: "tc", 1: "ffma"}


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch


@pytest.fixture(scope="module")
def w():
    from genomad_b200 import weights as W
    return W.load_weights()


_CLFS = {}


def clf(w, impl, mb):
    from genomad_b200 import engine
    if (impl, mb) not in _CLFS:
        c = engine.Classifier(w, device=0, max_batch=mb)
        c.set_option("conv_impl", impl)
        _CLFS[impl, mb] = c
    return _CLFS[impl, mb]


def windows(seed):
    """uint8 [n, 6000]: ACGT windows over a spread of GC content, N runs, an all-N window, a short padded tail, lower-case and
    IUPAC windows, and windows holding every byte value."""
    rng = np.random.default_rng(seed)
    out = []
    for gc in np.linspace(0.15, 0.85, 48):
        p = np.array([(1 - gc) / 2, gc / 2, gc / 2, (1 - gc) / 2])
        out.append(np.frombuffer(b"ACGT", np.uint8)[rng.choice(4, 6000, p=p)].copy())
    base = out[20]
    for a0, ln in ((0, 100), (2000, 1500), (5990, 10)):
        v = base.copy()
        v[a0:a0 + ln] = ord("N")
        out.append(v)
    out.append(np.full(6000, ord("N"), np.uint8))
    v = base.copy()
    v[150:] = ord("N")                                                   # a 150-base tail window
    out.append(v)
    out.append(np.where((base >= 65) & (base <= 90), base + 32, base).astype(np.uint8))   # lower case
    out.append(np.frombuffer(b"ACGTRYSWKMBDHVN", np.uint8)[rng.integers(0, 15, 6000)].copy())
    for s in range(4):
        out.append(np.arange(256, dtype=np.uint8)[rng.permutation(np.arange(6000) % 256)].copy())
    return np.stack(out)


@pytest.fixture(scope="module")
def X(torch, w):
    """float32 [n, 512]: encoder embeddings of windows() and arbitrary_rows(), on the host."""
    a = torch.from_numpy(windows(1)).cuda()
    _, emb = clf(w, 0, 1000).embed_ascii(a)
    return np.concatenate([emb.cpu().numpy(), arbitrary_rows(7)])


def run(torch, w, impl, mb, a, X_):
    """(probabilities [n, C], h2 of the last step) of Head.predict on a classifier with (impl, max_batch)."""
    from genomad_b200 import engine, weights as W
    c = clf(w, impl, mb)
    head = engine.Head(c, W.HeadFile(a, tuple(f"c{i}" for i in range(a["d2b"].shape[0])), ""))
    p = head.predict(torch.from_numpy(np.ascontiguousarray(X_)).cuda())
    last = (len(X_) - 1) % mb + 1
    h2 = c.debug_fetch("h2", last).cpu().numpy()
    torch.cuda.synchronize()
    head.close()
    return p.cpu().numpy(), h2


def check(a, X_, probs, h2, impl, tag):
    """Assert a run against folded() with kernel_bound; returns (worst h2 err / bound, worst log p err / bound, fold ratio)."""
    b = R.kernel_bound(a, X_, ROUTES[impl])
    ref = b["ref"]
    last = slice(len(X_) - len(h2), len(X_))
    qh = np.abs(h2.astype(np.float64) - ref["h"][last]) / b["dy"][last]
    assert (qh <= 1).all(), f"{tag}: h2 off by {qh.max():.3g} x the bound at row/unit {np.unravel_index(qh.argmax(), qh.shape)}"
    qp = R.check_probs(ref["logp"], b["dlogp"], probs)
    fold = np.abs(ref["logits"] - R.logits_exact(a, X_))
    fb = R.fold_bound(a, X_)
    assert (fold <= fb).all(), tag
    return float(qh.max()), qp, float((fold / fb).max()), float(fold.max())


# ------------------------------------------------------------------------------------------------ every class count
@pytest.mark.parametrize("impl", [0, 1])
def test_every_class_count(torch, w, X, impl):
    print(f"\nroute {ROUTES[impl]}: C, worst h2 err/bound, worst log p err/bound, fold gap / bound (max gap)")
    for C in range(2, 33):
        a = R.random_head(C, 100 + C)
        p, h2 = run(torch, w, impl, 1000, a, X)
        qh, qp, qf, gap = check(a, X, p, h2, impl, f"C={C}")
        print(f"  C={C:2d}  {qh:.3f}  {qp.max():.2e}  {qf:.3f} ({gap:.1e})")


# ------------------------------------------------------------------------------------------------ batch shapes
@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("mb", [64, 256, 1000])
def test_batch_shapes(torch, w, X, impl, mb):
    rng = np.random.default_rng(mb)
    n_long = 3 * mb + 17
    X_long = X[rng.integers(0, len(X), n_long)]
    C = {64: 5, 256: 17, 1000: 32}[mb]
    a = R.random_head(C, mb)
    p_long, h2 = run(torch, w, impl, mb, a, X_long)
    qh, qp, _, _ = check(a, X_long, p_long, h2, impl, f"mb={mb}")
    print(f"\nroute {ROUTES[impl]} max_batch {mb} C={C}: {n_long} rows, h2 {qh:.3f}, log p {qp.max():.2e} of the bound")
    for n in sorted({1, 63, 64, 65, 127, 128, 129, mb - 1, mb, mb + 1}):
        p, h2 = run(torch, w, impl, mb, a, X_long[:n])
        assert np.array_equal(p.view(np.uint32), p_long[:n].view(np.uint32)), f"n={n}: rows differ from the long call's"
        check(a, X_long[:n], p, h2, impl, f"mb={mb} n={n}")
    for i in sorted({0, 63, 64, 127, 128, mb - 1, mb, 2 * mb + 5, n_long - 1}):
        p, _ = run(torch, w, impl, mb, a, X_long[i:i + 1])
        assert np.array_equal(p.view(np.uint32), p_long[i:i + 1].view(np.uint32)), f"row {i} alone differs"


# ------------------------------------------------------------------------------------------------ BN regimes
REGIMES = [dict(ratio=r) for r in (0, 10, 100, 1000)] + [dict(var=v, ratio=10) for v in (0, 1e-6, 1, 1e4)] + \
          [dict(gamma_log2=(-10, 10))]


@pytest.mark.parametrize("impl", [0, 1])
def test_bn_regimes(torch, w, X, impl):
    print(f"\nroute {ROUTES[impl]}: regime, worst h2 err/bound, worst log p err/bound, fold gap / bound (max gap)")
    for i, regime in enumerate(REGIMES):
        C = 3 + 4 * i % 29
        a = R.bn_regime_head(X[:60], C, 40 + i, **regime)
        p, h2 = run(torch, w, impl, 1000, a, X)
        qh, qp, qf, gap = check(a, X, p, h2, impl, str(regime))
        print(f"  {str(regime):32s} C={C:2d}  {qh:.3f}  {qp.max():.2e}  {qf:.3f} ({gap:.1e})")


@pytest.fixture(scope="module")
def trained(torch, w):
    """A head trained by engine.HeadTrainer for 300 steps on encoder embeddings of the composition classes of
    test_gpu_head_module.py (GC 35 %, GC 65 %, a planted motif), and the embeddings."""
    from genomad_b200 import engine, weights as W
    rng = np.random.default_rng(11)
    rows, labels = [], []
    for y, kind in enumerate(("gc35", "gc65", "motif")):
        gc = {"gc35": 0.35, "gc65": 0.65, "motif": 0.5}[kind]
        p = np.array([(1 - gc) / 2, gc / 2, gc / 2, (1 - gc) / 2])
        s = np.frombuffer(b"ACGT", np.uint8)[rng.choice(4, (200, 6000), p=p)].copy()
        if kind == "motif":
            for a0 in range(0, 6000 - 12, 50):
                s[:, a0:a0 + 12] = np.frombuffer(b"TTAGGGTTAGGG", np.uint8)
        rows.append(s)
        labels += [y] * 200
    _, emb = clf(w, 0, 1000).embed_ascii(torch.from_numpy(np.concatenate(rows)).cuda())
    lab = torch.tensor(labels, dtype=torch.int32, device="cuda")
    tr = engine.HeadTrainer(W.initial_head(3, 5), device=0, max_batch=128, seed=5)
    cw = torch.ones(3, device="cuda")
    for step in range(300):
        tr.step(emb, torch.from_numpy(rng.choice(600, 128, replace=False)).cuda(), lab, cw)
    a = tr.weights()
    tr.close()
    ratio = np.abs(a["bn1m"]) / np.sqrt(a["bn1v"])
    q = np.quantile(ratio, [0.5, 0.9, 0.99, 1.0])
    print(f"\ntrained head: moving mean / moving std per unit: median {q[0]:.2f}, p90 {q[1]:.2f}, p99 {q[2]:.2f}, "
          f"max {q[3]:.2f}; moving variance min {a['bn1v'].min():.2e}, median {np.median(a['bn1v']):.2e}")
    return a, emb.cpu().numpy()


@pytest.mark.parametrize("impl", [0, 1])
def test_trained_head(torch, w, X, trained, impl):
    a, E = trained
    for name, X_ in (("training windows", E), ("window set", X)):
        p, h2 = run(torch, w, impl, 1000, a, X_)
        qh, qp, qf, gap = check(a, X_, p, h2, impl, name)
        print(f"route {ROUTES[impl]} trained head, {name}: h2 {qh:.3f}, log p {qp.max():.2e} of the bound; "
              f"fold gap {gap:.1e} ({qf:.3f} of its bound)")


# ------------------------------------------------------------------------------------------------ confidence
BINS = [(0, 9), (9, 17), (17, 40), (40, 110), (110, np.inf)]


@pytest.mark.parametrize("impl", [0, 1])
def test_confidence(torch, w, X, trained, impl):
    heads = {"random C=7": (R.random_head(7, 3), X), "trained": trained}
    print(f"\nroute {ROUTES[impl]}: head, k, rows per margin bin and worst log p err/bound per bin")
    seen = set()
    for name, (a0, X_) in heads.items():
        for k in range(9):
            a = R.sharpen(a0, k)
            p, h2 = run(torch, w, impl, 1000, a, X_)
            b = R.kernel_bound(a, X_, ROUTES[impl])
            lp = b["ref"]["logp"]
            q = R.check_probs(lp, b["dlogp"], p)
            srt = np.sort(lp, 1)
            mu = srt[:, -1] - srt[:, -2]
            cells = []
            for lo, hi in BINS:
                m = (mu >= lo) & (mu < hi)
                if m.any():
                    seen.add(lo)
                    cells.append(f"[{lo:g},{hi:g}): {int(m.sum())} rows {q[m].max():.1e}")
            print(f"  {name:10s} k={k}: " + "; ".join(cells))
            assert not np.isnan(p).any()
    assert seen == {lo for lo, _ in BINS}, "a margin bin was never reached"


# ------------------------------------------------------------------------------------------------ per-contig reductions
def _running(x):
    """fp32 running sums in row order of x [n, C] -> [C] (sequential: np.add.accumulate does not reorder)"""
    if len(x) == 0:
        return np.zeros(x.shape[1], np.float32)
    return np.add.accumulate(np.asarray(x, np.float32), axis=0, dtype=np.float32)[-1]


def _ref_segments(x, off, mean):
    C = x.shape[1]
    out = []
    for c in range(len(off) - 1):
        s = _running(x[off[c]:off[c + 1]])
        n = off[c + 1] - off[c]
        out.append(s / np.float32(max(n, 1)) if mean else np.r_[s, np.float32(n)].astype(np.float32))
    return np.stack(out) if out else np.zeros((0, C if mean else C + 1), np.float32)


def _head(w, C):
    from genomad_b200 import engine, weights as W
    return engine.Head(clf(w, 0, 64), W.HeadFile(R.random_head(max(C, 2), 1), tuple(f"c{i}" for i in range(max(C, 2))), ""))


@pytest.mark.parametrize("C", [1, 2, 3, 7, 31, 32])
@pytest.mark.parametrize("n_contigs", [127, 128, 129])
def test_head_segment_layouts(torch, w, C, n_contigs):
    rng = np.random.default_rng(C * 1000 + n_contigs)
    lens = rng.integers(0, 40, n_contigs)
    lens[::7] = 0
    lens[3::7] = 1
    off = np.r_[0, np.cumsum(lens)].astype(np.int32)
    x = rng.random((off[-1], C)).astype(np.float32)
    head = _head(w, C)
    xd, od = torch.from_numpy(x).cuda(), torch.from_numpy(off).cuda()
    mean, s = head.segment_mean(xd, od).cpu().numpy(), head.segment_sum(xd, od).cpu().numpy()
    assert mean.shape == (n_contigs, C) and s.shape == (n_contigs, C + 1)
    assert np.array_equal(mean, _ref_segments(x, off, True))
    assert np.array_equal(s, _ref_segments(x, off, False))
    assert np.array_equal(s[:, C], lens.astype(np.float32))
    assert not mean[lens == 0].any()


LONG = [10_000, 100_000, 167_000]


def _prob_rows(n, C, p0, seed):
    """float32 [n, C] probability-like rows: column 0 near p0, the rest sharing 1 - p0."""
    rng = np.random.default_rng(seed)
    x = np.empty((n, C), np.float32)
    x[:, 0] = p0 * (1 + 0.2 * rng.uniform(-1, 1, n))
    if C > 1:
        x[:, 1:] = ((1 - x[:, :1]) * rng.dirichlet(np.ones(C - 1), n)).astype(np.float32)
    return x


def _gamma(m):
    """the running-sum bound's factor: m additions lose at most m u / (1 - m u) of sum |x| (first order: m u)"""
    return m * R.U32 / (1 - m * R.U32)


def _long_check(got_mean, got_sum, x, off, tag):
    """bitwise the NumPy running sums; within (n - 1) u sum |x| of fp64; prints the mean's distance from fp64."""
    assert np.array_equal(got_sum, _ref_segments(x, off, False)[:, :got_sum.shape[1]]), tag
    assert np.array_equal(got_mean, _ref_segments(x, off, True)), tag
    out = []
    for c in range(len(off) - 1):
        seg = x[off[c]:off[c + 1]].astype(np.float64)
        n = len(seg)
        if n == 0:
            continue
        s64 = seg.sum(0)
        err = np.abs(got_sum[c, :x.shape[1]] - s64)
        assert (err <= _gamma(n - 1) * np.abs(seg).sum(0)).all(), tag
        rel = np.abs(got_mean[c] - s64 / n) / (s64 / n)
        out.append((n, float(rel[0]), float(rel.max())))
    return out


@pytest.mark.parametrize("C", [1, 3, 7, 32])
def test_head_segments_on_chromosome_length_contigs(torch, w, C):
    head = _head(w, C)
    print()
    for p0 in (0.5, 1e-3):
        x = _prob_rows(sum(LONG) + 3, C, p0, C)
        off = np.r_[0, np.cumsum([LONG[0], 1, LONG[1], 0, LONG[2], 2])].astype(np.int32)
        xd, od = torch.from_numpy(x).cuda(), torch.from_numpy(off).cuda()
        res = _long_check(head.segment_mean(xd, od).cpu().numpy(), head.segment_sum(xd, od).cpu().numpy(), x, off, f"C={C}")
        print(f"C={C} column 0 ~ {p0:g}: " + ", ".join(f"{n} windows: mean off fp64 by {r0:.1e} relative (all columns "
                                                      f"{rm:.1e})" for n, r0, rm in res if n >= 10_000))


def test_shipped_segments_on_chromosome_length_contigs(torch, w):
    c = clf(w, 0, 64)
    for p0 in (0.5, 1e-3):
        x = _prob_rows(sum(LONG), 3, p0, 9)
        off = np.r_[0, np.cumsum(LONG)].astype(np.int32)
        xd, od = torch.from_numpy(x).cuda(), torch.from_numpy(off).cuda()
        res = _long_check(c.segment_mean(xd, od).cpu().numpy(), c.segment_sum(xd, od).cpu().numpy(), x, off, "shipped")
        print(f"\nshipped, column 0 ~ {p0:g}: " + ", ".join(f"{n}: {r0:.1e}" for n, r0, _ in res))


def test_segment_sum_rows_carry_inside_a_chromosome_length_contig(torch, w):
    c = clf(w, 0, 64)
    n = LONG[2]
    rng = np.random.default_rng(4)
    x = np.maximum(rng.normal(0.3, 1.0, (n, 512)), 0).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    whole, _ = c.segment_sum_rows(xd, torch.tensor([0, n], dtype=torch.int32, device="cuda"))
    want = _running(x)
    assert np.array_equal(whole.cpu().numpy()[0], want)
    cuts = np.r_[0, np.sort(rng.choice(np.arange(1, n), 5, replace=False)), n]
    carry = None
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        _, carry = c.segment_sum_rows(xd[lo:hi], torch.tensor([0, hi - lo], dtype=torch.int32, device="cuda"), carry)
    assert np.array_equal(carry.cpu().numpy(), want), f"carry split at {cuts[1:-1].tolist()} changes the sum"
    s64 = x.astype(np.float64).sum(0)
    assert (np.abs(want - s64) <= _gamma(n - 1) * np.abs(x.astype(np.float64)).sum(0)).all()
    print(f"\nsegment_sum_rows, {n} rows: column sums off fp64 by {np.max(np.abs(want - s64) / s64):.1e} relative at most")


@pytest.mark.parametrize("C", list(range(1, 33)))
def test_both_strands_is_bitwise_the_fp32_mean(torch, C):
    from genomad_b200 import engine
    rng = np.random.default_rng(C)
    f, r = (rng.random((50, C)).astype(np.float32) * np.float32(2.0) ** rng.integers(-30, 30, (50, C)).astype(np.float32)
            for _ in range(2))
    want = ((f + r) * np.float32(0.5)).astype(np.float32)
    got = engine.both_strands(torch.from_numpy(f).cuda(), torch.from_numpy(r).cuda()).cpu().numpy()
    assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(engine.both_strands(r, f).view(np.uint32), want.view(np.uint32))


# ------------------------------------------------------------------------------------------------ refused heads
@pytest.mark.parametrize("key,value,message", [
    ("d1w", np.nan, "dense1_kernel not finite at index 7"), ("bn1g", np.inf, "bn1.gamma not finite at index 7"),
    ("bn1v", -1e-3, "bn1.moving_variance \\+ 1e-3 is not > 0 at unit 7"), ("d2b", np.nan, "dense2_bias not finite at index 1")])
def test_head_create_refuses_unusable_weights(torch, w, key, value, message):
    from genomad_b200 import engine, weights as W
    a = {k: v.copy() for k, v in R.random_head(3, 2).items()}
    a[key].reshape(-1)[1 if key == "d2b" else 7] = value
    with pytest.raises(engine.GnmError, match=f"^gnm_head_create: {message}$"):
        engine.Head(clf(w, 0, 64), W.HeadFile(a, ("a", "b", "c"), ""))
