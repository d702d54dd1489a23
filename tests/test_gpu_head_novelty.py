"""
Head novelty on an H100, against the fp64 oracle of tests/novelty_ref.py:
  * the fit (class means, center, scatter S, whitening P, whitened means m_c) on Gaussian clusters, post-ReLU-like sparse rows
    with dead columns, rows scaled from 1e-3 to 1e3 and a class with one row, at C in {2, 3, 32} and fit sizes at the tile and
    chunk edges; the window distances of the fitted model within novelty_ref.distance_bound and 1e-6 D + 1e-9;
  * bitwise: two fits, and a row's distances under chunking, permutation and repeats;
  * errors: an empty class, no within-class variation;
  * end to end: train-head --novelty, then nn-classification --head (calibration membership, class predictions unchanged),
    and a head trained on two of three synthetic classes against the held-out third.
"""
import numpy as np
import pytest

import novelty_ref as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch


@pytest.fixture(scope="module")
def clf(torch):
    from genomad_b200 import engine
    c = engine.Classifier(None, device=0, max_batch=64)
    yield c
    c.close()


def make_rows(kind, N, C, seed):
    """(X float32 [N, 512], labels int32 [N]) of one input kind; every class has a row."""
    rng = np.random.default_rng(seed)
    y = np.concatenate([np.arange(C), rng.integers(0, C, N - C)]).astype(np.int32) if N >= C else None
    rng.shuffle(y)
    if kind == "gauss":
        centers = rng.normal(0, 2, (C, 512))
        X = centers[y] + rng.normal(0, 1, (N, 512)) * rng.uniform(0.2, 2.0, 512)
    elif kind == "relu":                      # post-ReLU-like: sparse, 40 columns dead on every row
        centers = rng.normal(0, 1, (C, 512))
        X = np.maximum(centers[y] + rng.normal(0, 1, (N, 512)), 0)
        X[:, rng.choice(512, 40, replace=False)] = 0
    elif kind == "scaled":                    # rows scaled by 1e-3 .. 1e3
        centers = rng.normal(0, 1, (C, 512))
        X = (centers[y] + rng.normal(0, 0.5, (N, 512))) * 10.0 ** rng.uniform(-3, 3, (N, 1))
    else:
        raise ValueError(kind)
    return X.astype(np.float32), y


def gpu_fit(torch, clf, X, y, C, rows=None, stats=True):
    from genomad_b200 import engine
    Xd = torch.from_numpy(X).cuda()
    rows = torch.arange(len(X), dtype=torch.int64, device="cuda") if rows is None else torch.from_numpy(rows).cuda()
    return engine.novelty_fit(clf, Xd, rows, torch.from_numpy(y).cuda(), C, stats=stats)


def head_with(clf, C, fit, seed=0):
    from genomad_b200 import engine, weights as W
    h = engine.Head(clf, W.HeadFile(W.initial_head(C, seed), tuple(f"c{i}" for i in range(C)), ""))
    h.set_novelty(fit.center, fit.whitening, fit.means)
    return h


def check_fit(X, y, C, fit, label):
    ref = R.fit(X, y, C)
    mu_bar, c_bar = R.sum_bar(X, y, C)
    err_mu = np.abs(fit.class_means - ref["mu"])
    assert (err_mu <= mu_bar).all(), f"{label}: mu off by {(err_mu / np.maximum(mu_bar, 1e-300)).max():.3g} of its bar"
    assert (np.abs(fit.center - ref["center"]) <= c_bar).all(), f"{label}: center"
    s_bar = R.scatter_bar(ref, mu_bar)
    err_s = np.abs(fit.scatter - ref["S"])
    assert (err_s <= s_bar).all(), f"{label}: S off by {(err_s / np.maximum(s_bar, 1e-300)).max():.3g} of its bar"
    assert np.array_equal(fit.scatter, fit.scatter.T)
    p_bar, m_bar = R.whitening_bar(ref, len(X))
    err_p = np.abs(fit.whitening - ref["P"]).max()
    err_m = np.abs(fit.means - ref["m"]).max()
    assert err_p <= p_bar, f"{label}: P off by {err_p:.3g}, bar {p_bar:.3g}"
    assert err_m <= m_bar, f"{label}: m off by {err_m:.3g}, bar {m_bar:.3g}"
    assert not np.triu(fit.whitening, 1).any() and (np.diagonal(fit.whitening) > 0).all()
    print(f"{label}: mu {(err_mu / np.maximum(mu_bar, 1e-300)).max():.2g}, S {(err_s / np.maximum(s_bar, 1e-300)).max():.2g}, "
          f"P {err_p / p_bar:.2g}, m {err_m / m_bar:.2g} of their bars; kappa {np.linalg.cond(ref['Sigma']):.3g}")
    return ref


def check_distances(torch, clf, C, fit, x, label):
    h = head_with(clf, C, fit)
    got = h.novelty(torch.from_numpy(x).cuda()).cpu().numpy()
    h.close()
    want, bar = R.distance_bound(x, fit.center, fit.whitening, fit.means)
    err = np.abs(got.astype(np.float64) - want)
    assert (err <= bar).all(), f"{label}: D off by {(err / bar).max():.3g} of its bound"
    assert (err <= 1e-6 * want + 1e-9).all(), f"{label}: D off by more than 1e-6 D + 1e-9"
    return got


CASES = [("gauss", 1024, 3), ("relu", 1024, 2), ("scaled", 1024, 32), ("gauss", 15, 2), ("relu", 16, 3), ("gauss", 17, 2),
         ("scaled", 63, 3), ("gauss", 64, 2), ("relu", 65, 32), ("gauss", 8193, 3), ("relu", 100_000, 32),
         ("scaled", 100_000, 2)]


@pytest.mark.parametrize("kind,N,C", CASES)
def test_fit_and_distances_against_oracle(torch, clf, kind, N, C):
    X, y = make_rows(kind, N, C, seed=N + C)
    fit = gpu_fit(torch, clf, X, y, C)
    check_fit(X, y, C, fit, f"{kind} N={N} C={C}")
    n_score = min(N, 2000)
    for n in sorted({1, 15, 16, 17, 63, 64, 65, n_score} & set(range(1, n_score + 1))):
        check_distances(torch, clf, C, fit, X[:n], f"{kind} N={N} C={C} n={n}")
    # typical training rows sit near D = 1 for their own class
    d_own = check_distances(torch, clf, C, fit, X[:n_score], "own")[np.arange(n_score), y[:n_score]]
    print(f"{kind} N={N} C={C}: median own-class D {np.median(d_own):.3f}")


def test_class_with_one_row_and_fit_subset(torch, clf):
    X, y = make_rows("gauss", 3000, 3, seed=7)
    y[:] = np.where(y == 2, 1, y)
    y[1234] = 2                                             # class 2: one row
    rows = np.arange(0, 3000, 2, dtype=np.int64)            # fit on the even rows; the one-row class must be among them
    rows = np.union1d(rows, [1234]).astype(np.int64)
    fit = gpu_fit(torch, clf, X, y, 3, rows=rows)
    check_fit(X[rows], y[rows], 3, fit, "one-row class")


def test_bitwise_fit_and_scoring(torch, clf):
    X, y = make_rows("relu", 20_000, 5, seed=11)
    a, b = gpu_fit(torch, clf, X, y, 5), gpu_fit(torch, clf, X, y, 5)
    for f in ("center", "whitening", "means", "class_means", "scatter"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    assert a.min_pivot == b.min_pivot
    h = head_with(clf, 5, a)
    x = torch.from_numpy(X[:3001]).cuda()
    whole = h.novelty(x).cpu().numpy()
    parts = np.concatenate([h.novelty(x[i: j]).cpu().numpy() for i, j in ((0, 1), (1, 17), (17, 100), (100, 3001))])
    assert np.array_equal(whole, parts), "chunking changed a row's distances"
    perm = np.random.default_rng(0).permutation(3001)
    assert np.array_equal(h.novelty(x[torch.from_numpy(perm).cuda()]).cpu().numpy(), whole[perm]), "permutation"
    rep = torch.cat([x[:5]] * 40)
    assert np.array_equal(h.novelty(rep).cpu().numpy(), np.tile(whole[:5], (40, 1))), "repeats"
    h.close()


def test_fit_errors(torch, clf):
    from genomad_b200 import engine
    X, y = make_rows("gauss", 100, 3, seed=1)
    y2 = np.where(y == 1, 0, y).astype(np.int32)
    with pytest.raises(engine.GnmError, match="class 1 has no fit row"):
        gpu_fit(torch, clf, X, y2, 3)
    Xc = np.repeat(np.arange(2, dtype=np.float32)[:, None], 512, 1)[[0, 1, 0, 1]].copy()
    with pytest.raises(engine.GnmError, match="no within-class variation"):
        gpu_fit(torch, clf, Xc, np.array([0, 1, 0, 1], np.int32), 2)


# ---------------------------------------------------------------------------------------------------------------- end to end
def _write(path, seqs):
    with open(path, "w") as f:
        for name, s in seqs:
            f.write(f">{name}\n{s}\n")


def test_train_head_novelty_end_to_end(torch, tmp_path):
    import test_gpu_head_module as M
    from genomad_b200 import nn_classification as nnc, train_head, weights as W
    fa = tmp_path / "train.fna"
    M.write_set(fa, 1, 30)
    outs = []
    for k, nov in enumerate((True, True, False)):
        out = tmp_path / f"head{k}"
        train_head.main(fa, str(fa) + ".labels.tsv", out, epochs=4, batch_size=256, seed=3, validation_fraction=0.2,
                        verbose=False, novelty=nov)
        outs.append(out / "train_head.npz")
    assert outs[0].read_bytes() == outs[1].read_bytes(), "two train-head --novelty runs wrote different head files"
    w = W.load_weights()
    hn, hp = W.load_head(outs[0], w), W.load_head(outs[2], w)
    assert hp.novelty is None and hn.novelty is not None
    for k in W.HEAD_KEYS:
        assert np.array_equal(hn.arrays[k], hp.arrays[k])
    cal = hn.novelty["novelty_calibration"]
    # score the training FASTA: the validation sequences' novelty must be members of the calibration set, bitwise
    nnc.main(fa, tmp_path / "scored_nov", False, 128, False, 2, False, False, head=outs[0])
    nnc.main(fa, tmp_path / "scored_plain", False, 128, False, 2, False, False, head=outs[2])
    d1, d2 = tmp_path / "scored_nov" / "train_nn_classification", tmp_path / "scored_plain" / "train_nn_classification"
    a, b = np.load(d1 / "train_nn_classification_head.npz"), np.load(d2 / "train_nn_classification_head.npz")
    assert np.array_equal(a["predictions"], b["predictions"]), "a novelty model changed the head's class scores"
    assert not (d2 / "train_nn_classification_head_novelty.npz").exists()
    z = np.load(d1 / "train_nn_classification_head_novelty.npz")
    nov = z["novelty"]
    members = np.isin(nov, cal)
    assert members.sum() >= len(cal), f"only {members.sum()} sequences' novelty are calibration values ({len(cal)})"
    assert set(cal.tolist()) <= set(nov.tolist()), "a calibration value is not the novelty of any sequence"
    assert (z["p_value"][members] > 0).all() and np.isfinite(nov).all()
    print(f"calibration: {len(cal)} values, median {np.median(cal):.3f}; all sequences: median novelty {np.median(nov):.3f}")


def test_held_out_class_is_more_novel(torch, tmp_path):
    """A head trained on gc35 and gc65 only: the held-out motif class should be more novel than held-out sequences of the
    trained classes.  Unmeasured before this test; the medians are printed."""
    import test_gpu_head_module as M
    from genomad_b200 import nn_classification as nnc, train_head
    fa = tmp_path / "two.fna"
    rng = np.random.default_rng(21)
    seqs = [(f"t_{k}_{i}", M._contig(rng, k)) for i in range(30) for k in ("gc35", "gc65")]
    _write(fa, seqs)
    with open(str(fa) + ".labels.tsv", "w") as f:
        f.write("seq_name\tclass\n")
        f.writelines(f"{n}\t{n.split('_')[1]}\n" for n, _ in seqs)
    train_head.main(fa, str(fa) + ".labels.tsv", tmp_path / "h", epochs=4, batch_size=256, seed=1, verbose=False, novelty=True)
    test = tmp_path / "test.fna"
    rng = np.random.default_rng(22)
    _write(test, [(f"q_{k}_{i}", M._contig(rng, k)) for i in range(15) for k in ("gc35", "gc65", "motif")])
    nnc.main(test, tmp_path / "q", False, 128, False, 2, False, False, head=tmp_path / "h" / "two_head.npz")
    z = np.load(tmp_path / "q" / "test_nn_classification" / "test_nn_classification_head_novelty.npz")
    kind = np.array([str(n).split("_")[1] for n in z["contig_names"]])
    med_in = float(np.median(z["novelty"][kind != "motif"]))
    med_out = float(np.median(z["novelty"][kind == "motif"]))
    print(f"median novelty: trained classes {med_in:.3f}, held-out class {med_out:.3f}; median p "
          f"{np.median(z['p_value'][kind != 'motif']):.3f} / {np.median(z['p_value'][kind == 'motif']):.3f}")
    assert med_out > med_in
