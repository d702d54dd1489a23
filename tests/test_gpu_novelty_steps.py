"""
Head novelty step by step on an H100 (run with -s for the error / bound ratios and kappa(Sigma)).  Each step of the fit is
held to the derived bounds of tests/novelty_ref.py on its own computed inputs (shrinkage and Cholesky on the device's S; the
triangular inverse on its L; the whitened means on its P, mu and center), on top of the forward-error bars against the fp64
oracle fit that tests/test_gpu_head_novelty.py uses.  L is read from the fit workspace, whose layout this file mirrors from
NvLayout in csrc/api.cu; the S and P regions must be bitwise the returned scatter and whitening.
  * inputs: the encoder's own embeddings (composition contigs on one and both strands, the golden windows), rank-1, -8 and -64
    rows (rank 1 puts kappa(Sigma) at the shrinkage's ceiling, 1 + 512 (1 - alpha) / alpha), N from C + 1 up, offsets of 1e2
    and 1e4, columns scaled from 1e-3 to 1e3, 99.9 % of the rows in one class, one-row classes at C = 32, and fit-row lists
    that are unsorted, repeat rows, pick a subset of X, or end next to the 4,096-row sum blocks and 8,192-row scatter chunks;
  * window distances within the derived bound at every C from 2 to 32, on rows at fp32(mu_c), the center, zero rows, rows
    1e3 times the scale and rows with one huge column;
  * errors, each with its own message: a fit index of -1 or n_rows, a label of -1 or C, a NaN or infinity in a fit row; after
    each, a good fit on the same handle is bitwise that of a fresh handle;
  * end to end: nn-classification --head with a novelty head, with and without the provirus twin: distances within the
    per-contig bound of an fp64 recomputation from embed_windows, nearest_class where the margin exceeds it, p-values bitwise.
"""
import ctypes as C_
import shutil

import numpy as np
import pytest

import novelty_ref as R
from test_novelty_bounds_cpu import family, score_rows

pytestmark = pytest.mark.gpu

DIM = R.DIM
KAPPA_CEILING = 1 + DIM * (1 - R.ALPHA) / R.ALPHA


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


# ------------------------------------------------------------------------------------------------------- the fit, by steps
def nv_layout(n_fit, C):
    """Byte offsets of gnm_novelty_fit's workspace parts (NvLayout in csrc/api.cu: in this order, each 256-byte aligned)."""
    nb, nc = -(-n_fit // 4096), -(-n_fit // 8192)
    parts = (("status", 24), ("part", nb * C * DIM * 8), ("cnt", nb * C * 8), ("mu", C * DIM * 8), ("center", DIM * 8),
             ("counts", C * 8), ("spart", nc * 36 * 64 * 64 * 8), ("S", DIM * DIM * 8), ("L", DIM * DIM * 8),
             ("P", DIM * DIM * 8), ("m", C * DIM * 8))
    out, o = {}, 0
    for name, size in parts:
        out[name] = o
        o += -(-size // 256) * 256
    out["total"] = o
    return out


def fit_steps(torch, clf, X, labels, rows, C):
    """gnm_novelty_fit on rows `rows` of X (labels: one per row of X) with a workspace this test owns -> dict of the returned
    arrays plus L read from the workspace.  GnmError on a failed fit."""
    from genomad_b200 import engine
    n = len(rows)
    lay = nv_layout(n, C)
    need = int(clf.lib.gnm_novelty_fit_workspace_bytes(n, C))
    assert need == lay["total"], f"the workspace layout mirror is stale: {lay['total']} bytes, the library needs {need}"
    work = torch.empty(need + 256, dtype=torch.uint8, device="cuda")
    base = (-work.data_ptr()) % 256
    Xd = torch.from_numpy(np.ascontiguousarray(X, np.float32)).cuda()
    idx = torch.from_numpy(np.ascontiguousarray(rows, np.int64)).cuda()
    lab = torch.from_numpy(np.ascontiguousarray(labels, np.int32)).cuda()
    out = {"center": np.empty(DIM), "P": np.empty((DIM, DIM)), "m": np.empty((C, DIM)), "mu": np.empty((C, DIM)),
           "S": np.empty((DIM, DIM))}
    piv = C_.c_double()
    p = engine._ptr
    with torch.cuda.device(clf.device):
        engine._check(clf.lib, clf.lib.gnm_novelty_fit(clf._h, Xd.data_ptr(), len(X), idx.data_ptr(), n, lab.data_ptr(), C,
                                                       p(out["center"]), p(out["P"]), p(out["m"]), C_.byref(piv),
                                                       p(out["mu"]), p(out["S"]), work.data_ptr() + base, need, clf._stream()))
    torch.cuda.synchronize()
    ws = work[base: base + need].cpu().numpy()
    region = lambda name: ws[lay[name]: lay[name] + DIM * DIM * 8].view(np.float64).reshape(DIM, DIM)
    assert np.array_equal(region("S"), out["S"]), "the S region of the workspace is not the returned scatter: layout mirror"
    assert np.array_equal(region("P"), out["P"]), "the P region of the workspace is not the returned whitening: layout mirror"
    out["L"] = region("L").copy()
    out["min_pivot"] = piv.value
    return out


def check_steps(X, labels, rows, C, f, label):
    """The derived per-step bounds and the oracle forward-error bars; prints the ratios.  Returns kappa(Sigma)."""
    Xf, yf = X[rows], labels[rows]
    ref = R.fit(Xf, yf, C)
    mu_bar, c_bar = R.sum_bar(Xf, yf, C)
    r = {"mu": R._ratio(np.abs(f["mu"] - ref["mu"]), mu_bar), "center": R._ratio(np.abs(f["center"] - ref["center"]), c_bar),
         "S": R._ratio(np.abs(f["S"] - ref["S"]), R.scatter_bar(ref, mu_bar))}
    A, tr = R.shrink(f["S"])
    assert not np.triu(f["L"], 1).any(), f"{label}: L has entries above the diagonal"
    r["chol"] = R.cholesky_ratio(f["L"], A)
    r["pivot"] = R.pivot_ratio(f["min_pivot"], f["L"])
    r["inverse"] = R.inverse_ratio(f["L"], f["P"])
    r["means"] = R.whiten_ratio(f["P"], f["mu"], f["center"], f["m"])
    p_bar, m_bar = R.whitening_bar(ref, len(Xf))
    r["P oracle"] = np.abs(f["P"] - ref["P"]).max() / p_bar
    r["m oracle"] = np.abs(f["m"] - ref["m"]).max() / m_bar
    kappa = float(np.linalg.cond(A))
    print(f"\n{label}: N={len(rows)} C={C} kappa(Sigma) {kappa:.4g}; error / bound "
          + ", ".join(f"{k} {v:.2g}" for k, v in r.items()))
    assert np.array_equal(f["S"], f["S"].T) and not np.triu(f["P"], 1).any()
    for k, v in r.items():
        assert v <= 1.0, f"{label}: {k} at {v:.3g} of its bound"
    return kappa


def head_with(clf, C, f):
    from genomad_b200 import engine, weights as W
    h = engine.Head(clf, W.HeadFile(W.initial_head(C, 0), tuple(f"c{i}" for i in range(C)), ""))
    h.set_novelty(f["center"], f["P"], f["m"])
    return h


def check_distances(torch, clf, C, f, x, label):
    h = head_with(clf, C, f)
    got = h.novelty(torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()).cpu().numpy()
    h.close()
    D, bound = R.distance_bound(x, f["center"], f["P"], f["m"])
    ratio = R._ratio(np.abs(got.astype(np.float64) - D), bound)
    print(f"{label}: distances {ratio:.2g} of their bound ({len(x)} rows, median D {np.median(D):.3g})")
    assert ratio <= 1.0, f"{label}: a window distance at {ratio:.3g} of its bound"
    return got


def run_case(torch, clf, X, y, C, label, rows=None):
    rows = np.arange(len(X), dtype=np.int64) if rows is None else np.asarray(rows, np.int64)
    f = fit_steps(torch, clf, X, y, rows, C)
    kappa = check_steps(X, y, rows, C, f, label)
    check_distances(torch, clf, C, f, score_rows(X[rows], y[rows], C, f, np.random.default_rng(len(rows))), label)
    return f, kappa


# ------------------------------------------------------------------------------------------------------ real embeddings
def _composition(clf, seed, per_class, both_strands):
    import test_gpu_head_module as M
    rng = np.random.default_rng(seed)
    seqs, cls = [], []
    for i in range(per_class):
        for c, kind in enumerate(M.CLASSES):
            seqs.append(M._contig(rng, kind))
            cls.append(c)
    seq, offs = clf.contig_buffers(seqs)
    X, y = [], []
    for rev in ((False, True) if both_strands else (False,)):
        start, length, woff = clf.contig_windows(seq, offs, reverse=rev)
        X.append(clf.embed_windows(seq, start, length, reverse=rev)[1].cpu().numpy())
        y.append(np.repeat(np.array(cls, np.int32), np.diff(woff.cpu().numpy())))
    return np.concatenate(X), np.concatenate(y)


@pytest.mark.parametrize("both_strands", [False, True])
def test_encoder_embeddings_of_composition_contigs(torch, clf, both_strands):
    X, y = _composition(clf, 5, 40, both_strands)
    print(f"\nembeddings: {len(X)} windows, {np.mean(X == 0):.0%} exact zeros, {int((X == 0).all(0).sum())} dead columns")
    run_case(torch, clf, X, y, 3, f"composition contigs{' both strands' if both_strands else ''}")


def test_encoder_embeddings_of_golden_windows(torch, clf, golden_dir):
    z = np.load(golden_dir / "reference_encoder_golden.npz")
    X = []
    for k in ("graph_tokens", "tokens_tokens"):
        tok = torch.from_numpy(np.ascontiguousarray(z[k], np.uint16).view(np.int16)).cuda().view(torch.uint16)
        X.append(clf.embed_tokens(tok)[1].cpu().numpy())
    y = np.repeat(np.arange(2, dtype=np.int32), [len(X[0]), len(X[1])])
    run_case(torch, clf, np.concatenate(X), y, 2, "golden windows")


# ---------------------------------------------------------------------------------------------------- synthetic families
@pytest.mark.parametrize("kind", ["rank1", "rank8", "rank64", "offset1e2", "offset1e4", "colscale", "imbalance", "onerow32",
                                  "tiny"])
def test_families(torch, clf, kind):
    X, y, C = family(kind, seed=3)
    f, kappa = run_case(torch, clf, X, y, C, kind)
    if kind in ("rank1", "tiny"):
        assert abs(kappa / KAPPA_CEILING - 1) < 0.01, f"{kind}: kappa {kappa:.5g}, not the ceiling {KAPPA_CEILING:.5g}"


@pytest.mark.parametrize("N,C", [(3, 2), (33, 32), (300, 3)])
def test_fewer_rows_than_columns(torch, clf, N, C):
    rng = np.random.default_rng(N)
    y = np.concatenate([np.arange(C), rng.integers(0, C, N - C)]).astype(np.int32)
    X = (rng.normal(0, 2, (C, DIM))[y] + rng.normal(0, 1, (N, DIM))).astype(np.float32)
    run_case(torch, clf, X, y, C, f"N={N} < 512")


# ------------------------------------------------------------------------------------------------------------ fit-row lists
def test_fit_row_lists(torch, clf):
    X, y, C = family("offset1e2", seed=4)                     # 3,000 rows
    rng = np.random.default_rng(0)
    perm = rng.permutation(len(X))
    a = fit_steps(torch, clf, X, y, perm, C)
    check_steps(X, y, perm, C, a, "unsorted")
    dup = np.concatenate([perm[:1000], perm[:500], perm[2000:]])
    check_steps(X, y, dup, C, fit_steps(torch, clf, X, y, dup, C), "duplicates")
    sub = np.sort(rng.choice(len(X), 1700, replace=False))
    sub = np.union1d(sub, [np.flatnonzero(y == c)[0] for c in range(C)])
    check_steps(X, y, sub, C, fit_steps(torch, clf, X, y, sub, C), "strict subset")


@pytest.mark.parametrize("n_fit", [4095, 4096, 4097, 8191, 8192, 8193, 16385])
def test_fit_sizes_at_block_and_chunk_edges(torch, clf, n_fit):
    rng = np.random.default_rng(n_fit)
    n_rows, C = n_fit + 777, 4
    y = rng.integers(0, C, n_rows).astype(np.int32)
    X = np.maximum(rng.normal(0, 1, (C, DIM))[y] + rng.normal(0, 1, (n_rows, DIM)), 0).astype(np.float32)
    rows = rng.permutation(n_rows)[:n_fit]                    # unsorted, a strict subset of X
    assert (np.bincount(y[rows], minlength=C) > 0).all()
    check_steps(X, y, rows, C, fit_steps(torch, clf, X, y, rows, C), f"n_fit={n_fit}")


# ------------------------------------------------------------------------------------------------------ distances at every C
@pytest.mark.parametrize("C", range(2, 33))
def test_distances_at_every_class_count(torch, clf, C):
    from genomad_b200 import engine
    rng = np.random.default_rng(100 + C)
    N = 600 + 40 * C
    y = np.concatenate([np.arange(C), rng.integers(0, C, N - C)]).astype(np.int32)
    X = (rng.normal(0, 2, (C, DIM))[y] + rng.normal(0, 1, (N, DIM)) * rng.uniform(0.1, 3, DIM) + 5).astype(np.float32)
    fit = engine.novelty_fit(clf, torch.from_numpy(X).cuda(), torch.arange(N, device="cuda"), torch.from_numpy(y).cuda(), C,
                             stats=True)
    f = {"center": fit.center, "P": fit.whitening, "m": fit.means, "mu": fit.class_means}
    x = score_rows(X, y, C, f, rng)
    got = check_distances(torch, clf, C, f, x, f"C={C}")
    at_mu = got[min(N, 500): min(N, 500) + C]
    assert (np.diagonal(at_mu) < 1e-3 * np.median(got[:100])).all(), "a row at fp32(mu_c) is not near class c"


# ------------------------------------------------------------------------------------------------------------------ errors
@pytest.fixture(scope="module")
def fresh(torch):
    """A second handle, for the fit a failure on the first must not change."""
    from genomad_b200 import engine
    c = engine.Classifier(None, device=0, max_batch=64)
    yield c
    c.close()


def _bad_inputs():
    def idx(v):
        return lambda X, y, rows: (X, y, np.concatenate([rows[:10], [len(X) if v == "n_rows" else v], rows[10:]]))

    def label(v):
        def f(X, y, rows):
            y = y.copy()
            y[rows[7]] = v
            return X, y, rows
        return f

    def value(v):
        def f(X, y, rows):
            X = X.copy()
            X[rows[11], 300] = v
            return X, y, rows
        return f
    return [("index -1", idx(-1), "fit row index is outside"), ("index n_rows", idx("n_rows"), "fit row index is outside"),
            ("label -1", label(-1), "label is outside"), ("label C", label(3), "label is outside"),      # C = 3
            ("NaN", value(np.nan), "non-finite value"), ("+Inf", value(np.inf), "non-finite value"),
            ("-Inf", value(-np.inf), "non-finite value")]


@pytest.mark.parametrize("name,make,msg", _bad_inputs(), ids=[b[0] for b in _bad_inputs()])
def test_fit_errors_and_recovery(torch, clf, fresh, name, make, msg):
    from genomad_b200 import engine
    X, y, C = family("rank64", seed=9)
    rows = np.arange(len(X), dtype=np.int64)[::-1].copy()
    Xb, yb, rb = make(X, y, rows)
    with pytest.raises(engine.GnmError, match=msg):
        fit_steps(torch, clf, Xb, yb, rb, C)
    good = fit_steps(torch, clf, X, y, rows, C)
    want = fit_steps(torch, fresh, X, y, rows, C)
    for k in want:
        assert np.array_equal(good[k], want[k]), f"after '{name}' the next fit's {k} differs from a fresh handle's"


def test_no_variation_keeps_its_message(torch, clf):
    from genomad_b200 import engine
    X = np.repeat(np.arange(2, dtype=np.float32)[:, None], DIM, 1)[[0, 1, 0, 1]].copy()
    with pytest.raises(engine.GnmError, match=r"no within-class variation \(tr S = 0\)"):
        fit_steps(torch, clf, X, np.array([0, 1, 0, 1], np.int32), np.arange(4), 2)


# -------------------------------------------------------------------------------------------------------------- end to end
def _read_fasta(path):
    names, seqs = [], []
    for block in path.read_text().split(">")[1:]:
        head, _, body = block.partition("\n")
        names.append(head.split()[0])
        seqs.append(body.replace("\n", ""))
    return names, seqs


def _check_novelty_file(clf, npz, names_key, fasta, model, label):
    names, seqs = _read_fasta(fasta)
    z = np.load(npz)
    assert list(z[names_key]) == names
    seq, offs = clf.contig_buffers(seqs)
    start, length, woff = clf.contig_windows(seq, offs)
    emb = clf.embed_windows(seq, start, length)[1].cpu().numpy()
    D, bound = R.distance_bound(emb, model["novelty_center"], model["novelty_whitening"], model["novelty_means"])
    mean, cb = R.contig_bound(D, bound, woff.cpu().numpy())
    dist = z["distances"].astype(np.float64)
    has = np.diff(woff.cpu().numpy()) > 0
    ratio = R._ratio(np.abs(dist[has] - mean[has]), cb[has])
    print(f"\n{label}: {has.sum()} sequences with windows, per-contig distances {ratio:.2g} of their bound")
    assert ratio <= 1.0
    srt = np.sort(mean[has], 1)
    sure = np.flatnonzero(has)[(srt[:, 1] - srt[:, 0]) > 2 * cb[has].max(1)] if mean.shape[1] > 1 else np.flatnonzero(has)
    assert (z["nearest_class"][sure] == mean[sure].argmin(1)).all(), "nearest_class disagrees where the margin is clear"
    assert (z["nearest_class"][~has] == -1).all()
    cal = model["novelty_calibration"]
    for i, v in enumerate(z["novelty"]):
        want = R.p_value(v, cal)
        assert (np.isnan(want) and np.isnan(z["p_value"][i])) or want == z["p_value"][i], (i, want, z["p_value"][i])


def test_nn_classification_novelty_end_to_end(torch, clf, tmp_path, golden_dir):
    import test_gpu_head_module as M
    from genomad_b200 import nn_classification as nnc, weights as W
    X, y = _composition(clf, 11, 12, False)
    f = fit_steps(torch, clf, X, y, np.arange(len(X)), 3)
    model = {"novelty_center": f["center"], "novelty_whitening": f["P"], "novelty_means": f["m"],
             "novelty_calibration": np.sort(np.random.default_rng(0).uniform(0.5, 50, 25)).astype(np.float32)}
    head = tmp_path / "nov_head.npz"
    W.save_head(head, W.initial_head(3, 2), M.CLASSES, W.load_weights(), novelty=model)
    fa = tmp_path / "seeded.fna"
    M.write_set(fa, 13, 5)
    nnc.main(fa, tmp_path / "a", False, 128, False, 2, False, False, head=head)
    d = tmp_path / "a" / "seeded_nn_classification"
    _check_novelty_file(clf, d / "seeded_nn_classification_head_novelty.npz", "contig_names", fa, model, "seeded FASTA")
    assert not (d / "seeded_provirus_nn_classification_head_novelty.npz").exists()
    # the golden toy input with its find-proviruses outputs: the provirus twin too
    inp = golden_dir / "reference_module" / "input"
    out = tmp_path / "b"
    shutil.copytree(inp / "toy_find_proviruses", out / "toy_find_proviruses")
    nnc.main(inp / "toy.fna", out, False, 128, False, 2, False, False, head=head)
    d = out / "toy_nn_classification"
    _check_novelty_file(clf, d / "toy_nn_classification_head_novelty.npz", "contig_names", inp / "toy.fna", model, "toy")
    _check_novelty_file(clf, d / "toy_provirus_nn_classification_head_novelty.npz", "provirus_names",
                        inp / "toy_find_proviruses" / "toy_provirus.fna", model, "toy proviruses")
