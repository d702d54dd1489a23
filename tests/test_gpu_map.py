"""
The embedding map on an H100, stage by stage against the fp64 oracle of tests/map_ref.py, each stage on the device's own output
of the stage before (include/gnm.h, DESIGN.md "Embedding map"):
  * memberships: rho bitwise; sigma solves its equation within umap-learn's 1e-5 (or ends its 64 steps, or sits at its floor);
    w and the fuzzy union within 4 fp64 roundings of the oracle's on the device's rho and sigma; the emitting entries exact;
  * the CSR graph equal to the oracle's on the device's union;
  * the top-2 subspace against numpy.linalg.eigh of the device's S where l2 / l3 >= 1.1;
  * the initialisation bitwise the oracle's on the device's projections, and those within fp64 rounding;
  * one epoch from a given Y within the a-priori bound of map_ref.epoch_bound, with the same samples;
  * whole runs: bitwise repeatable, seed-dependent, and as trustworthy as the oracle's on blobs and on encoder embeddings of
    composition contigs;
  * edge cases: n = k + 1, exact duplicates, zero rows, all rows identical, n at the covariance kernels' block edges.
"""
import numpy as np
import pytest

import map_ref as R

pytestmark = pytest.mark.gpu
U64 = 2.0 ** -53


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch


@pytest.fixture(scope="module")
def blob_rows():
    return R.blobs()


def stages(torch, x, k, epochs):
    from genomad_b200 import engine as E
    rows = torch.from_numpy(x).cuda()
    sim, idx = E.embedding_neighbours(rows, None, k)
    m = E.map_membership(sim, idx)
    return rows, sim, idx, m, E.map_graph(m.union, idx, epochs)


def test_membership_and_graph(torch, blob_rows):
    x = blob_rows[0][:600]
    k, epochs = 15, 500
    _, sim, idx, m, g = stages(torch, x, k, epochs)
    s, ix = sim.cpu().numpy(), idx.cpu().numpy()
    mean_d, rho, _, steps, _, _ = R.membership(s, ix)
    assert np.array_equal(m.rho.cpu().numpy(), rho)
    assert abs(m.mean_d.item() - mean_d) <= 1e-12 * mean_d
    d = 1.0 - s.astype(np.float64)
    sg = m.sigma.cpu().numpy()
    res = np.abs(R.psum(d, rho[:, None], sg[:, None]) - np.log2(k + 1))
    floor_ = 1e-3 * np.where(rho > 0, d.mean(1), mean_d)
    ok = (res < 1e-5 * (1 + 1e-9)) | (sg == floor_) | (steps == 64)
    assert ok.all(), np.flatnonzero(~ok)[:5]
    w = m.w.cpu().numpy()
    x_ = d - rho[:, None]
    w_ref = np.where(x_ > 0, np.exp(-np.maximum(x_, 0) / sg[:, None]), 1.0)
    assert np.all(np.abs(w - w_ref) <= 4 * U64 * w_ref)
    un = m.union.cpu().numpy()
    emit = np.full(un.shape, -1.0)
    for i in range(len(ix)):
        for p in range(k):
            j = ix[i, p]
            q = np.flatnonzero(ix[j] == i)
            b = w[j, q[0]] if len(q) else 0.0
            if not len(q) or i < j:
                emit[i, p] = w[i, p] + b - w[i, p] * b
    assert np.array_equal(un < 0, emit < 0)
    assert np.all(np.abs(un - emit) <= 4 * U64 * np.abs(emit))
    row_ptr, col, wt, eps = R.graph(un, ix, epochs)
    assert np.array_equal(g.row_ptr.cpu().numpy(), row_ptr)
    assert np.array_equal(g.col.cpu().numpy(), col)
    assert np.array_equal(g.weight.cpu().numpy(), wt)
    assert np.array_equal(g.eps.cpu().numpy(), eps)
    for r in range(len(ix)):
        assert np.all(np.diff(col[row_ptr[r]: row_ptr[r + 1]]) > 0)


@pytest.mark.parametrize("n", [600, 4095, 4097, 8191, 8193])
def test_pca_subspace_and_init(torch, n):
    from genomad_b200 import engine as E
    x = R.blobs(n, 3, 3)[0]                                            # three blobs: a separated top-2 subspace
    rows = torch.from_numpy(x).cuda()
    xh, center, S, V = E.map_pca(rows)
    xh_ref = R.normalize(x)
    assert np.all(np.abs(xh.cpu().numpy() - xh_ref) <= 2.0 ** -23 * np.abs(xh_ref))   # one fp32 rounding of the fp64 quotient
    Sg, Vg = S.cpu().numpy(), V.cpu().numpy()
    _, c_ref, S_ref, _ = R.pca(x)
    assert np.abs(center.cpu().numpy() - c_ref).max() <= 1e-12
    assert np.abs(Sg - S_ref).max() <= 1e-10 * np.abs(S_ref).max()
    lam, vec = np.linalg.eigh(Sg)
    lam, vec = lam[::-1], vec[:, ::-1]
    assert lam[1] / lam[2] >= 1.1, "the test set must separate the top-2 subspace"
    P_ref, P = vec[:, :2] @ vec[:, :2].T, Vg.T @ Vg
    assert np.abs(P - P_ref).max() <= 1e-9
    assert np.abs(Vg @ Vg.T - np.eye(2)).max() <= 1e-12
    for c in range(2):                                                  # each vector, where its eigenvalue is separated
        v = vec[:, c] * np.sign(vec[np.argmax(np.abs(vec[:, c])), c])
        if lam[c] / lam[c + 1] >= 1.01:
            assert np.abs(Vg[c] - v).max() <= 1e-8
    Y, proj = E.map_init(xh, center, V, 7, projection=True)
    pr = proj.cpu().numpy()
    p_ref = (xh.cpu().numpy().astype(np.float64) - center.cpu().numpy()) @ Vg.T
    assert np.abs(pr - p_ref).max() <= 1e-13 * max(1.0, np.abs(p_ref).max())
    assert np.array_equal(Y.cpu().numpy(), R.init_from_projection(pr, 7))


@pytest.mark.parametrize("e", [1, 2, 57, 250, 499])
def test_one_epoch_within_bound(torch, blob_rows, e):
    from genomad_b200 import engine as E
    x = blob_rows[0][:800]
    epochs, seed = 500, 3
    rows, _, idx, m, g = stages(torch, x, 15, epochs)
    xh, center, _, V = E.map_pca(rows)
    Y = E.map_init(xh, center, V, seed)
    Y = E.map_epochs(g, Y, epochs, seed, 1, 40)                    # a layout with close pairs, clipped terms and spread
    out = E.map_epochs(g, Y, epochs, seed, e, e + 1).cpu().numpy().astype(np.float64)
    y = Y.cpu().numpy()
    G = [a.cpu().numpy() for a in (g.row_ptr, g.col, g.eps)]
    ref = R.epoch(*G, y, e, epochs, seed)
    bound = R.epoch_bound(*G, y, e, epochs, seed)
    worst = (np.abs(out - ref) / bound).max()
    print(f"epoch {e}: worst error / bound = {worst:.3f}")
    assert worst <= 1.0


def _run(torch, x, k, epochs, seed):
    from genomad_b200 import engine as E
    return E.embedding_map(torch.from_numpy(x).cuda(), k, epochs, seed).cpu().numpy()


def test_whole_runs_blobs(torch, blob_rows):
    x, lab = blob_rows
    a = _run(torch, x, 15, 500, 0)
    b = _run(torch, x, 15, 500, 0)
    c = _run(torch, x, 15, 500, 1)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert not np.array_equal(a, c)
    tw, acc = R.trustworthiness(x, a), R.knn_accuracy(a, lab)
    tw_ref = R.trustworthiness(x, R.run(x, 15, 500, 0))
    print(f"blobs: trustworthiness {tw:.4f} (oracle {tw_ref:.4f}), 15-NN accuracy {acc:.4f}")
    assert tw >= 0.9 and acc == 1.0
    assert abs(tw - tw_ref) <= 0.02


def test_composition_contigs(torch, tmp_path):
    from genomad_b200 import nn_classification as nnc
    from test_gpu_head_module import write_set
    fa = tmp_path / "comp.fna"
    write_set(fa, 11, 100)
    nnc.main(fa, tmp_path / "out", False, 128, False, 2, False, False, write_embeddings=True)
    z = np.load(tmp_path / "out" / "comp_nn_classification" / "comp_nn_classification_embeddings.npz")
    x = z["embeddings"].astype(np.float32)
    y = _run(torch, x, 15, 500, 0)
    tw, tw_ref = R.trustworthiness(x, y), R.trustworthiness(x, R.run(x, 15, 500, 0))
    print(f"composition contigs (n = {len(x)}): trustworthiness {tw:.4f}, oracle {tw_ref:.4f}")
    assert abs(tw - tw_ref) <= 0.02


def _check_map(y, n):
    assert y.shape == (n, 2) and y.dtype == np.float32 and np.isfinite(y).all()


def test_edge_cases(torch):
    from genomad_b200 import engine as E
    base = R.blobs(40, 4, 9)[0]
    _check_map(_run(torch, base[:16], 15, 50, 0), 16)                  # n = k + 1
    dup = np.concatenate([base, base[:10], base[:10]])                  # exact duplicates start apart and stay finite
    y = _run(torch, dup, 15, 100, 0)
    _check_map(y, len(dup))
    assert not np.array_equal(y[0], y[40])
    zero = base.copy()
    zero[[3, 17]] = 0                                                  # zero rows: d = 1 to everything
    _check_map(_run(torch, zero, 10, 100, 0), len(zero))
    same = np.repeat(base[:1], 30, axis=0)                              # S = 0: the map starts from the noise alone
    rows = torch.from_numpy(same).cuda()
    xh, center, S, V = E.map_pca(rows)
    assert not S.any()
    Y, proj = E.map_init(xh, center, V, 4, projection=True)
    assert not proj.any()
    assert np.array_equal(Y.cpu().numpy(), R.init_from_projection(np.zeros((30, 2)), 4))
    _check_map(_run(torch, same, 15, 100, 4), 30)
    with pytest.raises(ValueError):
        E.embedding_map(rows, 30)


def test_module_end_to_end(torch, tmp_path, blob_rows):
    from genomad_b200 import embedding_map as EM
    x = blob_rows[0][:500]
    p = tmp_path / "m_nn_classification_embeddings.npz"
    np.savez(p, contig_names=np.array([f"c{i}" for i in range(len(x))]), embeddings=x)
    EM.main(p, tmp_path / "out", 15, None, 2, False)
    z = np.load(tmp_path / "out" / "m_embedding_map.npz")
    assert np.array_equal(z["coordinates"], _run(torch, x, 15, 500, 2))
    assert int(z["epochs"]) == 500 and int(z["k"]) == 15 and int(z["seed"]) == 2
