"""
CPU tests of the embedding map (no GPU): the fp64 oracle of tests/map_ref.py against its own statements (sigma's equation, the
sampling rule, a and b, the map's quality on blobs), the one-epoch bound against an fp32 emulation and three injected faults,
and the embedding-map module and CLI with the neighbour search and the layout replaced by stand-ins.
"""
import numpy as np
import pytest
import torch
from click.testing import CliRunner

import map_ref as R
from genomad_b200 import cli, embedding_map as EM, embedding_neighbours as EN, engine
from test_neighbours_cpu import install as install_neighbours, rows, write_npz


def test_sigma_solves_its_equation():
    x, _ = R.blobs(300, 4, 1)
    x[7] = 0
    x[8] = x[9]
    for k in (1, 5, 15, 64):
        sim, idx = R.knn(x, k)
        mean_d, rho, sigma, steps, w, _ = R.membership(sim, idx)
        d = 1.0 - sim.astype(np.float64)
        floor_ = 1e-3 * np.where(rho > 0, d.mean(1), mean_d)
        res = np.abs(R.psum(d, rho[:, None], sigma[:, None]) - np.log2(k + 1))
        assert np.all((res < 1e-5) | (steps == 64) | (sigma == floor_))
        assert np.all(w.max(1) == 1.0)                                 # the entry at rho has f(0) = 1


def _accumulated(eps, epochs):
    nxt, out = eps, []
    for n in range(epochs):
        if nxt <= n:
            out.append(n)
            nxt += eps
    return out


def test_sampling_rule_is_the_accumulated_schedule():
    """floor(e / eps) > floor((e - 1) / eps) against umap-learn's running sum over 500 epochs.  In exact arithmetic they agree;
    in fp64 they part only where e / eps is an integer in exact arithmetic (w = m / 500 and the like): there one rule samples
    at e and the other at e + 1.  Those are the boundary cases, and the only ones."""
    epochs = 500
    ws = np.concatenate([np.linspace(1 / epochs, 1, 4000), 1 / np.arange(1, epochs + 1), np.arange(1, epochs + 1) / epochs])
    boundary = 0
    for w in ws:
        eps = 1.0 / w
        closed = np.flatnonzero(R.sampled(eps, np.arange(epochs))).tolist()
        acc = _accumulated(eps, epochs)
        if closed == acc:
            continue
        boundary += 1
        assert abs(len(closed) - len(acc)) <= 1
        for e in set(closed) ^ set(acc):
            assert min(abs(q - round(q)) for q in (e * w, (e - 1) * w)) <= 1e-9, (w, e)
    assert boundary < len(ws) // 10


def test_a_b_match_curve_fit():
    from scipy.optimize import curve_fit
    xv = np.linspace(0, 3, 300)
    yv = np.where(xv < 0.1, 1.0, np.exp(-(xv - 0.1)))
    (a, b), _ = curve_fit(lambda x, a, b: 1.0 / (1.0 + a * x ** (2 * b)), xv, yv)
    assert abs(a - engine.MAP_A) <= 1e-6 and abs(b - engine.MAP_B) <= 1e-6


def test_oracle_map_of_blobs():
    x, lab = R.blobs()
    y = R.run(x, 15, 500, 0)
    assert R.trustworthiness(x, y) >= 0.9
    assert R.knn_accuracy(y, lab) == 1.0


def _emulate_fp32(row_ptr, col, eps, Y, e, epochs, seed):
    """The kernel's epoch in NumPy fp32, summed per vertex in a different order (all attractions, then the negatives)."""
    f = np.float32
    a, b = f(R.A32), f(R.B32)
    n = len(Y)
    rows_ = np.repeat(np.arange(n), np.diff(row_ptr))
    p = np.flatnonzero(R.sampled(eps, e))
    i, j = rows_[p], col[p]
    F = np.zeros((n, 2), np.float32)

    def att(dy):
        d2 = (dy * dy).sum(1, dtype=np.float32)
        with np.errstate(divide="ignore", invalid="ignore"):
            gc = np.where(d2 > 0, (f(-2) * a * b) * np.power(d2, b - f(1)) / (a * np.power(d2, b) + f(1)), f(0)).astype(f)
        return np.clip(gc[:, None] * dy, -4, 4).astype(f)

    def rep(dy):
        d2 = (dy * dy).sum(1, dtype=np.float32)
        gc = np.where(d2 > 0, (f(2) * b) / ((f(0.001) + d2) * (a * np.power(d2, b) + f(1))), f(0)).astype(f)
        return np.clip(gc[:, None] * dy, -4, 4).astype(f)

    np.add.at(F, i, f(2) * att((Y[i] - Y[j]).astype(f)))
    neg = R.negatives(p, e, seed, n)
    for s in range(5):
        kk = neg[:, s]
        keep = kk != i
        np.add.at(F, i[keep], rep((Y[i[keep]] - Y[kk[keep]]).astype(f)))
    return (Y + f(R.alpha(e, epochs)) * F).astype(f)


@pytest.fixture(scope="module")
def epoch_case():
    x, _ = R.blobs(400, 4, 2)
    sim, idx = R.knn(x, 15)
    union = R.membership(sim, idx)[-1]
    row_ptr, col, _, eps = R.graph(union, idx, 200)
    xh, center, _, V = R.pca(x)
    Y = R.init_from_projection((xh.astype(np.float64) - center) @ V.T, 0)
    for e in range(1, 30):
        Y = R.epoch(row_ptr, col, eps, Y, e, 200, 0).astype(np.float32)
    Y[1] = Y[0] + np.float32(1e-3)                 # a near-coincident pair: clipped terms
    return row_ptr, col, eps, Y


@pytest.mark.parametrize("e", [1, 2, 30, 199])
def test_epoch_bound_holds_for_fp32(epoch_case, e):
    row_ptr, col, eps, Y = epoch_case
    ref = R.epoch(row_ptr, col, eps, Y, e, 200, 0)
    bound = R.epoch_bound(row_ptr, col, eps, Y, e, 200, 0)
    got = _emulate_fp32(row_ptr, col, eps, Y, e, 200, 0).astype(np.float64)
    assert np.all(np.abs(got - ref) <= bound)


@pytest.mark.parametrize("fault", [dict(att_factor=1.0), dict(n_neg=4), dict(clip=8.0), dict(clip=None)])
def test_epoch_bound_catches_faults(epoch_case, fault):
    row_ptr, col, eps, Y = epoch_case
    e = 30
    ref = R.epoch(row_ptr, col, eps, Y, e, 200, 0)
    bound = R.epoch_bound(row_ptr, col, eps, Y, e, 200, 0)
    bad = R.epoch(row_ptr, col, eps, Y, e, 200, 0, **fault)
    assert np.any(np.abs(bad - ref) > bound)


def test_noise_is_small_and_hashed():
    z = R.noise(0, 1000)
    assert z.dtype == np.float32 and np.abs(z).max() < 1e-4 and len(np.unique(z)) == z.size
    assert not np.array_equal(z, R.noise(1, 1000))


# ---- module and CLI with stand-ins
def np_layout(rows_, sim, idx, epochs, seed):
    """Stand-in for engine.map_layout: a deterministic function of the rows, the lists, the epochs and the seed."""
    x = rows_.cpu().numpy().astype(np.float64)
    s = sim.cpu().numpy().astype(np.float64).sum(1)
    return torch.from_numpy(np.stack([x[:, :7].sum(1) + s, x[:, 7:11].sum(1) + epochs + seed], 1).astype(np.float32))


@pytest.fixture(autouse=True)
def _stand_in(monkeypatch):
    for key in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(key, raising=False)
    install(monkeypatch.setattr)


def install(setattr_):
    install_neighbours(setattr_)
    setattr_(engine, "map_layout", np_layout)


def test_module_writes_tsv_and_npz(tmp_path):
    emb = rows(20, 1)
    p = write_npz(tmp_path / "s_nn_classification_embeddings.npz", 0, emb=emb)
    EM.main(p, tmp_path / "out", 4, None, 3, False)
    names = np.load(p)["contig_names"].astype(str)
    sim, idx = EN.search(emb, None, 4, __import__("genomad_b200").dist.init_process_group_if_needed())
    y = np_layout(torch.from_numpy(emb), torch.from_numpy(sim), torch.from_numpy(idx), 500, 3).numpy()
    tsv = (tmp_path / "out" / "s_embedding_map.tsv").read_text()
    assert tsv == "seq_name\tx\ty\n" + "".join(f"{n}\t{a:.6f}\t{b:.6f}\n" for n, (a, b) in zip(names, y.astype(float)))
    z = np.load(tmp_path / "out" / "s_embedding_map.npz")
    assert sorted(z.files) == ["both_strands", "coordinates", "epochs", "k", "seed", "seq_names"]
    assert z["coordinates"].dtype == np.float32 and np.array_equal(z["coordinates"], y)
    assert int(z["k"]) == 4 and int(z["epochs"]) == 500 and int(z["seed"]) == 3 and not bool(z["both_strands"])
    assert list(z["seq_names"]) == list(names)


def test_default_epochs():
    assert engine.map_default_epochs(10000) == 500 and engine.map_default_epochs(10001) == 200


@pytest.mark.parametrize("k, n, msg", [(20, 20, "smaller than"), (65, 100, r"\[1, 64\]"), (0, 10, r"\[1, 64\]")])
def test_bad_k_refused_before_device_work(tmp_path, monkeypatch, k, n, msg):
    p = write_npz(tmp_path / "s_nn_classification_embeddings.npz", 0, emb=rows(n, 2))
    monkeypatch.setattr(EN, "search", lambda *a, **kw: pytest.fail("searched"))
    with pytest.raises(ValueError, match=msg):
        EM.main(p, tmp_path / "out", k, None, 0, False)


def test_bad_epochs_and_seed(tmp_path):
    p = write_npz(tmp_path / "s_nn_classification_embeddings.npz", 0, emb=rows(10, 2))
    with pytest.raises(ValueError, match="epochs"):
        EM.main(p, tmp_path / "out", 3, 0, 0, False)
    with pytest.raises(ValueError, match="seed"):
        EM.main(p, tmp_path / "out", 3, None, -1, False)


def test_bad_npz_and_missing_both_strands(tmp_path):
    bad = tmp_path / "bad.npz"
    bad.write_bytes(b"not a zip")
    with pytest.raises(EN.EmbeddingsFileError):
        EM.main(bad, tmp_path / "out", 3, None, 0, False)
    p = write_npz(tmp_path / "s_nn_classification_embeddings.npz", 0, emb=rows(10, 2))
    with pytest.raises(EN.EmbeddingsFileError, match="both-strands"):
        EM.main(p, tmp_path / "out", 3, None, 0, False, both_strands=True)


def test_both_strands_reads_its_key(tmp_path):
    fwd, both = rows(12, 3), rows(12, 4)
    p = tmp_path / "b_nn_classification_embeddings.npz"
    np.savez(p, contig_names=np.array([f"c{i}" for i in range(12)]), embeddings=fwd, embeddings_both_strands=both)
    EM.main(p, tmp_path / "out", 3, 10, 0, False, both_strands=True)
    z = np.load(tmp_path / "out" / "b_embedding_map.npz")
    assert bool(z["both_strands"])
    sim, idx = EN.search(both, None, 3, __import__("genomad_b200").dist.init_process_group_if_needed())
    y = np_layout(torch.from_numpy(both), torch.from_numpy(sim), torch.from_numpy(idx), 10, 0).numpy()
    assert np.array_equal(z["coordinates"], y)


def test_cli(tmp_path):
    p = write_npz(tmp_path / "s_nn_classification_embeddings.npz", 0, emb=rows(15, 5))
    r = CliRunner().invoke(cli.cli, ["embedding-map", str(p), str(tmp_path / "out"), "-k", "5", "--epochs", "7", "--seed", "9",
                                     "--quiet"])
    assert r.exit_code == 0, r.output
    z = np.load(tmp_path / "out" / "s_embedding_map.npz")
    assert int(z["k"]) == 5 and int(z["epochs"]) == 7 and int(z["seed"]) == 9
    r = CliRunner().invoke(cli.cli, ["embedding-map", str(p), str(tmp_path / "out2"), "-k", "15"])
    assert r.exit_code != 0
