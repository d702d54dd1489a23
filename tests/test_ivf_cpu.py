"""
CPU tests of the embedding index (no GPU):
  * the NumPy oracle of tests/ivf_ref.py on tie-free fp64 inputs: the training order is NumPy's reproduction of the hashed order,
    the build is repeatable, and the oracle catches three seeded faults (a re-seed that takes the highest best similarity, an
    unstable layout sort, a probe set off by one), and at nprobe = L its search is the exact search;
  * the embedding-index module and CLI and embedding-neighbours / embedding-map --index with NumPy stand-ins for the device:
    file keys, every refusal before any device call (bad L or nprobe, an index of another file, row count or strand key, a
    malformed index, a build under torchrun with more than one process), and the list shards of torchrun.
"""
import numpy as np
import pytest
import torch
from click.testing import CliRunner

import ivf_ref as R
from genomad_b200 import cli, embedding_index as EI, embedding_map as EM, embedding_neighbours as EN, engine
from test_neighbours_cpu import install as install_neighbours, rows, write_npz


def tiefree(n, seed):
    return np.random.default_rng(seed).standard_normal((n, 512))


def test_training_order_and_repeatable_build():
    from genomad_b200.synth import _keys, _mix32
    order = R.training_rows(5000, 4, 7)
    with np.errstate(over="ignore"):
        h = _mix32(np.arange(5000, dtype=np.int64) ^ _keys(7)[0])
    assert len(order) == 1024 and (np.diff(h[order]) >= 0).all()
    assert len(R.training_rows(100, 4, 7)) == 100
    x = tiefree(400, 1)
    a, b = R.build(x, 9, 4, 3), R.build(x, 9, 4, 3)
    assert all(np.array_equal(u, v) for u, v in zip(a, b))
    cent, rows_, off = a
    assert np.array_equal(np.sort(rows_), np.arange(400)) and off[-1] == 400


def test_full_probe_is_exact_search():
    x = tiefree(300, 2)
    cent, rows_, off = R.build(x, 6, 3, 0)
    s, i = R.search(x, x, cent, rows_, off, 7, 6, self_index0=0)
    S = R.cosine64(x, x)
    es, ei = R.top(S, 7, exclude=np.arange(300))
    assert np.array_equal(i, ei) and np.array_equal(s, es)


def test_seeded_faults_are_caught():
    x = tiefree(200, 3)
    xhat = R.normalize(x)
    train = R.training_rows(200, 10, 0)
    best, a = R.assign(R.cosine64, xhat[train], xhat[train][:10])
    a = a.copy()
    a[a == 3] = 4                                          # list 3 empty
    cent = R.centroids(xhat[train], a, 10)
    good, empty = R.reseed(cent, xhat[train], train, best, a)
    assert list(empty) == [3]
    bad = cent.copy()
    bad[empty] = xhat[train][np.lexsort((train, -best))[:1]]     # highest best similarity
    assert not np.array_equal(good, bad)
    # an unstable sort reorders rows within a list
    lists_of = np.random.default_rng(0).integers(0, 5, 500)
    rows_, _ = R.layout(lists_of, 5)
    unstable = np.argsort(lists_of, kind="quicksort")
    assert not np.array_equal(rows_, unstable)
    for l in range(5):
        assert (np.diff(rows_[lists_of[rows_] == l]) > 0).all()
    # a probe set off by one changes the search
    cent, rows_, off = R.build(x, 8, 3, 1)
    s, i = R.search(x, x, cent, rows_, off, 5, 3, self_index0=0)
    s2, i2 = R.search(x, x, cent, rows_, off, 5, 2, self_index0=0)
    s4, i4 = R.search(x, x, cent, rows_, off, 5, 4, self_index0=0)
    assert not np.array_equal(i, i2) and not np.array_equal(i, i4)


def test_chunks_and_shards():
    off = np.array([0, 0, 3, 10, 10, 30, 31])
    assert engine.ivf_chunks(off, 0, 6, 10) == [(0, 4, 0, 10), (4, 5, 10, 20), (4, 5, 20, 30), (5, 6, 30, 31)]
    assert engine.ivf_chunks(off, 2, 4, 100) == [(2, 4, 3, 10)]
    shards = [EN.list_shard(off, 3, r) for r in range(3)]
    assert shards[0][0] == 0 and shards[-1][1] == 6 and all(a[1] == b[0] for a, b in zip(shards, shards[1:]))
    assert engine.ivf_default_lists(1_000_000) == 4000 and engine.ivf_default_lists(3) == 3


# ------------------------------------------------------------------------------------------------ module stand-ins
def np_build(x, lists, iterations=20, seed=0):
    c, r, o = R.build(x.cpu().numpy(), lists, iterations, seed)
    return engine.IvfIndex(torch.from_numpy(c), torch.from_numpy(r), torch.from_numpy(o))


def np_search(query, reference, index, k, nprobe, *, ref_index0=0, self_index0=None, lists=None, probes=None,
              reference_shard=False):
    q = query.cpu().numpy()
    r = q if reference is None else reference.cpu().numpy()
    self0 = (ref_index0 if reference is None else -1) if self_index0 is None else self_index0
    engine.ivf_nprobe(nprobe, index.centroids.shape[0])
    off = index.offsets.cpu().numpy().copy()
    rows_ = index.rows.cpu().numpy()
    if reference_shard:                                    # the shard's rows in list order: put them back in row order
        full = np.zeros((len(rows_), r.shape[1]), r.dtype)
        full[rows_[off[lists[0]]:off[lists[1]]]] = r
        r = full
    if lists is not None:                                  # keep only the shard's lists: empty the others
        l0, l1 = lists
        keep = np.zeros(len(rows_), bool)
        keep[off[l0]:off[l1]] = True
        sizes = np.diff(off) * ((np.arange(len(off) - 1) >= l0) & (np.arange(len(off) - 1) < l1))
        rows_ = rows_[keep]
        off = np.concatenate([[0], np.cumsum(sizes)])
    s, i = R.search(q, r, index.centroids.cpu().numpy(), rows_, off, k, nprobe, self0)
    return torch.from_numpy(s.astype(np.float32)), torch.from_numpy(np.where(i >= 0, i + ref_index0, -1))


def install(setattr_):
    install_neighbours(setattr_)
    setattr_(engine, "ivf_build", np_build)
    setattr_(engine, "ivf_search", np_search)


@pytest.fixture(autouse=True)
def _stand_in(monkeypatch):
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    install(monkeypatch.setattr)


def make_index(tmp_path, n=40, lists=5, **kw):
    p = write_npz(tmp_path / "r_nn_classification_embeddings.npz", n, 1)
    EI.main(p, tmp_path / "ix", lists, 3, 0, False, **kw)
    return p, tmp_path / "ix" / "r_embedding_index.npz"


def test_index_file_and_search(tmp_path):
    p, ix = make_index(tmp_path)
    z = np.load(ix)
    assert set(z.files) == set(EI._KEYS) and int(z["lists"]) == 5 and str(z["embeddings_key"]) == "embeddings"
    assert z["rows"].dtype == np.int64 and z["offsets"].shape == (6,) and z["centroids"].dtype == np.float32
    EN.main(p, None, tmp_path / "o", 4, False, index=ix, nprobe=5)
    EN.main(p, None, tmp_path / "e", 4, False)
    a, b = np.load(tmp_path / "o" / "r_embedding_neighbours.npz"), np.load(tmp_path / "e" / "r_embedding_neighbours.npz")
    assert np.array_equal(a["neighbour_index"], b["neighbour_index"])      # nprobe = L: the exact search
    assert int(a["nprobe"]) == 5 and str(a["index_sha256"]) == EI.file_sha256(ix) and "nprobe" not in b.files
    q = write_npz(tmp_path / "q.npz", 6, 9)
    EN.main(q, p, tmp_path / "o2", 3, False, index=ix, nprobe=2)
    assert np.load(tmp_path / "o2" / "q_embedding_neighbours.npz")["neighbour_index"].shape == (6, 3)


@pytest.mark.parametrize("bad", ["other_file", "row_count", "strand_key", "malformed", "offsets", "rows", "nprobe_missing",
                                 "nprobe_zero", "nprobe_big", "nprobe_alone"])
def test_refusals_before_device(tmp_path, monkeypatch, bad):
    p, ix = make_index(tmp_path)
    def boom(*a, **k):
        raise AssertionError("device call before the inputs were checked")
    for name in ("ivf_search", "embedding_neighbours", "ivf_build"):
        monkeypatch.setattr(engine, name, boom)
    q, kw = p, {"index": ix, "nprobe": 2}
    if bad == "other_file":
        q = write_npz(tmp_path / "other.npz", 40, 2)
    elif bad == "row_count":
        q = write_npz(tmp_path / "short.npz", 39, 1)
    elif bad == "strand_key":
        z = dict(np.load(p))
        z["embeddings_both_strands"] = z["embeddings"]
        np.savez(tmp_path / "bs.npz", **z)
        q = tmp_path / "bs.npz"
    elif bad in ("malformed", "offsets", "rows"):
        z = dict(np.load(ix))
        if bad == "malformed":
            del z["centroids"]
        elif bad == "offsets":
            z["offsets"] = z["offsets"][::-1].copy()
        else:
            z["rows"] = np.zeros_like(z["rows"])
        np.savez(tmp_path / "bad_ix.npz", **z)
        kw["index"] = tmp_path / "bad_ix.npz"
    elif bad == "nprobe_missing":
        kw["nprobe"] = None
    elif bad == "nprobe_zero":
        kw["nprobe"] = 0
    elif bad == "nprobe_big":
        kw["nprobe"] = 6
    else:
        kw = {"nprobe": 3}
    with pytest.raises(ValueError):
        EN.main(q, None, tmp_path / "out", 3, False, both_strands=bad == "strand_key", **kw)
    with pytest.raises(ValueError):
        EM.main(q, tmp_path / "out", 3, 10, 0, False, both_strands=bad == "strand_key", **kw)
    assert not (tmp_path / "out").exists()


def test_map_refuses_padded_lists(tmp_path):
    p = write_npz(tmp_path / "m_nn_classification_embeddings.npz", 30, 5)
    EI.main(p, tmp_path / "ix", 10, 3, 0, False)
    ix = tmp_path / "ix" / "m_embedding_index.npz"
    sizes = np.diff(np.load(ix)["offsets"])
    k = int(sizes.min())                                   # the smallest list holds k rows: k - 1 others at nprobe 1
    assert 1 <= k < 29
    with pytest.raises(ValueError, match="fewer than"):
        EM.main(p, tmp_path / "out", k, 10, 0, False, index=ix, nprobe=1)
    assert not (tmp_path / "out").exists()


def test_probes_are_checked():
    ok = torch.tensor([[0, 2], [1, 0]])
    assert engine.ivf_check_probes(ok, 2, 2, 3).dtype == torch.int32
    for bad in (torch.tensor([[0, 0], [1, 2]]), torch.tensor([[0, 3], [1, 2]]), torch.tensor([[0, -1], [1, 2]]),
                torch.tensor([[0, 1, 2], [1, 2, 0]])):
        with pytest.raises(ValueError):
            engine.ivf_check_probes(bad, 2, 2, 3)


def test_build_refusals(tmp_path, monkeypatch):
    p = write_npz(tmp_path / "r.npz", 10, 1)
    for lists in (0, 11):
        with pytest.raises(ValueError):
            EI.main(p, tmp_path / "ix", lists, 3, 0, False)
    with pytest.raises(ValueError):
        EI.main(p, tmp_path / "ix", 3, -1, 0, False)
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(RuntimeError):
        EI.main(p, tmp_path / "ix", 3, 3, 0, False)
    assert not (tmp_path / "ix").exists()


def test_cli(tmp_path):
    p = write_npz(tmp_path / "c_nn_classification_embeddings.npz", 30, 2)
    res = CliRunner().invoke(cli.cli, ["embedding-index", str(p), "-q", "--lists", "4", "--iterations", "2", str(tmp_path / "i")])
    assert res.exit_code == 0, res.output
    ix = tmp_path / "i" / "c_embedding_index.npz"
    res = CliRunner().invoke(cli.cli, ["embedding-neighbours", str(p), "-k", "3", "--index", str(ix), "--nprobe", "2", "-q",
                                       str(tmp_path / "o")])
    assert res.exit_code == 0, res.output
    assert int(np.load(tmp_path / "o" / "c_embedding_neighbours.npz")["nprobe"]) == 2
    res = CliRunner().invoke(cli.cli, ["embedding-neighbours", str(p), "--index", str(ix), str(tmp_path / "o3")])
    assert res.exit_code != 0 and not (tmp_path / "o3").exists()
    # the default list count
    res = CliRunner().invoke(cli.cli, ["embedding-index", str(p), "-q", "--iterations", "1", str(tmp_path / "d")])
    assert res.exit_code == 0, res.output
    assert int(np.load(tmp_path / "d" / "c_embedding_index.npz")["lists"]) == 22
