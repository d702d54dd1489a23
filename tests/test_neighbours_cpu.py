"""
CPU tests of the embedding-neighbours module and CLI (no GPU): gnm_embedding_neighbours and gnm_neighbours_merge are replaced
by a NumPy fp64 stand-in with the same contract (tests/test_gpu_neighbours.py holds the device to fp64).  Covered: output
names and prefixes, TSV bytes, NPZ keys and dtypes, both name keys, padding when k exceeds the candidates, self-exclusion,
the merge order on ties, and the rejection of malformed embeddings files before any device call.
"""
import numpy as np
import pytest
import torch
from click.testing import CliRunner

from genomad_b200 import cli, embedding_neighbours as EN, engine


def np_neighbours(query, reference=None, k=10, *, ref_index0=0, self_index0=None):
    """fp64 stand-in for engine.embedding_neighbours: same order, padding and self-exclusion."""
    q = query.cpu().numpy().astype(np.float64)
    r = q if reference is None else reference.cpu().numpy().astype(np.float64)
    self0 = (ref_index0 if reference is None else -1) if self_index0 is None else self_index0
    nq_, nr_ = np.linalg.norm(q, axis=1), np.linalg.norm(r, axis=1)
    qn = np.divide(q, nq_[:, None], out=np.zeros_like(q), where=nq_[:, None] > 0)
    rn = np.divide(r, nr_[:, None], out=np.zeros_like(r), where=nr_[:, None] > 0)
    c = (qn @ rn.T).astype(np.float32)
    sim = np.full((len(q), k), -np.inf, np.float32)
    idx = np.full((len(q), k), -1, np.int64)
    for i in range(len(q)):
        g = np.arange(len(r), dtype=np.int64) + ref_index0
        keep = g != (self0 + i if self0 >= 0 else -1)
        s, gi = c[i][keep], g[keep]
        o = np.lexsort((gi, -s))[:k]
        sim[i, :len(o)], idx[i, :len(o)] = s[o], gi[o]
    return torch.from_numpy(sim).to(query.device), torch.from_numpy(idx).to(query.device)


def np_merge(sim, idx, sim_b, idx_b):
    """fp64 stand-in for engine.neighbours_merge (in place)."""
    k = sim.shape[1]
    s = torch.cat([sim, sim_b], 1).cpu().numpy()
    x = torch.cat([idx, idx_b], 1).cpu().numpy()
    out_s, out_x = np.empty_like(s[:, :k]), np.empty_like(x[:, :k])
    for i in range(len(s)):
        real = x[i] >= 0
        o = np.lexsort((x[i][real], -s[i][real]))[:k]
        row_s = np.full(k, -np.inf, np.float32); row_x = np.full(k, -1, np.int64)
        row_s[:len(o)], row_x[:len(o)] = s[i][real][o], x[i][real][o]
        out_s[i], out_x[i] = row_s, row_x
    sim.copy_(torch.from_numpy(out_s)); idx.copy_(torch.from_numpy(out_x))
    return sim, idx


def install(setattr_):
    setattr_(engine, "embedding_neighbours", np_neighbours)
    setattr_(engine, "neighbours_merge", np_merge)
    setattr_(EN, "_device", lambda info: torch.device("cpu"))


def rows(n, seed):
    rng = np.random.default_rng(seed)
    return (np.maximum(rng.standard_normal((n, 512)), 0) * (rng.random((n, 512)) < 0.3)).astype(np.float32)


def write_npz(path, n, seed=0, key="contig_names", emb=None):
    emb = rows(n, seed) if emb is None else emb
    np.savez(path, **{key: np.array([f"seq_{i}" for i in range(len(emb))]), "embeddings": emb})
    return path


@pytest.fixture(autouse=True)
def _stand_in(monkeypatch):
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    install(monkeypatch.setattr)


def test_prefix_and_paths(tmp_path):
    assert EN.output_prefix("a/sample_nn_classification_embeddings.npz") == "sample"
    assert EN.output_prefix("sample_provirus_nn_classification_embeddings.npz") == "sample_provirus"
    assert EN.output_prefix("other.npz") == "other"
    tsv, npz = EN.output_paths("x/s_nn_classification_embeddings.npz", tmp_path)
    assert tsv == tmp_path / "s_embedding_neighbours.tsv" and npz == tmp_path / "s_embedding_neighbours.npz"


def test_all_vs_all_outputs(tmp_path):
    q = write_npz(tmp_path / "s_nn_classification_embeddings.npz", 12)
    EN.main(q, None, tmp_path / "out", 3, False)
    z = np.load(tmp_path / "out" / "s_embedding_neighbours.npz")
    assert set(z.files) == {"query_names", "reference_names", "neighbour_index", "similarity", "k"}
    assert z["neighbour_index"].dtype == np.int64 and z["similarity"].dtype == np.float32 and int(z["k"]) == 3
    assert z["neighbour_index"].shape == (12, 3) and list(z["query_names"]) == [f"seq_{i}" for i in range(12)]
    assert not np.any(z["neighbour_index"] == np.arange(12)[:, None])                   # self-exclusion
    sim, idx = np_neighbours(torch.from_numpy(np.load(q)["embeddings"]), None, 3)
    assert np.array_equal(z["neighbour_index"], idx.numpy()) and np.array_equal(z["similarity"], sim.numpy())
    want = "seq_name\trank\tneighbour_name\tcosine_similarity\n" + "".join(
        f"seq_{i}\t{r + 1}\tseq_{idx[i, r]}\t{float(sim[i, r]):.6f}\n" for i in range(12) for r in range(3))
    assert (tmp_path / "out" / "s_embedding_neighbours.tsv").read_text() == want


def test_reference_provirus_key_and_padding(tmp_path):
    q = write_npz(tmp_path / "p_provirus_nn_classification_embeddings.npz", 4, 1, key="provirus_names")
    r = write_npz(tmp_path / "ref.npz", 3, 2)
    EN.main(q, r, tmp_path / "out", 5, False)
    z = np.load(tmp_path / "out" / "p_provirus_embedding_neighbours.npz")
    assert list(z["reference_names"]) == ["seq_0", "seq_1", "seq_2"]
    assert np.all(z["neighbour_index"][:, 3:] == -1) and np.all(np.isneginf(z["similarity"][:, 3:]))
    assert np.all(z["neighbour_index"][:, :3] >= 0)
    lines = (tmp_path / "out" / "p_provirus_embedding_neighbours.tsv").read_text().splitlines()
    assert len(lines) == 1 + 4 * 3 and all(ln.split("\t")[1] in "123" for ln in lines[1:])


def test_ties_go_to_the_lower_index(tmp_path):
    e = rows(6, 3)
    e[4] = e[1]
    e[5] = 2 * e[1]                                       # same direction: the same cosine
    q = write_npz(tmp_path / "t.npz", 0, emb=e)
    EN.main(q, None, tmp_path / "out", 3, False)
    z = np.load(tmp_path / "out" / "t_embedding_neighbours.npz")
    assert list(z["neighbour_index"][1][:2]) == [4, 5] and list(z["neighbour_index"][5][:2]) == [1, 4]
    # the merge keeps the total order across lists
    s = torch.tensor([[0.5, 0.25, -np.inf]], dtype=torch.float32)
    i = torch.tensor([[7, 2, -1]])
    np_merge(s, i, torch.tensor([[0.5, 0.25, 0.1]], dtype=torch.float32), torch.tensor([[3, 9, 4]]))
    assert i.tolist() == [[3, 7, 2]] and s.tolist() == [[0.5, 0.5, 0.25]]


@pytest.mark.parametrize("bad", ["width", "nan", "names", "key", "ndim"])
def test_malformed_inputs_rejected_before_device(tmp_path, monkeypatch, bad):
    def boom(*a, **k):
        raise AssertionError("device call before the inputs were checked")
    monkeypatch.setattr(engine, "embedding_neighbours", boom)
    good = write_npz(tmp_path / "good.npz", 4)
    e = rows(4, 0)
    path = tmp_path / "bad.npz"
    if bad == "width":
        np.savez(path, contig_names=np.array(["a", "b", "c", "d"]), embeddings=e[:, :511])
    elif bad == "nan":
        e[2, 7] = np.nan
        np.savez(path, contig_names=np.array(["a", "b", "c", "d"]), embeddings=e)
    elif bad == "names":
        np.savez(path, contig_names=np.array(["a", "b", "c"]), embeddings=e)
    elif bad == "key":
        np.savez(path, names=np.array(["a", "b", "c", "d"]), embeddings=e)
    else:
        np.savez(path, contig_names=np.array(["a"]), embeddings=e[0])
    for qp, rp in ((path, None), (good, path)):
        with pytest.raises(EN.EmbeddingsFileError):
            EN.main(qp, rp, tmp_path / "out", 3, False)
    assert not (tmp_path / "out").exists()


def test_cli(tmp_path):
    q = write_npz(tmp_path / "c_nn_classification_embeddings.npz", 5)
    r = write_npz(tmp_path / "r.npz", 7, 4)
    res = CliRunner().invoke(cli.cli, ["embedding-neighbours", str(q), "--reference", str(r), "-k", "2", "-q", str(tmp_path / "o")])
    assert res.exit_code == 0, res.output
    z = np.load(tmp_path / "o" / "c_embedding_neighbours.npz")
    assert z["neighbour_index"].shape == (5, 2) and int(z["k"]) == 2
    res = CliRunner().invoke(cli.cli, ["embedding-neighbours", str(q), "-k", "65", str(tmp_path / "o2")])
    assert res.exit_code != 0 and not (tmp_path / "o2").exists()
