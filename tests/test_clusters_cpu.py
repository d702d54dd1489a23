"""
CPU tests of the embedding-clusters module and CLI (no GPU): gnm_embedding_neighbours, gnm_neighbours_merge and gnm_cluster_block
are replaced by NumPy fp64 stand-ins with the same contracts (tests/test_gpu_clusters.py holds the device to fp64).  Covered: the
result against a brute-force statement of the definition, greedy rather than connected components, duplicates, zero rows,
n = 0 and 1, independence of the block and chunk sizes, TSV bytes, NPZ keys and dtypes, both name keys, the CLI and its
required threshold, and the rejection of malformed input before any device call.
"""
import numpy as np
import pytest
import torch
from click.testing import CliRunner

from genomad_b200 import cli, embedding_clusters as EC, engine
from test_neighbours_cpu import install as install_neighbours, np_neighbours, rows, write_npz


def cos32(q, r):
    """The stand-ins' similarity: fp64 cosine rounded to fp32, the formula of np_neighbours."""
    q, r = np.asarray(q, np.float64), np.asarray(r, np.float64)
    nq_, nr_ = np.linalg.norm(q, axis=1), np.linalg.norm(r, axis=1)
    qn = np.divide(q, nq_[:, None], out=np.zeros_like(q), where=nq_[:, None] > 0)
    rn = np.divide(r, nr_[:, None], out=np.zeros_like(r), where=nr_[:, None] > 0)
    return (qn @ rn.T).astype(np.float32)


def np_cluster_block(rows_, covered, min_similarity):
    """fp64 stand-in for engine.cluster_block."""
    thr = engine.cluster_threshold(min_similarity)
    c = cos32(rows_.cpu().numpy(), rows_.cpu().numpy())
    cov = covered.cpu().numpy() != 0
    reps = []
    for j in range(len(cov)):
        if not cov[j] and all(c[j, i] < thr for i in reps):
            reps.append(j)
    return torch.tensor(reps, dtype=torch.int64, device=rows_.device)


def install(setattr_):
    install_neighbours(setattr_)
    setattr_(engine, "cluster_block", np_cluster_block)


@pytest.fixture(autouse=True)
def _stand_in(monkeypatch):
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    install(monkeypatch.setattr)


def brute_force(emb, t):
    """The definition, stated directly: (representative_index, similarity, representatives)."""
    thr = float(np.float32(t))
    c = cos32(emb, emb)
    reps = []
    for j in range(len(emb)):
        if all(c[j, i] < thr for i in reps):
            reps.append(j)
    reps = np.array(reps, np.int64)
    rep_index, sim = np.empty(len(emb), np.int64), np.ones(len(emb), np.float32)
    for j in range(len(emb)):
        if j in set(reps.tolist()):
            rep_index[j] = j
            continue
        o = np.lexsort((reps, -c[j, reps]))[0]
        rep_index[j], sim[j] = reps[o], c[j, reps[o]]
        assert sim[j] >= thr
    return rep_index, sim, reps


def families(n_fam, per, noise, seed):
    """Families of noisy copies of sparse rows, shuffled: clusters of several members."""
    rng = np.random.default_rng(seed)
    base = rows(n_fam, seed)
    x = np.repeat(base, per, axis=0)
    x = x * (1 + noise * rng.standard_normal(x.shape))
    return x[rng.permutation(len(x))].astype(np.float32)


def run(tmp_path, emb, t, name="s_nn_classification_embeddings.npz", out="out", key="contig_names", **kw):
    p = write_npz(tmp_path / name, 0, key=key, emb=emb)
    EC.main(p, tmp_path / out, t, False, **kw)
    prefix = name[: -len("_nn_classification_embeddings.npz")] if name.endswith("_nn_classification_embeddings.npz") else name[:-4]
    return np.load(tmp_path / out / f"{prefix}_embedding_clusters.npz"), tmp_path / out / f"{prefix}_embedding_clusters.tsv"


@pytest.mark.parametrize("seed,t,block", [(0, 0.9, 8192), (1, 0.95, 7), (2, 0.8, 1), (3, 0.5, 16)])
def test_matches_the_definition(tmp_path, seed, t, block):
    emb = families(12, 5, 0.3, seed)
    z, _ = run(tmp_path, emb, t, block=block, rep_chunk=3)
    want = brute_force(emb, t)
    assert np.array_equal(z["representatives"], want[2])
    assert np.array_equal(z["representative_index"], want[0]) and np.array_equal(z["similarity"], want[1])
    assert 1 < len(want[2]) < len(emb)                                       # neither all singletons nor one cluster
    assert np.array_equal(z["cluster_size"], np.bincount(np.searchsorted(want[2], want[0])))
    members = want[0] != np.arange(len(emb))
    sim, idx = np_neighbours(torch.from_numpy(emb[members]), torch.from_numpy(emb[want[2]]), 1)
    assert np.array_equal(want[2][idx.numpy()[:, 0]], want[0][members])      # = a k = 1 search against the representatives


def test_greedy_not_connected_components(tmp_path):
    th1, th2 = np.arccos(0.95), np.arccos(0.9)
    emb = np.zeros((3, 512), np.float32)
    for r, a in enumerate((0.0, th1, th1 + th2)):                             # s(a, b) = 0.95, s(b, c) = 0.9, s(a, c) = 0.72
        emb[r, 0], emb[r, 1] = np.cos(a), np.sin(a)
    z, _ = run(tmp_path, emb, 0.85)
    assert z["representatives"].tolist() == [0, 2] and z["representative_index"].tolist() == [0, 0, 2]
    assert z["cluster_size"].tolist() == [2, 1]


def test_duplicates_and_zero_rows(tmp_path):
    emb = rows(8, 4)
    emb[4] = emb[1]
    emb[6] = 3 * emb[1]
    emb[3] = 0
    emb[7] = 0
    z, tsv = run(tmp_path, emb, 0.99)
    ri = z["representative_index"]
    assert ri[4] == 1 and ri[6] == 1 and ri[3] == 3 and ri[7] == 7           # zero rows: singletons
    assert z["similarity"][3] == 1.0 and z["similarity"][7] == 1.0
    lines = tsv.read_text().splitlines()
    assert lines[4] == "seq_3\tseq_3\t1.000000" and lines[8] == "seq_7\tseq_7\t1.000000"
    assert lines[5].startswith("seq_4\tseq_1\t")


def test_empty_and_single(tmp_path):
    z, tsv = run(tmp_path, np.zeros((0, 512), np.float32), 0.9, out="o0")
    assert z["representatives"].shape == (0,) and z["representative_index"].shape == (0,)
    assert z["representatives"].dtype == np.int64 and z["cluster_size"].dtype == np.int64
    assert tsv.read_text() == "seq_name\trepresentative\tcosine_similarity\n"
    z, tsv = run(tmp_path, rows(1, 2), 1.0, out="o1")
    assert z["representatives"].tolist() == [0] and z["cluster_size"].tolist() == [1]
    assert tsv.read_text().splitlines()[1] == "seq_0\tseq_0\t1.000000"


def test_block_and_chunk_sizes_give_identical_files(tmp_path):
    emb = families(40, 4, 0.2, 9)
    out = []
    for i, (block, chunk) in enumerate([(1, 1), (7, 5), (128, 2**18), (8192, 13)]):
        _, tsv = run(tmp_path, emb, 0.9, out=f"o{i}", block=block, rep_chunk=chunk)
        out.append((tsv.read_bytes(), tsv.with_suffix(".npz").read_bytes()))
    assert all(o == out[0] for o in out)


def test_outputs_and_name_keys(tmp_path):
    emb = families(4, 3, 0.1, 5)
    z, tsv = run(tmp_path, emb, 0.9, name="p_provirus_nn_classification_embeddings.npz", key="provirus_names")
    assert tsv.name == "p_provirus_embedding_clusters.tsv"
    assert set(z.files) == {"seq_names", "representative_index", "similarity", "representatives", "cluster_size",
                            "min_similarity"}
    assert z["representative_index"].dtype == np.int64 and z["similarity"].dtype == np.float32
    assert z["representatives"].dtype == np.int64 and z["cluster_size"].dtype == np.int64
    assert z["min_similarity"].dtype == np.float64 and float(z["min_similarity"]) == float(np.float32(0.9))
    assert list(z["seq_names"]) == [f"seq_{i}" for i in range(12)]
    ri, s = z["representative_index"], z["similarity"]
    want = "seq_name\trepresentative\tcosine_similarity\n" + "".join(
        f"seq_{i}\tseq_{ri[i]}\t{float(s[i]):.6f}\n" for i in range(12))
    assert tsv.read_text() == want
    assert z["cluster_size"].sum() == 12 and np.all(np.diff(z["representatives"]) > 0)
    assert EC.output_paths("x/other.npz", tmp_path)[1] == tmp_path / "other_embedding_clusters.npz"


def test_cli(tmp_path):
    p = write_npz(tmp_path / "c_nn_classification_embeddings.npz", 0, emb=families(3, 3, 0.1, 6))
    res = CliRunner().invoke(cli.cli, ["embedding-clusters", str(p), str(tmp_path / "o"), "--min-similarity", "0.9", "-q"])
    assert res.exit_code == 0, res.output
    assert np.load(tmp_path / "o" / "c_embedding_clusters.npz")["representative_index"].shape == (9,)
    res = CliRunner().invoke(cli.cli, ["embedding-clusters", str(p), str(tmp_path / "o2")])
    assert res.exit_code != 0 and "--min-similarity" in res.output and not (tmp_path / "o2").exists()
    for bad in ("0", "-0.5", "1.5", "nan"):
        res = CliRunner().invoke(cli.cli, ["embedding-clusters", str(p), str(tmp_path / "o3"), "--min-similarity", bad])
        assert res.exit_code != 0 and not (tmp_path / "o3").exists(), bad
    for bad in (0.0, -0.1, 1.01, float("nan"), 1e-50):
        with pytest.raises(ValueError):
            EC.main(p, tmp_path / "o4", bad, False)
    assert not (tmp_path / "o4").exists()


@pytest.mark.parametrize("bad", ["width", "nan", "names", "key", "ndim"])
def test_malformed_inputs_rejected_before_device(tmp_path, monkeypatch, bad):
    def boom(*a, **k):
        raise AssertionError("device call before the inputs were checked")
    monkeypatch.setattr(engine, "embedding_neighbours", boom)
    monkeypatch.setattr(engine, "cluster_block", boom)
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
    from genomad_b200 import embedding_neighbours as EN
    with pytest.raises(EN.EmbeddingsFileError):
        EC.main(path, tmp_path / "out", 0.9, False)
    assert not (tmp_path / "out").exists()
