"""
CPU tests of embedding-clusters --index (no GPU): the slot search and the probed block step are replaced by NumPy stand-ins with
the contracts of include/gnm.h (tests/test_gpu_clusters_index.py holds the device to them), over the fp64 stand-ins of
tests/test_clusters_cpu.py.  Covered: the result against a NumPy statement of the definition at nprobe < L, the exact clustering
at nprobe = L, independence of the block size, the slots' append order, the files and keys, every refusal before any device
work (--nprobe without --index, an index of another file or strand key, nprobe out of range, an index whose home lists disagree
with its probes, too little device memory), and the CLI.
"""
import numpy as np
import pytest
import torch
from click.testing import CliRunner

from genomad_b200 import cli, embedding_clusters as EC, embedding_index as EI, engine
from test_clusters_cpu import cos32, families, install as install_clusters
from test_neighbours_cpu import write_npz


def np_slots_append(slots, rows_, gidx, home):
    """engine.cluster_slots_append with the raw rows in place of the TF32 halves."""
    m = slots.end.shape[0]
    for r, g, h in zip(rows_, gidx.tolist(), home.tolist()):
        j = int(h) - slots.l0
        if 0 <= j < m:
            pos = int(slots.end[j])
            assert pos < slots.offsets[j + 1], "slot overflow"
            slots.hi[pos], slots.index[pos] = r, g
            slots.end[j] += 1


def np_slots_search(slots, query, probes):
    """engine.cluster_slots_search: the best (s, row) under (s descending, row ascending) in the probed lists' prefixes."""
    q = query.cpu().numpy()
    sim = np.full((len(q), 1), -np.inf, np.float32)
    idx = np.full((len(q), 1), -1, np.int64)
    for a, pr in enumerate(probes.cpu().numpy()):
        cand = [s for l in pr if 0 <= l - slots.l0 < len(slots.offsets) - 1
                for s in range(int(slots.offsets[l - slots.l0]), int(slots.end[l - slots.l0]))]
        if cand:
            c = cos32(q[a:a + 1], slots.hi[cand].numpy())[0]
            g = slots.index[cand].numpy()
            o = np.lexsort((g, -c))[0]
            sim[a, 0], idx[a, 0] = c[o], g[o]
    return torch.from_numpy(sim), torch.from_numpy(idx)


def np_block_probed(rows_, covered, min_similarity, probes, home):
    thr = engine.cluster_threshold(min_similarity)
    c = cos32(rows_.cpu().numpy(), rows_.cpu().numpy())
    cov, pr, hm = covered.cpu().numpy() != 0, probes.cpu().numpy(), home.cpu().numpy()
    reps = []
    for j in range(len(cov)):
        if not cov[j] and all(c[j, i] < thr for i in reps if hm[i] in pr[j]):
            reps.append(j)
    return torch.tensor(reps, dtype=torch.int64)


def install(setattr_):
    install_clusters(setattr_)
    setattr_(engine, "cluster_slots_append", np_slots_append)
    setattr_(engine, "cluster_slots_search", np_slots_search)
    setattr_(engine, "cluster_block_probed", np_block_probed)


@pytest.fixture(autouse=True)
def _stand_in(monkeypatch):
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    install(monkeypatch.setattr)


def probes_of(emb, cent, nprobe):
    """The stand-ins' probes: each row's nprobe nearest centroids under (s descending, list ascending)."""
    c = cos32(emb, cent)
    return np.stack([np.lexsort((np.arange(len(cent)), -row))[:nprobe] for row in c])


def write_index(path, names, emb, lists, seed=0, key="embeddings"):
    """An index file whose lists are each row's nearest centroid under the stand-ins' similarity (so home(i) = P(i)[0]), with
    seeded rows as centroids."""
    rng = np.random.default_rng(seed)
    cent = emb[rng.choice(len(emb), lists, replace=False)].astype(np.float32)
    home = probes_of(emb, cent, 1)[:, 0]
    rows_ = np.argsort(home, kind="stable")
    off = np.concatenate([[0], np.cumsum(np.bincount(home, minlength=lists))])
    np.savez(path, centroids=cent, rows=rows_.astype(np.int64), offsets=off.astype(np.int64), lists=np.int64(lists),
             iterations=np.int64(0), seed=np.uint64(seed), training_rows=np.int64(len(emb)), embeddings_key=np.str_(key),
             embeddings_sha256=np.str_(EI.embeddings_sha256(names, emb)))
    return path


def definition(emb, t, home, pr):
    """The clustering through the index, stated directly: (representative_index, similarity, representatives)."""
    thr = float(np.float32(t))
    c = cos32(emb, emb)
    reps = []
    for j in range(len(emb)):
        if all(c[j, i] < thr for i in reps if home[i] in pr[j]):
            reps.append(j)
    rep_index, sim = np.arange(len(emb)), np.ones(len(emb), np.float32)
    for j in sorted(set(range(len(emb))) - set(reps)):
        cand = np.array([i for i in reps if home[i] in pr[j]])
        o = np.lexsort((cand, -c[j, cand]))[0]
        rep_index[j], sim[j] = cand[o], c[j, cand[o]]
        assert sim[j] >= thr
    return rep_index, sim, np.array(reps, np.int64)


def setup(tmp_path, emb, lists=6, name="s_nn_classification_embeddings.npz"):
    p = write_npz(tmp_path / name, 0, emb=emb)
    names = np.load(p)["contig_names"].astype(str)
    ix = write_index(tmp_path / "ix.npz", names, emb, lists)
    return p, ix, EI.read_index(ix, names, emb, "embeddings")


def info():
    from genomad_b200 import dist
    return dist.init_process_group_if_needed()


@pytest.mark.parametrize("nprobe", [1, 2, 4])
def test_definition_and_blocks(tmp_path, nprobe):
    emb = families(12, 5, 0.35, 3)
    emb[7] = 0                                                  # a zero row: always a singleton
    emb[20] = emb[3]                                            # a duplicate
    _, _, ix = setup(tmp_path, emb)
    home = EC.home_lists(ix)
    pr = probes_of(emb, ix["centroids"], nprobe)
    assert np.array_equal(pr[:, 0], home)
    want = definition(emb, 0.9, home, pr)
    for block in (1, 7, 64):
        got = EC.cluster(emb, 0.9, info(), block, index=ix, nprobe=nprobe)
        for a, b in zip(got, want):
            assert np.array_equal(a, b), block
    assert want[0][7] == 7 and not np.isin(7, want[0][np.arange(len(emb)) != 7])
    assert 20 not in want[2] or 3 not in want[2]


def test_full_probe_is_exact(tmp_path):
    emb = families(10, 4, 0.3, 5)
    _, _, ix = setup(tmp_path, emb, lists=5)
    exact = EC.cluster(emb, 0.85, info(), 16)
    via = EC.cluster(emb, 0.85, info(), 16, index=ix, nprobe=5)
    for a, b in zip(exact, via):
        assert np.array_equal(a, b)


def test_slots_layout():
    slots = engine.cluster_slots(np.array([0, 3, 5, 9]), 1, 3, "cpu")
    assert list(slots.offsets) == [0, 2, 6] and slots.l0 == 1 and slots.hi.shape == (6, 512)
    x = torch.arange(5 * 512, dtype=torch.float32).reshape(5, 512)
    np_slots_append(slots, x, torch.tensor([2, 5, 8, 9, 11]), torch.tensor([2, 0, 2, 1, 2]))
    assert slots.end.tolist() == [1, 5] and slots.index[0] == 9 and slots.index[2:5].tolist() == [2, 8, 11]
    assert engine.cluster_slots_counts(slots).tolist() == [1, 3]


def test_files_and_keys(tmp_path):
    emb = families(8, 3, 0.3, 9)
    p, ixp, ix = setup(tmp_path, emb, lists=4)
    EC.main(p, tmp_path / "o", 0.9, False, index=ixp, nprobe=2)
    EC.main(p, tmp_path / "e", 0.9, False)
    a, b = np.load(tmp_path / "o" / "s_embedding_clusters.npz"), np.load(tmp_path / "e" / "s_embedding_clusters.npz")
    assert set(a.files) == set(b.files) | {"nprobe", "index_sha256"}
    assert int(a["nprobe"]) == 2 and str(a["index_sha256"]) == EI.file_sha256(ixp)
    want = definition(emb, 0.9, EC.home_lists(ix), probes_of(emb, ix["centroids"], 2))
    assert np.array_equal(a["representative_index"], want[0]) and np.array_equal(a["representatives"], want[2])
    head = (tmp_path / "o" / "s_embedding_clusters.tsv").read_text().splitlines()[0]
    assert head == "seq_name\trepresentative\tcosine_similarity"


@pytest.mark.parametrize("bad", ["nprobe_alone", "nprobe_missing", "nprobe_zero", "nprobe_big", "other_file", "strand_key",
                                 "home", "memory"])
def test_refusals_before_device(tmp_path, monkeypatch, bad):
    emb = families(8, 3, 0.3, 9)
    p, ixp, _ = setup(tmp_path, emb, lists=4)
    def boom(*a, **k):
        raise AssertionError("device work before the inputs were checked")
    for name in ("cluster_slots_search", "cluster_block_probed", "cluster_block", "cluster_slots"):
        monkeypatch.setattr(engine, name, boom)
    kw, err = {"index": ixp, "nprobe": 2}, ValueError
    if bad == "nprobe_alone":
        kw = {"nprobe": 2}
    elif bad == "nprobe_missing":
        kw["nprobe"] = None
    elif bad == "nprobe_zero":
        kw["nprobe"] = 0
    elif bad == "nprobe_big":
        kw["nprobe"] = 5
    elif bad == "other_file":
        p = write_npz(tmp_path / "other.npz", 0, emb=families(8, 3, 0.3, 10))
    elif bad == "strand_key":
        z = dict(np.load(p))
        z["embeddings_both_strands"] = z["embeddings"]
        np.savez(tmp_path / "bs.npz", **z)
        p = tmp_path / "bs.npz"
    elif bad == "home":                                         # edited centroids: the lists no longer follow them
        z = dict(np.load(ixp))
        z["centroids"] = z["centroids"][[1, 0, 2, 3]]
        np.savez(tmp_path / "edited.npz", **z)
        kw["index"], err = tmp_path / "edited.npz", EI.IndexFileError
    else:
        monkeypatch.setattr(EC, "_free_bytes", lambda dev: 1000.0)
        err = MemoryError
    with pytest.raises(err):
        EC.main(p, tmp_path / "out", 0.9, False, both_strands=bad == "strand_key", **kw)
    assert not (tmp_path / "out").exists()


def test_cli(tmp_path):
    emb = families(8, 3, 0.3, 9)
    p, ixp, _ = setup(tmp_path, emb, lists=4, name="c_nn_classification_embeddings.npz")
    res = CliRunner().invoke(cli.cli, ["embedding-clusters", str(p), str(tmp_path / "o"), "--min-similarity", "0.9",
                                       "--index", str(ixp), "--nprobe", "3", "-q"])
    assert res.exit_code == 0, res.output
    assert int(np.load(tmp_path / "o" / "c_embedding_clusters.npz")["nprobe"]) == 3
    for extra in (["--index", str(ixp)], ["--nprobe", "2"]):
        res = CliRunner().invoke(cli.cli, ["embedding-clusters", str(p), str(tmp_path / "o2"), "--min-similarity", "0.9", "-q",
                                           *extra])
        assert res.exit_code != 0 and not (tmp_path / "o2").exists()
