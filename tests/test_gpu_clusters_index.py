"""
Embedding clusters through the index on an H100 (include/gnm.h and DESIGN.md, "Embedding clusters through the index"):
  * nprobe = L: bitwise the exact clustering (EC.cluster without an index) on families, distinct rows, duplicates and zero rows,
    at n = 8,191 / 8,192 / 8,193 / 16,385, on layouts with empty, one-row and sub-tile lists and lists longer than one 1,536-row
    range;
  * nprobe < L: bitwise a NumPy statement of the definition on the device's own similarity matrix (engine.embedding_neighbours
    at k = 64 against 64-row reference chunks) and the device's probes;
  * the threshold: t set to a pair's similarity covers, the next float above it does not, across blocks and inside one;
  * bitwise invariance to the block size (1, 7, 1,000, 8,192) and repeats;
  * the guarantees: every member's similarity >= t, a duplicate of a representative is never one, a zero row is a singleton;
  * the module end to end: the TSV bytes equal the exact run's at nprobe = L.
"""
import numpy as np
import pytest
import torch

from genomad_b200 import dist, embedding_clusters as EC, embedding_index as EI, engine

pytestmark = pytest.mark.gpu
ONE = dist.DistInfo()


@pytest.fixture(autouse=True)
def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def index_rows(sizes, seed, fams=4, spread=0.3):
    """Rows whose lists are known: list l's rows live on coordinates [32 l, 32 l + 32) (around `fams` family centres each), its
    centroid is that block's unit vector, so every row's nearest centroid is its list.  Rows are shuffled over lists in file
    order; a list of size 0 stays empty.  Returns (x float32 [n, 512], index dict as embedding_index.read_index gives)."""
    rng = np.random.default_rng(seed)
    L = len(sizes)
    assert L <= 16
    lab = rng.permutation(np.repeat(np.arange(L), sizes))
    n = len(lab)
    base = np.abs(rng.standard_normal((L, fams, 32))) + 0.5
    x = 0.02 * np.abs(rng.standard_normal((n, 512)))
    f = rng.integers(0, fams, n)
    for i in range(n):
        x[i, 32 * lab[i]:32 * lab[i] + 32] += base[lab[i], f[i]] * (1 + spread * rng.standard_normal(32))
    cent = np.zeros((L, 512), np.float32)
    for l in range(L):
        cent[l, 32 * l:32 * l + 32] = 1 / np.sqrt(32)
    rows = np.argsort(lab, kind="stable").astype(np.int64)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    return x.astype(np.float32), {"centroids": cent, "rows": rows, "offsets": off, "lists": L, "sha256": "-"}


def as_index(ix):
    return {"centroids": ix.centroids.cpu().numpy(), "rows": ix.rows.cpu().numpy(), "offsets": ix.offsets.cpu().numpy(),
            "lists": ix.centroids.shape[0], "sha256": "-"}


def same(a, b):
    return np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32)) and np.array_equal(a[2], b[2])


SIZES = [40, 1, 7, 191, 0, 193, 1600, 3100, 1, 400, 0, 384, 1537, 60, 2]      # 8-tile range = 1,536 rows


@pytest.mark.parametrize("t", [0.9, 0.995])
def test_full_probe_is_exact_edges(t):
    x, ix = index_rows(SIZES, 1)
    x[5] = 0.0
    x[x.shape[0] // 2] = 0.0                                  # zero rows: their nearest centroid is list 0
    x[17] = x[3]
    x[x.shape[0] - 3] = x[3]                                  # duplicates
    hx = EC.home_lists(ix)
    for z in (5, x.shape[0] // 2):                            # move the zero rows to list 0 (their probes' first list)
        hx[z] = 0
    for d in (17, x.shape[0] - 3):
        hx[d] = hx[3]
    ix["rows"] = np.argsort(hx, kind="stable").astype(np.int64)
    ix["offsets"] = np.concatenate([[0], np.cumsum(np.bincount(hx, minlength=ix["lists"]))]).astype(np.int64)
    got = EC.cluster(x, t, ONE, index=ix, nprobe=ix["lists"])
    assert same(got, EC.cluster(x, t, ONE))
    assert got[0][5] == 5 and (got[0] == 5).sum() == 1       # a zero row is a singleton
    assert 17 not in got[2] or 3 not in got[2]


@pytest.mark.parametrize("n", [8191, 8192, 8193, 16385])
def test_full_probe_is_exact_sizes(n):
    sizes = [n // 8] * 7 + [n - 7 * (n // 8)]
    for t, fams in ((0.97, 3), (0.999, 64)):                  # families, then mostly distinct rows
        x, ix = index_rows(sizes, n, fams)
        assert same(EC.cluster(x, t, ONE, index=ix, nprobe=8), EC.cluster(x, t, ONE)), t


def device_similarities(x):
    """S[j, i] = the search's similarity of query j, reference i, bit for bit: k = 64 against 64-row reference chunks."""
    xt = torch.from_numpy(x).cuda()
    n = x.shape[0]
    S = np.empty((n, n), np.float32)
    for a in range(0, n, 64):
        b = min(n, a + 64)
        sim, idx = engine.embedding_neighbours(xt, xt[a:b], b - a, ref_index0=a)
        s, i = sim.cpu().numpy(), idx.cpu().numpy()
        np.put_along_axis(S[:, a:b], i - a, s, axis=1)
    return S


def definition(S, t, home, pr):
    thr = np.float32(t)
    n = S.shape[0]
    reps = []
    ok = np.zeros((n, len(home)), bool)
    for j in range(n):
        seen = np.isin(home, pr[j])
        ok[j] = seen
        if not any(S[j, i] >= thr for i in reps if seen[i]):
            reps.append(j)
    reps = np.array(reps, np.int64)
    rep_index, sim = np.arange(n), np.ones(n, np.float32)
    for j in np.setdiff1d(np.arange(n), reps):
        cand = reps[ok[j, reps]]
        o = np.lexsort((cand, -S[j, cand]))[0]
        rep_index[j], sim[j] = cand[o], S[j, cand[o]]
    return rep_index, sim, reps


@pytest.mark.parametrize("nprobe", [1, 2, 5])
def test_definition(nprobe):
    from test_gpu_ivf import clustered
    x = clustered(3000, 40, 7, spread=0.25)
    x[100] = x[50]
    x[200] = 0.0
    ix = as_index(engine.ivf_build(torch.from_numpy(x).cuda(), 12, 5, 0))
    S = device_similarities(x)
    pr = engine.ivf_probes(torch.from_numpy(x).cuda(), torch.from_numpy(ix["centroids"]).cuda(), nprobe).cpu().numpy()
    home = EC.home_lists(ix)
    assert np.array_equal(pr[:, 0], home)
    t = float(np.quantile(S[np.triu_indices(3000, 1)], 0.999))
    want = definition(S, t, home, pr)
    got = EC.cluster(x, t, ONE, 1000, index=ix, nprobe=nprobe)
    assert same(got, want)
    assert (got[1] >= np.float32(t)).all()
    assert 100 not in got[2] or got[0][50] != 50               # a duplicate of a representative never is one
    assert got[0][200] == 200 and (got[0] == 200).sum() == 1


@pytest.mark.parametrize("block", [1, 2])
def test_threshold_is_the_search_similarity(block):
    from test_gpu_ivf import clustered
    x = clustered(2, 1, 3, spread=0.1)
    xt = torch.from_numpy(x).cuda()
    v = np.float32(engine.embedding_neighbours(xt[1:], xt[:1], 1)[0].item())      # s(1, 0)
    assert 0 < v < 1
    ix = {"centroids": x[:1] / np.linalg.norm(x[:1]), "rows": np.arange(2), "offsets": np.array([0, 2]), "lists": 1,
          "sha256": "-"}
    at = EC.cluster(x, float(v), ONE, block, index=ix, nprobe=1)           # block 1: covering; block 2: the block step
    assert list(at[2]) == [0] and at[1][1].view(np.uint32) == v.view(np.uint32)
    above = EC.cluster(x, float(np.nextafter(v, np.float32(2))), ONE, block, index=ix, nprobe=1)
    assert list(above[2]) == [0, 1]


def test_block_invariance_and_repeats():
    from test_gpu_ivf import clustered
    x = clustered(9000, 300, 11, spread=0.2)
    ix = as_index(engine.ivf_build(torch.from_numpy(x).cuda(), 30, 5, 0))
    ref = EC.cluster(x, 0.95, ONE, index=ix, nprobe=4)
    assert 30 < len(ref[2]) < 9000
    for block in (1, 7, 1000, 8192, 8192):
        assert same(EC.cluster(x, 0.95, ONE, block, index=ix, nprobe=4), ref), block


def test_module(tmp_path):
    from test_gpu_ivf import clustered
    from test_neighbours_cpu import write_npz
    p = write_npz(tmp_path / "m_nn_classification_embeddings.npz", 0, emb=clustered(5000, 50, 13, spread=0.3))
    EI.main(p, tmp_path / "ix", 20, 5, 0, False)
    ixp = tmp_path / "ix" / "m_embedding_index.npz"
    EC.main(p, tmp_path / "full", 0.95, False, index=ixp, nprobe=20)
    EC.main(p, tmp_path / "exact", 0.95, False)
    EC.main(p, tmp_path / "part", 0.95, False, index=ixp, nprobe=3)
    tsv = "m_embedding_clusters.tsv"
    assert (tmp_path / "full" / tsv).read_bytes() == (tmp_path / "exact" / tsv).read_bytes()
    z = np.load(tmp_path / "part" / "m_embedding_clusters.npz")
    assert int(z["nprobe"]) == 3 and str(z["index_sha256"]) == EI.file_sha256(ixp)
    assert (z["similarity"] >= np.float32(0.95)).all()
