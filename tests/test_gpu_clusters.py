"""
Embedding clusters on the H100 (gnm_cluster_block and the embedding-clusters module): the threshold mask bitwise the comparison
of gnm_embedding_neighbours' own similarities (the threshold set to a pair's similarity and to the next float above it), the
full result equal to the fp64 greedy on inputs with no pair near the threshold, every decision on real encoder embeddings
explained by fp64 up to a pair within 2 EPS of the threshold, members' (representative, similarity) bitwise a k = 1 search
against the representatives, and bitwise independence of the block size, the representative chunk size and repeats.
"""
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from genomad_b200 import dist, embedding_clusters as EC, engine
from test_gpu_neighbours import EPS, cos64, sparse_rows

pytestmark = pytest.mark.gpu
ONE = dist.DistInfo()


def decides_pair(x, i, j, t):
    """Block x with every row covered except i < j: j is a new representative iff the mask bit (j, i) is clear."""
    cov = torch.ones(x.shape[0], dtype=torch.uint8, device=x.device)
    cov[i] = cov[j] = 0
    new = engine.cluster_block(x, cov, t).tolist()
    assert new[0] == i and len(new) in (1, 2)
    return len(new) == 1                                                     # True: j covered by i, s(j, i) >= t


def check_pairs(x, pairs, s):
    """s[(j, i)] = the search's similarity of query j, reference i: the bit is set at t = s and clear at the next float."""
    for (j, i) in pairs:
        v = np.float32(s[(j, i)])
        if not 0 < v < 1:
            continue
        assert decides_pair(x, i, j, float(v)), f"pair ({j}, {i}): s = {v!r} not >= itself in the mask"
        assert not decides_pair(x, i, j, float(np.nextafter(v, np.float32(2)))), f"pair ({j}, {i}): bit set above s"


def test_mask_bits_all_pairs_small():
    for n in (2, 33, 64):
        x = torch.from_numpy(sparse_rows(n, 40 + n)).cuda()
        sim, idx = engine.embedding_neighbours(x, x, n)                      # all-vs-all lists, k = n, no self-exclusion
        sim, idx = sim.cpu().numpy(), idx.cpu().numpy()
        s = {(j, int(idx[j, r])): sim[j, r] for j in range(n) for r in range(n)}
        check_pairs(x, [(j, i) for j in range(n) for i in range(j)], s)


@pytest.mark.parametrize("n", [129, 193, 385, 1000, 8192])
def test_mask_bits_sampled_at_tile_edges(n):
    x = torch.from_numpy(sparse_rows(n, n)).cuda()
    edges = [e for e in (0, 1, 31, 32, 127, 128, 129, 191, 192, 193, 255, 256, 383, 384, n - 2, n - 1) if e < n]
    rng = np.random.default_rng(n)
    pairs = {(max(a, b), min(a, b)) for a in edges for b in edges if a != b}
    pairs |= {(int(j), int(rng.integers(0, j))) for j in rng.integers(1, n, 60)}
    pairs = sorted(pairs)[:150]
    s = {}
    for (j, i) in pairs:
        v, _ = engine.embedding_neighbours(x[j:j + 1], x[i:i + 1], 1)
        s[(j, i)] = v.item()
    check_pairs(x, pairs, s)


def families(n, t, seed, check=True):
    """n rows in shuffled families: within a family every cos64 >= t + 1e-3, across families every cos64 <= t - 1e-3."""
    rng = np.random.default_rng(seed)
    base = sparse_rows(max(1, n // 4), seed)
    fam = rng.integers(0, len(base), n)
    x = base[fam] * (1 + 0.02 * rng.standard_normal((n, 512)))
    x[rng.random(n) < 0.05] *= 0                                             # a few zero rows
    x = x.astype(np.float32)
    if not check:
        return x, None
    c = cos64(x, x)
    same = (fam[:, None] == fam[None, :]) & (np.abs(x).sum(1)[:, None] > 0) & (np.abs(x).sum(1)[None, :] > 0)
    np.fill_diagonal(same, False)
    off = ~same
    np.fill_diagonal(off, False)
    assert (c[same] >= t + 1e-3).all() and (c[off] <= t - 1e-3).all(), "construction: a pair near the threshold"
    return x, c


def greedy64(c, t):
    n = len(c)
    reps = []
    for j in range(n):
        if all(c[j, i] < t for i in reps):
            reps.append(j)
    reps = np.array(reps, np.int64)
    ri = reps[np.argmax(c[:, reps], axis=1)] if n else np.zeros(0, np.int64)
    ri[reps] = reps
    return ri, reps


def check_members(x, t, ri, sim, reps):
    """Bitwise: members' similarity >= t, and (representative, similarity) = a k = 1 search against the representatives."""
    members = np.flatnonzero(ri != np.arange(len(ri)))
    assert np.all(sim[reps] == 1) and np.all(sim[members] >= np.float32(t))
    if len(members):
        dx = torch.from_numpy(x).cuda()
        s, i = engine.embedding_neighbours(dx[torch.from_numpy(members).cuda()], dx[torch.from_numpy(reps).cuda()], 1)
        assert np.array_equal(sim[members], s.cpu().numpy()[:, 0])
        assert np.array_equal(ri[members], reps[i.cpu().numpy()[:, 0]])


@pytest.mark.parametrize("n", [1, 127, 128, 129, 191, 192, 193, 383, 385, 3000])
def test_families_against_fp64(n):
    t = 0.95
    x, c = families(n, t, n)
    ri64, reps64 = greedy64(c, t)
    for block in sorted({n, 128, engine.CLUSTER_MAX_BLOCK}):
        ri, sim, reps = EC.cluster(x, t, ONE, block=block)
        assert np.array_equal(reps, reps64) and np.array_equal(ri, ri64), f"block {block}"
        assert np.all(np.abs(sim.astype(np.float64) - c[np.arange(n), ri])[ri != np.arange(n)] <= EPS)
        check_members(x, t, ri, sim, reps)


def test_bitwise_independence_of_block_chunk_and_repeats():
    n, t = 20000, 0.95
    x, _ = families(n, t, 77, check=False)
    x[n // 2:] = sparse_rows(n - n // 2, 78)                                 # the second half: mostly singletons
    ref = EC.cluster(x, t, ONE)
    assert 1000 < len(ref[2]) < n
    check_members(x, t, *ref)
    for block, chunk in ((engine.CLUSTER_MAX_BLOCK, engine.NEIGHBOURS_CHUNK), (1000, 777), (4097, 5000), (128, 2 ** 18),
                         (8191, 100)):
        got = EC.cluster(x, t, ONE, block=block, rep_chunk=chunk)
        assert all(np.array_equal(a, b) for a, b in zip(got, ref)), (block, chunk)


def test_real_embeddings(weights_npz):
    from oracle import igloo_model as M
    c = engine.Classifier(M.load_npz_weights(weights_npz), device=0, max_batch=64)
    try:
        rng = np.random.default_rng(23)
        seqs = [np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, ln)].tobytes() for ln in rng.integers(6000, 20000, 300)]
        seqs += [s[: len(s) // 2 + 3000] for s in seqs[:40]] + seqs[40:60]        # prefixes and exact copies
        *_, emb = c.classify_contigs(seqs, return_embeddings=True)
        x = emb.cpu().numpy()
    finally:
        c.close()
    c64 = cos64(x, x)
    off = c64[~np.eye(len(x), dtype=bool)]
    for q in (0.5, 0.9, 0.99):
        t = float(np.float32(np.quantile(off, q)))
        ri, sim, reps = EC.cluster(x, t, ONE, block=128)
        is_rep = np.zeros(len(x), bool)
        is_rep[reps] = True
        for j in range(len(x)):                      # each decision, given the GPU's earlier representatives
            earlier = reps[reps < j]
            rep64 = bool(np.all(c64[j, earlier] < t))
            if rep64 != is_rep[j]:
                assert np.min(np.abs(c64[j, earlier] - t)) <= 2 * EPS, f"t = {t}: row {j} decided against fp64"
        members = np.flatnonzero(~is_rep)
        best = np.max(c64[members][:, reps], axis=1)
        assert np.all(c64[members, ri[members]] >= best - 2 * EPS)
        check_members(x, t, ri, sim, reps)


def test_errors():
    x = torch.zeros((8193, 512), device="cuda")
    with pytest.raises(ValueError):
        engine.cluster_block(x, torch.zeros(8193, dtype=torch.uint8, device="cuda"), 0.9)
    with pytest.raises(ValueError):
        engine.cluster_block(x[:4], torch.zeros(4, dtype=torch.uint8, device="cuda"), 0.0)
    lib = engine.load_library()
    d = torch.zeros((4, 512), device="cuda")
    assert lib.gnm_cluster_block(d.data_ptr(), 4, d.data_ptr(), 1.5, d.data_ptr(), d.data_ptr(), d.data_ptr(), 1 << 20, None)
    assert b"min_similarity" in lib.gnm_last_error()
    assert lib.gnm_cluster_block(d.data_ptr(), 4, d.data_ptr(), 0.5, d.data_ptr(), d.data_ptr(), d.data_ptr(), 16, None)
    assert b"workspace too small" in lib.gnm_last_error()
    assert lib.gnm_cluster_block_workspace_bytes(8193) == 0 and b"n_block" in lib.gnm_last_error()


def test_module_end_to_end(tmp_path):
    from genomad_b200 import _paths, nn_classification
    rng = np.random.default_rng(19)
    fa = tmp_path / "sample.fna"
    seqs = ["".join(rng.choice(list("ACGT"), n)) for n in (9000, 15000, 6500, 20000, 7000)]
    seqs += [seqs[1], seqs[3][:15000]]
    fa.write_text("".join(f">seq{i}\n{s}\n" for i, s in enumerate(seqs)))
    nn_classification.main(fa, tmp_path / "nn", False, 128, False, 2, False, False, write_embeddings=True)
    emb_npz = _paths.NNOutputs("sample", tmp_path / "nn").nn_classification_embeddings_output
    EC.main(emb_npz, tmp_path / "out", 0.9999, False)
    z = np.load(tmp_path / "out" / "sample_embedding_clusters.npz")
    assert z["representative_index"][5] == 1 and z["similarity"][5] >= np.float32(0.9999)
    lines = (tmp_path / "out" / "sample_embedding_clusters.tsv").read_text().splitlines()
    assert lines[0] == "seq_name\trepresentative\tcosine_similarity" and len(lines) == 1 + 7
    assert lines[6].split("\t")[:2] == ["seq5", "seq1"] and lines[1] == "seq0\tseq0\t1.000000"
    if torch.cuda.device_count() >= 2:                                       # torchrun x2: bitwise the files of one process
        s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
        r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                            "--master-addr", "127.0.0.1", "--master-port", str(port), "-m", "genomad_b200.cli",
                            "embedding-clusters", str(emb_npz), str(tmp_path / "out2"), "--min-similarity", "0.9999", "-q"],
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        for ext in ("tsv", "npz"):
            assert (tmp_path / "out" / f"sample_embedding_clusters.{ext}").read_bytes() == \
                (tmp_path / "out2" / f"sample_embedding_clusters.{ext}").read_bytes()
