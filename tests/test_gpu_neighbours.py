"""
Embedding neighbours on the H100 (gnm_embedding_neighbours; run with `-m gpu -s` for the measured errors): every returned
similarity within EPS of the fp64 cosine of the fp32 rows, the returned set agreeing with fp64's top-k up to 2 EPS, lists in
the total order (similarity descending, index ascending), padding, self-exclusion, and the bitwise identities the
multi-chunk and multi-GPU paths rest on (chunks + merges = one call, index offsets, query permutations, repeats).
"""
import time
from pathlib import Path

import numpy as np
import pytest
import torch

from genomad_b200 import engine, synth

pytestmark = pytest.mark.gpu

EPS = 1e-5          # a third of 512 * 2^-24, the fp32 linear accumulation bound; split-TF32's dropped terms add ~2^-20
WORST = {"err": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    print(f"\n{Path(__file__).name}: {time.time() - t0:.0f} s; worst |s - cos64| = {WORST['err']:.3e} (bar {EPS:.0e})")


def cos64(q, r):
    q64, r64 = q.astype(np.float64), r.astype(np.float64)
    nq, nr = np.linalg.norm(q64, axis=1), np.linalg.norm(r64, axis=1)
    q64 = np.divide(q64, nq[:, None], out=np.zeros_like(q64), where=nq[:, None] > 0)
    r64 = np.divide(r64, nr[:, None], out=np.zeros_like(r64), where=nr[:, None] > 0)
    return q64 @ r64.T


def check(q, r, k, sim, idx, ref_index0=0, self_index0=-1, dup_of=None):
    """sim, idx: numpy results of the GPU.  dup_of[j] = the lowest index of the rows identical to row j (ties)."""
    c = cos64(q, r)
    nq, nr = c.shape
    assert sim.shape == idx.shape == (nq, k) and sim.dtype == np.float32 and idx.dtype == np.int64
    for i in range(nq):
        cand = np.ones(nr, bool)
        if self_index0 >= 0 and 0 <= self_index0 + i - ref_index0 < nr:
            cand[self_index0 + i - ref_index0] = False
        n_cand = int(cand.sum())
        m = min(k, n_cand)
        s_i, x_i = sim[i], idx[i]
        assert np.all(x_i[m:] == -1) and np.all(np.isneginf(s_i[m:])), f"query {i}: padding"
        x, s = x_i[:m] - ref_index0, s_i[:m]
        assert np.all((x >= 0) & (x < nr)) and np.all(cand[x]) and len(set(x.tolist())) == m, f"query {i}: indices"
        err = np.abs(s.astype(np.float64) - c[i, x])
        WORST["err"] = max(WORST["err"], float(err.max(initial=0.0)))
        assert err.max(initial=0.0) <= EPS, f"query {i}: |s - cos64| = {err.max():.3e}"
        order = sorted(range(m), key=lambda j: (-float(s[j]), int(x[j])))
        assert order == list(range(m)), f"query {i}: list not in (similarity desc, index asc) order"
        if m == 0:
            continue
        ci = np.where(cand, c[i], -np.inf)
        t = np.sort(ci)[::-1][m - 1]
        must = np.flatnonzero(ci > t + 2 * EPS)
        assert set(must.tolist()) <= set(x.tolist()), f"query {i}: a reference above t + 2 eps is missing"
        assert np.all(c[i, x] >= t - 2 * EPS), f"query {i}: a returned reference is below t - 2 eps"
        if dup_of is not None:
            for j in x:
                lo = dup_of[j]
                assert lo == j or lo in set(x.tolist()) or not cand[lo], f"query {i}: duplicate {j} returned before {lo}"


def run(q, r=None, k=10, **kw):
    dq = torch.from_numpy(q).cuda()
    dr = None if r is None else torch.from_numpy(r).cuda()
    sim, idx = engine.embedding_neighbours(dq, dr, k, **kw)
    torch.cuda.synchronize()
    return sim.cpu().numpy(), idx.cpu().numpy()


def sparse_rows(n, seed):
    rng = np.random.default_rng(seed)
    x = np.maximum(rng.standard_normal((n, 512)), 0) * (rng.random((n, 512)) < 0.3)
    return x.astype(np.float32)


@pytest.mark.parametrize("nq", [1, 63, 64, 65, 129, 1000])
@pytest.mark.parametrize("nr", [1, 255, 256, 257, 5000])
def test_sizes_against_fp64(nq, nr):
    q, r = sparse_rows(nq, 1 + nq), sparse_rows(nr, 2 + nr)
    for k in (1, 10, 64):
        sim, idx = run(q, r, k)
        check(q, r, k, sim, idx)


@pytest.mark.parametrize("n", [1, 65, 257, 1000])
def test_all_vs_all_excludes_self(n):
    x = sparse_rows(n, 7)
    for k in (1, 10, 64):
        sim, idx = run(x, None, k)
        check(x, x, k, sim, idx, self_index0=0)
        assert not np.any(idx == np.arange(n)[:, None])


def test_near_duplicates_exact_duplicates_and_zero_rows():
    rng = np.random.default_rng(5)
    base = sparse_rows(40, 9)
    fam = [base]
    for rel in (1e-4, 1e-5, 1e-6, 1e-7):
        fam.append((base * (1 + rel * rng.standard_normal(base.shape))).astype(np.float32))
    r = np.concatenate([sparse_rows(700, 10)] + fam + [np.zeros((3, 512), np.float32)])     # families at rows 700 .. 899
    # exact duplicates across the 192-row reference tiles and the 128-row query tiles
    dup_of = np.arange(len(r) + 4)
    extra = []
    for src in (191, 5, 383):
        extra.append(r[src])
    r = np.concatenate([r, np.stack(extra)])
    for j, src in zip(range(len(r) - 3, len(r)), (191, 5, 383)):
        dup_of[j] = src
    r[192] = r[191]; dup_of[192] = 191
    r[128] = r[127]; dup_of[128] = 127
    dup_of = dup_of[: len(r)]
    q = np.concatenate([base, r[[191, 127, 5]], np.zeros((2, 512), np.float32)])
    for k in (1, 10, 64):
        sim, idx = run(q, r, k)
        check(q, r, k, sim, idx, dup_of=dup_of)
        assert np.all(sim[-2:][np.isfinite(sim[-2:])] == 0)                 # a zero query: similarity 0 with everything
    sim, idx = run(r, None, 10)                                              # all-vs-all: a row's duplicate is its neighbour
    check(r, r, 10, sim, idx, self_index0=0, dup_of=dup_of)
    assert idx[191, 0] == 192 and idx[192, 0] == 191 and sim[191, 0] == sim[192, 0]


def test_real_embeddings(weights_npz, golden_dir):
    from oracle import igloo_model as M
    c = engine.Classifier(M.load_npz_weights(weights_npz), device=0, max_batch=64)
    try:
        tok = np.load(golden_dir / "encoder_batch_tokens.npz")["tokens"]
        _, emb = c.embed_tokens(torch.from_numpy(tok.view(np.int16)).cuda().view(torch.uint16))
        rng = np.random.default_rng(11)
        seqs = [np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, ln)].tobytes() for ln in (30000, 500, 14000, 9000, 6000)]
        seqs += [seqs[0][:12000], seqs[2]]                                 # a prefix and an exact copy
        *_, cemb = c.classify_contigs(seqs, return_embeddings=True)
        for e in (emb, cemb):
            x = e.cpu().numpy()
            for k in (1, 10, 64):
                sim, idx = run(x, None, k)
                check(x, x, k, sim, idx, self_index0=0)
        x = cemb.cpu().numpy()
        sim, idx = run(x, None, 1)
        assert idx[2, 0] == 6 and idx[6, 0] == 2                            # the exact copy is the nearest
    finally:
        c.close()


def test_all_vs_all_100k_sampled():
    n = 100_000
    x = sparse_rows(n, 21)
    x[n // 2: n // 2 + 1000] = (x[:1000] * 1.0000001).astype(np.float32)   # near-duplicate pairs far apart
    t0 = time.time()
    sim, idx = run(x, None, 10)
    print(f"\nall-vs-all n = {n}, k = 10: {time.time() - t0:.2f} s including copies")
    sample = np.random.default_rng(3).choice(n, 200, replace=False)
    sample[:5] = [0, 1, n // 2, n // 2 + 1, n - 1]
    for i in sample:
        c = cos64(x[i:i + 1], x)[0]
        c[i] = -np.inf
        t = np.sort(c)[::-1][9]
        s, j = sim[i], idx[i]
        assert np.all(np.abs(s.astype(np.float64) - c[j]) <= EPS)
        WORST["err"] = max(WORST["err"], float(np.abs(s.astype(np.float64) - c[j]).max()))
        assert set(np.flatnonzero(c > t + 2 * EPS).tolist()) <= set(j.tolist())
        assert np.all(c[j] >= t - 2 * EPS) and i not in set(j.tolist())
        assert sorted(range(10), key=lambda a: (-float(s[a]), int(j[a]))) == list(range(10))


def test_bitwise_identities():
    q, r = sparse_rows(300, 31), sparse_rows(2000, 32)
    r[1500] = r[100]                                                        # a tie across chunks
    dq, dr = torch.from_numpy(q).cuda(), torch.from_numpy(r).cuda()
    for k in (1, 10, 64):
        s1, i1 = engine.embedding_neighbours(dq, dr, k)
        s2, i2 = engine.embedding_neighbours(dq, dr, k)
        assert torch.equal(s1, s2) and torch.equal(i1, i2), "repeat"
        # three chunks with their global offsets + merges
        cuts = [0, 700, 1401, 2000]
        sm, im = engine.embedding_neighbours(dq, dr[cuts[0]:cuts[1]], k, ref_index0=0)
        for a, b in zip(cuts[1:-1], cuts[2:]):
            sb, ib = engine.embedding_neighbours(dq, dr[a:b], k, ref_index0=a)
            engine.neighbours_merge(sm, im, sb, ib)
        assert torch.equal(sm, s1) and torch.equal(im, i1), "chunks + merges"
        # shifted ref_index0
        s3, i3 = engine.embedding_neighbours(dq, dr, k, ref_index0=10**12)
        assert torch.equal(s3, s1) and torch.equal(i3, i1 + 10**12), "ref_index0"
        # permuted queries
        perm = torch.from_numpy(np.random.default_rng(k).permutation(len(q))).cuda()
        s4, i4 = engine.embedding_neighbours(dq[perm], dr, k)
        assert torch.equal(s4, s1[perm]) and torch.equal(i4, i1[perm]), "query permutation"
        # all-vs-all in chunks with self-exclusion = one call
        sa, ia = engine.embedding_neighbours(dr, None, k)
        sc, ic = engine.embedding_neighbours(dr, dr[:1000], k, ref_index0=0, self_index0=0)
        sd, idd = engine.embedding_neighbours(dr, dr[1000:], k, ref_index0=1000, self_index0=0)
        engine.neighbours_merge(sc, ic, sd, idd)
        assert torch.equal(sc, sa) and torch.equal(ic, ia), "all-vs-all in chunks"


def test_errors():
    d = torch.zeros((4, 512), device="cuda")
    with pytest.raises(ValueError):
        engine.embedding_neighbours(d, None, 0)
    with pytest.raises(ValueError):
        engine.embedding_neighbours(d, None, 65)
    lib = engine.load_library()
    assert lib.gnm_embedding_neighbours(d.data_ptr(), 4, d.data_ptr(), 4, 0, -1, 10, d.data_ptr(), d.data_ptr(), d.data_ptr(),
                                        16, None) != 0
    assert b"workspace too small" in lib.gnm_last_error()
    assert lib.gnm_neighbours_workspace_bytes(4, 4, 0) == 0 and b"k must be" in lib.gnm_last_error()
    assert lib.gnm_embedding_neighbours(d.data_ptr(), 2**31, d.data_ptr(), 4, 0, -1, 10, None, None, None, 0, None) != 0
    assert b"2^30" in lib.gnm_last_error()


def test_empty_reference_gives_padding():
    q = torch.from_numpy(sparse_rows(5, 1)).cuda()
    sim, idx = engine.embedding_neighbours(q, q[:0], 4)
    assert torch.all(idx == -1) and torch.all(torch.isneginf(sim))


def test_module_end_to_end(tmp_path):
    from genomad_b200 import _paths, embedding_neighbours as EN, nn_classification
    rng = np.random.default_rng(17)
    fa = tmp_path / "sample.fna"
    seqs = ["".join(rng.choice(list("ACGT"), n)) for n in (9000, 15000, 6500, 20000, 7000)]
    seqs.append(seqs[1])
    fa.write_text("".join(f">seq{i}\n{s}\n" for i, s in enumerate(seqs)))
    nn_classification.main(fa, tmp_path / "nn", False, 128, False, 2, False, False, write_embeddings=True)
    emb_npz = _paths.NNOutputs("sample", tmp_path / "nn").nn_classification_embeddings_output
    EN.main(emb_npz, None, tmp_path / "out", 3, False)
    z = np.load(tmp_path / "out" / "sample_embedding_neighbours.npz")
    e = np.load(emb_npz)
    x = e["embeddings"]
    check(x, x, 3, z["similarity"], z["neighbour_index"], self_index0=0)
    assert list(z["query_names"]) == list(e["contig_names"]) and int(z["k"]) == 3
    assert z["neighbour_index"][1, 0] == 5 and z["neighbour_index"][5, 0] == 1
    lines = (tmp_path / "out" / "sample_embedding_neighbours.tsv").read_text().splitlines()
    assert lines[0] == "seq_name\trank\tneighbour_name\tcosine_similarity" and len(lines) == 1 + 6 * 3
    assert lines[1 + 3 * 1].split("\t")[:3] == ["seq1", "1", "seq5"]
