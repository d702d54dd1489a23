"""
Embedding neighbours and clusters on the H100 at the edges of their input (run with `-m gpu -s` for the measured errors):
nb_prep_kernel's TF32 halves bitwise those of the CPU statement tests/nb_prep_ref.py on signed, one-hot, zero, subnormal and
extreme-scale rows; results bitwise invariant when every row is scaled by its own power of two; signed rows and negative
similarities against fp64 at the tile edges; exact ties pinned to the list the total order defines, across tiles, splits and
chunks; every k from 1 to 64; clustering of exact copies and of long chains against the fp64 greedy; and a query count past the
65,535 query tiles a 2-D grid's y dimension would allow.
"""
import time
from pathlib import Path

import numpy as np
import pytest
import torch

import nb_prep_ref as P
from genomad_b200 import embedding_clusters as EC, engine
from test_gpu_clusters import ONE, check_members, families, greedy64
from test_gpu_neighbours import EPS, WORST, check, cos64, run, sparse_rows

pytestmark = pytest.mark.gpu

F32 = np.float32
SCALES = (-140, -100, -76, -70, 0, 60, 62, 100)


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0, WORST["err"] = time.time(), 0.0
    yield
    print(f"\n{Path(__file__).name}: {time.time() - t0:.0f} s; worst |s - cos64| = {WORST['err']:.3e} (bar {EPS:.0e})")


def signed_rows(n, seed, density=0.5):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((n, 512)) * (rng.random((n, 512)) < density)).astype(F32)


def exact_scaling(x, xs):
    """Every nonzero entry of x and of its scaled copy xs is a normal float (none underflowed to zero): xs is x times 2^e exactly."""
    a, b = np.abs(x), np.abs(xs)
    tiny = np.finfo(F32).tiny
    return bool(np.all((a == 0) == (b == 0)) and np.all((a == 0) | (a >= tiny)) and np.all((b == 0) | (b >= tiny)))


def scale_rows(x, e):
    """Row i times 2^e[i], rounded once to float32."""
    return (x.astype(np.float64) * np.exp2(np.asarray(e, np.float64))[:, None]).astype(F32)


def gpu_halves(x):
    """The query halves nb_prep_kernel writes, read back from a workspace the test owns.  nb_plan (csrc/api.cu) lays the
    workspace out as q_hi at byte 0, then q_lo at nb_align(nq * 2048) (nb_align: up to a multiple of 256), then the reference's."""
    lib = engine.load_library()
    nq = x.shape[0]
    dq, dr = torch.from_numpy(x).cuda(), torch.ones((1, 512), device="cuda")
    need = int(lib.gnm_neighbours_workspace_bytes(nq, 1, 1))
    work = torch.zeros(need, dtype=torch.uint8, device="cuda")
    sim = torch.empty((nq, 1), dtype=torch.float32, device="cuda")
    idx = torch.empty((nq, 1), dtype=torch.int64, device="cuda")
    assert lib.gnm_embedding_neighbours(dq.data_ptr(), nq, dr.data_ptr(), 1, 0, -1, 1, sim.data_ptr(), idx.data_ptr(),
                                        work.data_ptr(), need, torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    off = (nq * 2048 + 255) // 256 * 256
    hi = work[: nq * 2048].view(torch.float32).reshape(nq, 512).cpu().numpy()
    lo = work[off: off + nq * 2048].view(torch.float32).reshape(nq, 512).cpu().numpy()
    return hi, lo


def prep_rows():
    rng = np.random.default_rng(50)
    one_hot = np.zeros((4, 512), F32)
    one_hot[np.arange(4), [0, 3, 200, 511]] = [1.0, -2.5, 0.375, 7.0]
    sub = (sparse_rows(3, 51) * F32(2.0 ** -135)).astype(F32)               # subnormal entries and a subnormal maximum
    sub[0, :] = 0
    sub[0, 17] = np.float32(2.0 ** -149)                                     # the smallest subnormal alone
    mixed = rng.standard_normal((3, 512)) * np.where(rng.random((3, 512)) < 0.5, 2.0 ** 60, 2.0 ** -60)
    return np.concatenate([sparse_rows(6, 52), signed_rows(6, 53), signed_rows(4, 54, 1.0), one_hot, np.zeros((2, 512), F32),
                           sub, mixed.astype(F32)])


def test_prep_halves_bitwise():
    x = prep_rows()
    base = P.prep(x)
    for e in SCALES:
        with np.errstate(over="ignore"):
            xs = scale_rows(x, np.full(len(x), e))
        keep = np.flatnonzero(np.isfinite(xs).all(axis=1))
        hi, lo = gpu_halves(np.ascontiguousarray(xs[keep]))
        want_hi, want_lo = P.prep(xs[keep])
        assert np.array_equal(hi.view(np.uint32), want_hi.view(np.uint32)), f"2^{e}: hi differs from nb_prep_ref"
        assert np.array_equal(lo.view(np.uint32), want_lo.view(np.uint32)), f"2^{e}: lo differs from nb_prep_ref"
        for j, i in enumerate(keep):                                         # scale invariance while every entry is normal
            if exact_scaling(x[i], xs[i]):
                assert np.array_equal(hi[j].view(np.uint32), base[0][i].view(np.uint32)), f"2^{e}: row {i} hi"
                assert np.array_equal(lo[j].view(np.uint32), base[1][i].view(np.uint32)), f"2^{e}: row {i} lo"


def random_scales(x, seed, lo=-100, hi=100):
    """A power of two per row with every nonzero entry of the scaled row still a normal float."""
    e = np.random.default_rng(seed).integers(lo, hi + 1, len(x))
    xs = scale_rows(x, e)
    assert all(exact_scaling(a, b) for a, b in zip(x, xs)) and np.isfinite(xs).all()
    return xs


def test_scale_invariance_end_to_end():
    q, r = sparse_rows(300, 60), sparse_rows(2000, 61)
    q[:5] = r[[0, 191, 192, 1000, 1999]]                                     # exact copies across reference tiles
    qs, rs = random_scales(q, 62), random_scales(r, 63)
    for k in (1, 10, 64):
        s0, i0 = run(q, r, k)
        s1, i1 = run(qs, rs, k)
        assert np.array_equal(s1, s0) and np.array_equal(i1, i0), f"k = {k}: query vs reference"
        check(qs, rs, k, s1, i1)
        s0, i0 = run(r, None, k)
        s1, i1 = run(rs, None, k)
        assert np.array_equal(s1, s0) and np.array_equal(i1, i0), f"k = {k}: all vs all"
        check(rs, rs, k, s1, i1, self_index0=0)


def test_cluster_scale_invariance():
    t = 0.95
    x, c = families(3000, t, 64)
    xs = random_scales(x, 65)
    ri64, reps64 = greedy64(c, t)
    for block in (engine.CLUSTER_MAX_BLOCK, 128):
        ref = EC.cluster(x, t, ONE, block=block)
        got = EC.cluster(xs, t, ONE, block=block)
        assert all(np.array_equal(a, b) for a, b in zip(got, ref)), f"block {block}"
        assert np.array_equal(got[2], reps64) and np.array_equal(got[0], ri64)


@pytest.mark.parametrize("nq", [1, 63, 64, 65, 129, 1000])
@pytest.mark.parametrize("nr", [1, 255, 256, 257, 5000])
def test_signed_sizes_against_fp64(nq, nr):
    q = np.concatenate([signed_rows(nq, 70 + nq), signed_rows(nq, 71 + nq, 0.3)])[::2].copy()
    r = np.concatenate([signed_rows(nr, 72 + nr), signed_rows(nr, 73 + nr, 0.3)])[1::2].copy()
    m = min(nq, nr, 40)
    r[:m] = -q[:m]                                                           # antipodes: s = -1
    for k in (1, 10, 64):
        sim, idx = run(q, r, k)
        check(q, r, k, sim, idx)
        if nr <= k:                                                          # the whole list: the antipode last, then pads
            assert np.all(idx[:m, nr - 1] == np.arange(m)) and np.all(sim[:m, nr - 1] <= -1 + EPS)


def test_all_negative_lists_and_antipodes():
    for nr in (1, 5, 63, 257):
        r = np.abs(signed_rows(nr, 80 + nr, 1.0))                            # positive references
        q = -np.abs(signed_rows(70, 81 + nr, 1.0))                           # negative queries: every s < 0
        for k in (1, 10, 64):
            sim, idx = run(q, r, k)
            check(q, r, k, sim, idx)
            fin = np.isfinite(sim)
            assert np.all(sim[fin] < 0) and fin.sum() == 70 * min(k, nr)
    x = signed_rows(30, 82)
    x = np.concatenate([x, -x])                                              # every row and its antipode: 59 candidates < 64
    sim, idx = run(x, None, 64)
    check(x, x, 64, sim, idx, self_index0=0)
    n = len(x)
    assert np.all(idx[:, 58] == (np.arange(n) + 30) % n) and np.all(sim[:, 58] <= -1 + EPS)
    assert np.all(idx[:, 59:] == -1) and np.all(np.isneginf(sim[:, 59:]))


def test_cluster_family_and_its_negation():
    t = 0.95
    x, _ = families(1000, t, 83, check=False)
    perm = np.random.default_rng(84).permutation(2000)
    x = np.concatenate([x, -x])[perm]
    at = np.argsort(perm)
    partner = at[(perm + 1000) % 2000]                                       # the position of each row's negation
    c = cos64(x, x)
    nz = np.abs(x).sum(1) > 0
    off = ~np.eye(len(x), dtype=bool) & nz[:, None] & nz[None, :]
    assert not np.any(np.abs(c[off] - t) < 1e-3), "construction: a pair near the threshold"
    ri64, reps64 = greedy64(c, t)
    for block in (engine.CLUSTER_MAX_BLOCK, 128):
        ri, sim, reps = EC.cluster(x, t, ONE, block=block)
        assert np.array_equal(reps, reps64) and np.array_equal(ri, ri64), f"block {block}"
        assert np.all(ri != ri[partner]), "a row shares a cluster with its negation"
        check_members(x, t, ri, sim, reps)


# ------------------------------------------------------------------------------------------------ exact ties
def tie_reference():
    """~3,000 bitwise copies of 5 well-separated base rows, interleaved at random: every tile, split and chunk holds copies."""
    rng = np.random.default_rng(90)
    base = sparse_rows(5, 91)
    c = cos64(base, base)
    assert np.max(c[np.triu_indices(5, 1)]) < 0.9
    which = rng.integers(0, 5, 3001)
    return base, which, base[which]


def expected_ties(qb_cos, which, k, drop=-1):
    """The list the total order defines when every copy of base b has one similarity, ordered as the bases' cos64: the
    copies of the best base by index, then those of the next base, ...; `drop` is the excluded row (self)."""
    out = []
    for b in np.argsort(-qb_cos, kind="stable"):
        rows = np.flatnonzero(which == b)
        out += [int(j) for j in rows if j != drop][: k - len(out)]
        if len(out) == k:
            break
    return np.array(out, np.int64)


def check_ties(q, base, which, k, sim, idx, ref_index0=0, self_rows=None):
    qb = cos64(q, base)
    for i in range(len(q)):
        drop = -1 if self_rows is None else self_rows[i]
        if not np.any(q[i]):                                                 # a zero query: similarity +0 with everything
            want = np.array([j for j in range(len(which)) if j != drop][:k], np.int64)
            assert np.all(sim[i] == 0) and not np.any(np.signbit(sim[i])), f"query {i}: not +0"
        else:
            assert np.min(np.diff(np.sort(qb[i]))) > 100 * EPS, f"construction: query {i} near two bases alike"
            want = expected_ties(qb[i], which, k, drop)
            got_b = which[idx[i] - ref_index0]
            for b in np.unique(got_b):                                       # every copy of a base: one similarity
                assert len(set(sim[i][got_b == b].tolist())) == 1, f"query {i}: copies of base {b} differ"
            err = np.abs(sim[i].astype(np.float64) - qb[i][got_b])
            WORST["err"] = max(WORST["err"], float(err.max()))
            assert err.max() <= EPS
        assert np.array_equal(idx[i], want + ref_index0), f"query {i}: {idx[i][:8]} ... against {want[:8] + ref_index0} ..."


@pytest.mark.parametrize("chunk", [None, 700])
def test_exact_ties_pinned(chunk, monkeypatch):
    if chunk:
        monkeypatch.setattr(engine, "NEIGHBOURS_CHUNK", chunk)               # read at call time: ties cross chunk merges
    base, which, r = tie_reference()
    rng = np.random.default_rng(92)
    pert = (base * (1 + 1e-3 * rng.standard_normal(base.shape))).astype(F32)
    q = np.concatenate([base, pert, np.zeros((2, 512), F32)])
    for k in (1, 10, 33, 64):
        dq, dr = torch.from_numpy(q).cuda(), torch.from_numpy(r).cuda()
        sim, idx = engine.embedding_neighbours(dq, dr, k, ref_index0=10**9 + 7)
        check_ties(q, base, which, k, sim.cpu().numpy(), idx.cpu().numpy(), ref_index0=10**9 + 7)
        sim, idx = run(r, None, k)                                           # all-vs-all: self-exclusion removes one copy
        check_ties(r, base, which, k, sim, idx, self_rows=np.arange(len(r)))


# ------------------------------------------------------------------------------------------------ every k
def test_every_k():
    nq, nr = 130, 1000                                                       # two query tiles (one partial), six reference tiles
    r = np.concatenate([signed_rows(nr // 2, 100), sparse_rows(nr - nr // 2, 101)])[np.random.default_rng(102).permutation(nr)]
    q = r[:nq]
    dq, dr = torch.from_numpy(q).cuda(), torch.from_numpy(r).cuda()
    for k in range(1, 65):
        s1, i1 = engine.embedding_neighbours(dq, dr, k, self_index0=-1)
        check(q, r, k, s1.cpu().numpy(), i1.cpu().numpy())
        sa, ia = engine.embedding_neighbours(dq, dr, k, self_index0=0)
        check(q, r, k, sa.cpu().numpy(), ia.cpu().numpy(), self_index0=0)
        for s0, i0, self0 in ((s1, i1, -1), (sa, ia, 0)):                    # two chunks + a merge = one call, bitwise
            sm, im = engine.embedding_neighbours(dq, dr[:577], k, ref_index0=0, self_index0=self0)
            sb, ib = engine.embedding_neighbours(dq, dr[577:], k, ref_index0=577, self_index0=self0)
            engine.neighbours_merge(sm, im, sb, ib)
            assert torch.equal(sm, s0) and torch.equal(im, i0), f"k = {k}, self_index0 = {self0}: chunks + merge"


# ------------------------------------------------------------------------------------------------ clustering edges
def test_cluster_exact_copies():
    base = sparse_rows(3, 110)
    x = np.repeat(base[:1], 9000, axis=0)                                    # one block of copies crossing a block edge
    ri, sim, reps = EC.cluster(x, 0.99, ONE)
    assert np.array_equal(reps, [0]) and np.all(ri == 0) and len(set(sim[1:].tolist())) == 1
    print(f"\na row's similarity with its exact copy: {sim[1]!r} (1 - s = {1 - float(sim[1]):.2e})")
    x = base[np.random.default_rng(111).integers(0, 3, 5000)]                # three interleaved blocks of copies
    first = [int(np.flatnonzero((x == b).all(1))[0]) for b in base]
    for block in (engine.CLUSTER_MAX_BLOCK, 128):
        ri, sim, reps = EC.cluster(x, 0.99, ONE, block=block)
        assert np.array_equal(reps, sorted(first))
        check_members(x, 0.99, ri, sim, reps)


def arcs(n_planes, steps, delta, seed):
    """Rows cos(th) e_2p + sin(th) e_2p+1 along an arc of `steps` angles delta apart in plane p, planes taken round-robin in
    file order (row i of every plane, then row i + 1, ...): within a plane cos64 = cos(m delta), across planes 0."""
    rng = np.random.default_rng(seed)
    th0 = rng.uniform(0, 2 * np.pi, n_planes)
    sign = rng.choice([-1.0, 1.0], n_planes)
    x = np.zeros((steps, n_planes, 512))
    th = th0[None, :] + sign[None, :] * delta * np.arange(steps)[:, None]
    p = np.arange(n_planes)
    x[:, p, 2 * p], x[:, p, 2 * p + 1] = np.cos(th), np.sin(th)
    return x.reshape(steps * n_planes, 512).astype(F32), np.tile(p, steps)


def test_cluster_long_chains():
    t, delta = 0.99, 0.05                                                    # cos(2 delta) = 0.9950, cos(3 delta) = 0.9888
    x, plane = arcs(167, 120, delta, 112)                                    # 20,040 rows
    reps64 = []
    for p in range(plane.max() + 1):                                         # the fp64 greedy plane by plane (others: cos 0)
        rows = np.flatnonzero(plane == p)
        c = cos64(x[rows], x[rows])
        assert not np.any(np.abs(c - t) < 1e-4), "construction: a pair near the threshold"
        reps64 += rows[greedy64(c, t)[1]].tolist()
    reps64 = np.array(sorted(reps64))
    for block in (engine.CLUSTER_MAX_BLOCK, 1000, 128):
        ri, sim, reps = EC.cluster(x, t, ONE, block=block)
        assert np.array_equal(reps, reps64), f"block {block}"
        members = np.flatnonzero(ri != np.arange(len(x)))
        assert np.all(plane[ri] == plane)
        for j in members:                                                    # the best representative, up to 2 EPS
            rows = reps[plane[reps] == plane[j]]
            c = cos64(x[j:j + 1], x[rows])[0]
            assert cos64(x[j:j + 1], x[ri[j]:ri[j] + 1])[0, 0] >= c.max() - 2 * EPS
        check_members(x, t, ri, sim, reps)


# ------------------------------------------------------------------------------------------------ the query-tile count
def test_more_query_tiles_than_a_grid_dimension():
    """65,536 * 128 + 1 query rows: 65,537 query tiles, past gridDim.y's 65,535.  About 52 GB of device memory."""
    free, _ = torch.cuda.mem_get_info()
    if free < 64 * 2 ** 30:
        pytest.skip(f"needs 64 GB of free device memory, {free / 2 ** 30:.0f} GB free")
    nq, m = 65_536 * 128 + 1, 7
    distinct = torch.from_numpy(signed_rows(m, 120)).cuda()
    ref = torch.from_numpy(signed_rows(3, 121)).cuda()
    small_s, small_i = engine.embedding_neighbours(distinct, ref, 1)
    rep = torch.arange(nq, device="cuda") % m
    q = distinct[rep]
    lib = engine.load_library()
    need = int(lib.gnm_neighbours_workspace_bytes(nq, 3, 1))
    work = torch.empty(need, dtype=torch.uint8, device="cuda")
    sim = torch.empty((nq, 1), dtype=torch.float32, device="cuda")
    idx = torch.empty((nq, 1), dtype=torch.int64, device="cuda")
    rc = lib.gnm_embedding_neighbours(q.data_ptr(), nq, ref.data_ptr(), 3, 0, -1, 1, sim.data_ptr(), idx.data_ptr(),
                                      work.data_ptr(), need, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.gnm_last_error()
    torch.cuda.synchronize()
    assert torch.equal(sim, small_s[rep]) and torch.equal(idx, small_i[rep])
    print(f"\n{nq} query rows in one call ({need / 2 ** 30:.1f} GB workspace): equal to the {m} distinct rows' call")
    del q, work, sim, idx
    torch.cuda.empty_cache()
