"""
NumPy oracle of the embedding index (include/gnm.h, "Embedding index"; DESIGN.md): the training order, the initial centroids,
the re-seed rule, the final layout and the probed-union search.  Every step takes the similarity as a function
sim(Q, R) -> [len(Q), len(R)], so the same code states the rules in fp64 (tests/test_ivf_cpu.py) and, given the device's own
similarities, checks the device's steps (tests/test_gpu_ivf.py).
"""
import numpy as np

from genomad_b200.synth import _keys, _mix32

M32 = 0xFFFFFFFF
TRAIN_PER_LIST = 256


def cosine64(Q, R):
    """fp64 cosine similarity; a zero row has similarity 0 with every row."""
    def unit(x):
        x = np.asarray(x, np.float64)
        n = np.linalg.norm(x, axis=1, keepdims=True)
        return np.divide(x, n, out=np.zeros_like(x), where=n > 0)
    return unit(Q) @ unit(R).T


def training_rows(n, lists, seed):
    """The training rows: rows ordered by (mix32(key ^ row), row), the first min(n, 256 lists)."""
    r = np.arange(n, dtype=np.int64)
    with np.errstate(over="ignore"):
        h = _mix32((r & M32) ^ _keys(seed)[0])
    return np.lexsort((r, h))[: min(n, TRAIN_PER_LIST * lists)]


def normalize(x):
    """x / its fp64 norm, rounded to fp32 (a zero row stays zero)."""
    x = np.asarray(x, np.float32).astype(np.float64)
    n = np.sqrt(np.sum(x * x, axis=1, keepdims=True))
    return np.divide(x, n, out=np.zeros_like(x), where=n > 0).astype(np.float32)


def top(S, k, exclude=None):
    """Per row of S [nq, nr]: the first k columns under (s descending, column ascending), padded with (-inf, -1).
    exclude [nq]: a column each row skips (-1: none)."""
    nq, nr = S.shape
    sim = np.full((nq, k), -np.inf, np.float64)
    idx = np.full((nq, k), -1, np.int64)
    cols = np.arange(nr)
    for i in range(nq):
        keep = cols != (exclude[i] if exclude is not None else -1)
        o = np.lexsort((cols[keep], -S[i][keep]))[:k]
        sim[i, :len(o)], idx[i, :len(o)] = S[i][keep][o], cols[keep][o]
    return sim, idx


def assign(sim, X, C):
    """k = 1 centroid of each row, the row as the query: (best similarity, list)."""
    s, i = top(sim(X, C), 1)
    return s[:, 0], i[:, 0]


def centroids(xhat, lists_of, lists):
    """Each list's normalised mean of its normalised rows (fp64 sums); an empty list gives the zero row."""
    sums = np.zeros((lists, xhat.shape[1]), np.float64)
    np.add.at(sums, lists_of, np.asarray(xhat, np.float64))
    return normalize(sums)


def reseed(cent, xhat, train, best, lists_of):
    """Empty lists, ascending, each take the normalised training row not yet taken with the lowest best similarity (ties: the
    lowest row).  Returns (centroids, the reseeded lists)."""
    lists = cent.shape[0]
    empty = np.flatnonzero(np.bincount(lists_of, minlength=lists) == 0)
    order = np.lexsort((train, best))
    out = cent.copy()
    out[empty] = xhat[order[: len(empty)]]
    return out, empty


def layout(lists_of, lists):
    """(rows, offsets): the rows stably sorted by list."""
    rows = np.argsort(lists_of, kind="stable").astype(np.int64)
    offsets = np.zeros(lists + 1, np.int64)
    np.cumsum(np.bincount(lists_of, minlength=lists), out=offsets[1:])
    return rows, offsets


def build(rows, lists, iterations, seed, sim=cosine64):
    """The whole build: (centroids, rows, offsets)."""
    train = training_rows(len(rows), lists, seed)
    xhat = normalize(rows[train])
    cent = xhat[:lists].copy()
    for _ in range(iterations):
        best, a = assign(sim, xhat, cent)
        cent, _ = reseed(centroids(xhat, a, lists), xhat, train, best, a)
    _, a = assign(sim, rows, cent)
    r, off = layout(a, lists)
    return cent, r, off


def probes(Q, cent, nprobe, sim=cosine64):
    return top(sim(Q, cent), nprobe)[1]


def search(Q, R, cent, rows, offsets, k, nprobe, self_index0=-1, sim=cosine64):
    """The top-k under the total order over the rows of each query's probed lists, its self index excluded: (sim, idx)."""
    P = probes(Q, cent, nprobe, sim)
    S = sim(Q, R)
    out_s = np.full((len(Q), k), -np.inf, np.float64)
    out_i = np.full((len(Q), k), -1, np.int64)
    for q in range(len(Q)):
        cand = np.concatenate([rows[offsets[l]:offsets[l + 1]] for l in P[q]]) if len(P[q]) else np.zeros(0, np.int64)
        if self_index0 >= 0:
            cand = cand[cand != self_index0 + q]
        o = np.lexsort((cand, -S[q, cand]))[:k]
        out_s[q, :len(o)], out_i[q, :len(o)] = S[q, cand[o]], cand[o]
    return out_s, out_i
