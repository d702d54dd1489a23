"""
NumPy fp64 oracle of the embedding map's steps 2-5 (include/gnm.h and DESIGN.md, "Embedding map"): memberships and their fuzzy
union, the CSR graph, the PCA initialisation with its hashed noise, and the synchronous layout epochs with their hashed
negatives, plus the a-priori bound of one GPU epoch (fp32 per term) against the fp64 epoch.
"""
import numpy as np

from genomad_b200 import engine
from genomad_b200.synth import _keys, _mix32

M32 = 0xFFFFFFFF
A32, B32 = float(np.float32(engine.MAP_A)), float(np.float32(engine.MAP_B))   # the kernel's fp32 constants
U32 = 2.0 ** -24


def key(seed: int) -> int:
    return _keys(seed)[0]


def mix32(x):
    with np.errstate(over="ignore"):
        return _mix32(np.asarray(x, np.int64) & M32)


def knn(emb, k):
    """All-vs-all lists in gnm_embedding_neighbours' order (s descending, index ascending), s the fp64 cosine in fp32."""
    x = np.asarray(emb, np.float64)
    nr = np.linalg.norm(x, axis=1)
    xn = np.divide(x, nr[:, None], out=np.zeros_like(x), where=nr[:, None] > 0)
    c = (xn @ xn.T).astype(np.float32)
    n = len(x)
    sim, idx = np.empty((n, k), np.float32), np.empty((n, k), np.int64)
    for i in range(n):
        g = np.delete(np.arange(n), i)
        o = np.lexsort((g, -c[i, g]))[:k]
        sim[i], idx[i] = c[i, g[o]], g[o]
    return sim, idx


def psum(d, rho, sigma):
    x = d - rho
    return np.where(x > 0, np.exp(-np.maximum(x, 0) / sigma), 1.0).sum(-1)


def membership(sim, idx):
    """(mean_d, rho [n], sigma [n], steps [n], w [n, k], union [n, k]) as gnm_map_membership states them; steps = the
    bisection steps taken (64 = no early exit)."""
    d = 1.0 - sim.astype(np.float64)
    n, k = d.shape
    mean_d = d.mean()
    target = np.log2(k + 1.0)
    rho = np.array([row[row > 0].min() if (row > 0).any() else 0.0 for row in d])
    sigma, steps = np.empty(n), np.empty(n, np.int64)
    for i in range(n):
        lo, hi, mid = 0.0, np.inf, 1.0
        it = 0
        for it in range(64):
            ps = psum(d[i], rho[i], mid)
            if abs(ps - target) < 1e-5:
                break
            if ps > target:
                hi = mid
                mid = (lo + hi) / 2.0
            else:
                lo = mid
                mid = mid * 2.0 if hi == np.inf else (lo + hi) / 2.0
        else:
            it = 64
        steps[i] = it
        fl = 1e-3 * (d[i].mean() if rho[i] > 0 else mean_d)
        sigma[i] = max(mid, fl)
    x = d - rho[:, None]
    w = np.where(x > 0, np.exp(-np.maximum(x, 0) / sigma[:, None]), 1.0)
    union = np.full((n, k), -1.0)
    for i in range(n):
        for p in range(k):
            j = idx[i, p]
            q = np.flatnonzero(idx[j] == i)
            b = w[j, q[0]] if len(q) else 0.0
            if not len(q) or i < j:
                union[i, p] = w[i, p] + b - w[i, p] * b
    return mean_d, rho, sigma, steps, w, union


def graph(union, idx, epochs):
    """(row_ptr, col, weight, eps): both directions of every union weight >= max / epochs, rows sorted by column."""
    n, k = union.shape
    u = union.reshape(-1)
    mw = u.max()
    e = np.flatnonzero(u >= mw / epochs)
    i, j, w = e // k, idx.reshape(-1)[e], u[e]
    rows, cols, ws = np.concatenate([i, j]), np.concatenate([j, i]), np.concatenate([w, w])
    o = np.lexsort((cols, rows))
    rows, cols, ws = rows[o], cols[o], ws[o]
    row_ptr = np.zeros(n + 1, np.int64)
    row_ptr[1:] = np.cumsum(np.bincount(rows, minlength=n))
    return row_ptr, cols, ws, mw / ws


def normalize(x):
    x = np.asarray(x, np.float64)
    nr = np.sqrt((x * x).sum(1))
    return np.divide(x, nr[:, None], out=np.zeros_like(x), where=nr[:, None] > 0).astype(np.float32)


def pca(rows):
    """(xhat fp32, center, S, V [2, 512]) in fp64 with numpy.linalg.eigh, signed as gnm_map_pca signs."""
    xh = normalize(rows)
    x = xh.astype(np.float64)
    center = x.mean(0)
    S = (x - center).T @ (x - center) / len(x)
    lam, vec = np.linalg.eigh(S)
    V = vec[:, ::-1][:, :2].T.copy()
    for v in V:
        if v[np.argmax(np.abs(v))] < 0:
            v *= -1
    return xh, center, S, V


def noise(seed, n):
    """float32 [n, 2]: (mix32(mix32(key ^ row) + axis) - 2^31 + 0.5) * 1e-4 / 2^31."""
    r = np.arange(n, dtype=np.int64)[:, None]
    h = mix32(mix32(r ^ key(seed)) + np.arange(2)[None, :])
    return ((h.astype(np.float64) - 2147483647.5) * (1e-4 / 2147483648.0)).astype(np.float32)


def init_from_projection(proj, seed):
    """gnm_map_init after its projection, in the kernel's fp32 and fp64 operations."""
    m = np.abs(proj).max()
    base = (proj * (10.0 / m)).astype(np.float32) if m > 0 else np.zeros(proj.shape, np.float32)
    y = (base + noise(seed, len(proj))).astype(np.float32)
    lo, hi = y.min(0), y.max(0)
    rng = (hi - lo).astype(np.float32)
    out = np.zeros_like(y)
    for a in range(2):
        if rng[a] > 0:
            out[:, a] = (np.float32(10) * (y[:, a] - lo[a])) / rng[a]
    return out.astype(np.float32)


def sampled(eps, e):
    return (e >= 1) & (np.floor(e / eps) > np.floor((e - 1) / eps))


def negatives(p, e, seed, n):
    """[len(p), 5] negative vertices of CSR positions p at epoch e."""
    hp = mix32(mix32(key(seed) ^ e) + np.asarray(p, np.int64))
    return mix32(hp[:, None] + np.arange(5)[None, :]) % n


def _att(d2):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(d2 > 0, -2.0 * A32 * B32 * d2 ** (B32 - 1) / (1.0 + A32 * d2 ** B32), 0.0)


def _rep(d2):
    return np.where(d2 > 0, 2.0 * B32 / ((float(np.float32(0.001)) + d2) * (1.0 + A32 * d2 ** B32)), 0.0)


def epoch_terms(row_ptr, col, eps, Y, e, seed, *, att_factor=2.0, n_neg=5, clip=4.0):
    """The terms of epoch e, fp64 on the fp32 Y: (vertex [m], term [m, 2]), in CSR order, each entry's attraction (times
    att_factor) then its negatives."""
    n = len(Y)
    y = np.asarray(Y, np.float64)
    rows = np.repeat(np.arange(n), np.diff(row_ptr))
    p = np.flatnonzero(sampled(eps, e))
    i, j = rows[p], col[p]
    cl = (lambda t: np.clip(t, -clip, clip)) if clip is not None else (lambda t: t)
    dy = y[i] - y[j]
    verts, terms, raw = [i], [att_factor * cl(_att((dy * dy).sum(1))[:, None] * dy)], [_att((dy * dy).sum(1))[:, None] * dy]
    neg = negatives(p, e, seed, n)
    for s in range(n_neg):
        kk = neg[:, s]
        keep = kk != i
        dy = y[i[keep]] - y[kk[keep]]
        t = _rep((dy * dy).sum(1))[:, None] * dy
        verts.append(i[keep]), terms.append(cl(t)), raw.append(t)
    return np.concatenate(verts), np.concatenate(terms), np.concatenate(raw)


def alpha(e, epochs):
    return float(np.float32(1.0 - e / epochs))


def epoch(row_ptr, col, eps, Y, e, epochs, seed, **inject):
    """Y after epoch e in fp64 (Y fp32 [n, 2] in); inject: epoch_terms' fault switches."""
    v, t, _ = epoch_terms(row_ptr, col, eps, Y, e, seed, **inject)
    F = np.zeros((len(Y), 2))
    np.add.at(F, v, t)
    return np.asarray(Y, np.float64) + alpha(e, epochs) * F


def epoch_bound(row_ptr, col, eps, Y, e, epochs, seed):
    """Elementwise a-priori bound on |GPU epoch - epoch()| for the same Y and samples.  Per term: d^2 from fp32 differences and
    products (gamma_4 relative), two powf each allowed 8 ulp (16 u relative), the fp32 constants, products, sum and quotient
    (8 u): delta = (|b - 1| + b) gamma_4 + 2 * 16 u + 8 u, doubled for second-order terms, on the unclipped term; clip is
    1-Lipschitz and a term whose |T| (1 - delta) >= 4 clips to the same value.  The fp32 sum of m terms in any order adds
    gamma_(m-1) sum |T|; alpha * sum and the update add u each."""
    u = U32
    g4 = 4 * u / (1 - 4 * u)
    delta = 2 * ((abs(B32 - 1) + B32) * g4 + 32 * u + 8 * u)
    v, t, raw = epoch_terms(row_ptr, col, eps, Y, e, seed)
    fac = np.ones(len(v))
    n_att = np.flatnonzero(sampled(eps, e)).size
    fac[:n_att] = 2.0
    err = np.where(np.abs(raw) * (1 - delta) >= 4.0, 0.0, delta * np.abs(raw)) * fac[:, None]
    n = len(Y)
    E, A, M = np.zeros((n, 2)), np.zeros((n, 2)), np.bincount(v, minlength=n)
    np.add.at(E, v, err)
    np.add.at(A, v, np.abs(t) + err)
    F = np.zeros((n, 2))
    np.add.at(F, v, t)
    gm = np.maximum(M - 1, 0)[:, None] * u
    gm = gm / (1 - gm)
    a = alpha(e, epochs)
    Yn = np.abs(np.asarray(Y, np.float64) + a * F)
    return a * (E + gm * A) + u * a * (np.abs(F) + E + gm * A) + u * (Yn + a * (E + gm * A)) * (1 + 2 * u) + 1e-30


def run(emb, k, epochs, seed, trace=None):
    """The whole map in fp64 from the rows (kNN, memberships, graph, PCA initialisation, epochs); float64 [n, 2].  The epochs
    are computed in fp64 throughout and read Y rounded to fp32, as the kernel does."""
    sim, idx = knn(emb, k)
    _, _, _, _, _, union = membership(sim, idx)
    row_ptr, col, _, eps = graph(union, idx, epochs)
    xh, center, _, V = pca(emb)
    proj = (xh.astype(np.float64) - center) @ V.T
    Y = init_from_projection(proj, seed)
    for e in range(1, epochs):
        Y = epoch(row_ptr, col, eps, Y, e, epochs, seed).astype(np.float32)
    return Y


def blobs(n=2000, c=5, seed=0, scale=1.0):
    """n post-ReLU rows in c Gaussian blobs in 512-D, labels [n]."""
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((c, 512))
    lab = np.arange(n) % c
    x = np.maximum(centers[lab] + scale * rng.standard_normal((n, 512)), 0)
    return x.astype(np.float32), lab


def trustworthiness(emb, Y, k=15):
    from sklearn.manifold import trustworthiness as tw
    return float(tw(np.asarray(emb, np.float64), np.asarray(Y, np.float64), n_neighbors=k, metric="cosine"))


def knn_accuracy(Y, labels, k=15):
    from sklearn.model_selection import cross_val_score
    from sklearn.neighbors import KNeighborsClassifier
    return float(cross_val_score(KNeighborsClassifier(k), np.asarray(Y, np.float64), labels, cv=5).mean())
