"""
fp64 NumPy oracle of the window-region decode (DESIGN.md, "Window regions"; gnm_window_regions, include/gnm.h).

Forward-backward runs in the log domain (logsumexp), an independent formulation from the kernel's scaled linear recursion.
Viterbi keeps the kernel's tie rule: stay first, then the lowest class index; the final state is the lowest index at the max.
"""
from __future__ import annotations

import numpy as np

WINDOW = 6000


def emissions(p, stride: int) -> np.ndarray:
    """eps [n, C] = (s / 6000) ln max(p, 1e-30) in fp64."""
    return (stride / WINDOW) * np.log(np.maximum(np.asarray(p, np.float64), 1e-30))


def gaps(start, stride: int) -> np.ndarray:
    """g_w = (a_w - a_{w-1}) / s for w >= 1 (g_0 = 1, unused)."""
    a = np.asarray(start, np.int64)
    g = np.ones(len(a), np.int64)
    g[1:] = (a[1:] - a[:-1]) // stride
    return g


def transition(C: int, stride: int, L: float, g):
    """(T_g, O_g): stay and move-to-a-given-other-class probabilities after g strides, computed as 1/C + (1 - 1/C) lambda^g and
    (1 - T_g) / (C - 1) without cancellation: O_g = -expm1(g log1p(-rho C / (C - 1))) / C, T_g = 1 - (C - 1) O_g."""
    rho = stride / L
    x = np.asarray(g, np.float64) * np.log1p(-rho * C / (C - 1))
    O = -np.expm1(x) / C
    return 1.0 - (C - 1) * O, O


def log_transition(C: int, stride: int, L: float, g):
    """(ln T_g, ln O_g) as the kernel forms them."""
    rho = stride / L
    x = np.asarray(g, np.float64) * np.log1p(-rho * C / (C - 1))
    O = -np.expm1(x) / C
    return np.log1p(-(C - 1) * O), np.log(O)


def _log_A(C, lt, lo):
    A = np.full((C, C), lo)
    np.fill_diagonal(A, lt)
    return A


def _lse(x, axis):
    m = np.max(x, axis=axis, keepdims=True)
    return (m + np.log(np.sum(np.exp(x - m), axis=axis, keepdims=True))).squeeze(axis)


def forward_backward(eps, g, C: int, stride: int, L: float) -> np.ndarray:
    """gamma [n, C]."""
    n = eps.shape[0]
    if n == 0:
        return np.zeros((0, C))
    lt, lo = log_transition(C, stride, L, g)
    la = np.empty((n, C))
    la[0] = eps[0] - np.log(C)
    for w in range(1, n):
        la[w] = eps[w] + _lse(la[w - 1][:, None] + _log_A(C, lt[w], lo[w]), 0)
    lb = np.zeros((n, C))
    for w in range(n - 2, -1, -1):
        lb[w] = _lse(_log_A(C, lt[w + 1], lo[w + 1]) + (eps[w + 1] + lb[w + 1])[None, :], 1)
    z = la + lb
    return np.exp(z - _lse(z, 1)[:, None])


def viterbi(eps, g, C: int, stride: int, L: float):
    """(path int [n], best score): delta_w(k) = eps_w(k) + max(delta_{w-1}(k) + ln T, max_{j != k} delta_{w-1}(j) + ln O); a
    tie goes to staying, then to the lowest j; the final state is the lowest index at the max."""
    n = eps.shape[0]
    if n == 0:
        return np.zeros(0, np.int64), 0.0
    lt, lo = log_transition(C, stride, L, g)
    d = eps[0] - np.log(C)
    back = np.zeros((n, C), np.int64)
    idx = np.arange(C)
    for w in range(1, n):
        order = np.lexsort((idx, -d))          # descending value, ascending index
        a1, a2 = order[0], order[1]
        other = np.where(idx == a1, d[a2], d[a1])
        arg_other = np.where(idx == a1, a2, a1)
        stay, move = d + lt[w], other + lo[w]
        st = stay >= move
        back[w] = np.where(st, idx, arg_other)
        d = eps[w] + np.where(st, stay, move)
    s = int(np.flatnonzero(d == d.max())[0])
    best = float(d[s])
    path = np.empty(n, np.int64)
    path[-1] = s
    for w in range(n - 1, 0, -1):
        s = int(back[w, s])
        path[w - 1] = s
    return path, best


def path_score(path, eps, g, C: int, stride: int, L: float) -> float:
    """ln(1/C) + sum_w eps_w(s_w) + sum_{w>=1} ln A_{g_w}(s_{w-1}, s_w), summed in fp64 in window order."""
    n = len(path)
    if n == 0:
        return 0.0
    lt, lo = log_transition(C, stride, L, g)
    tot = -np.log(C) + eps[0, path[0]]
    for w in range(1, n):
        tot += (lt[w] if path[w] == path[w - 1] else lo[w]) + eps[w, path[w]]
    return float(tot)


def margins(eps, g, C: int, stride: int, L: float) -> np.ndarray:
    """Per window, the gap between the best path score and the best score of a path through another state at that window
    (max-marginals): where it exceeds the decode's rounding, every optimal path has the same state there."""
    n = eps.shape[0]
    if n == 0:
        return np.zeros(0)
    lt, lo = log_transition(C, stride, L, g)
    fw = np.empty((n, C))
    fw[0] = eps[0] - np.log(C)
    for w in range(1, n):
        fw[w] = eps[w] + np.max(fw[w - 1][:, None] + _log_A(C, lt[w], lo[w]), 0)
    bw = np.zeros((n, C))
    for w in range(n - 2, -1, -1):
        bw[w] = np.max(_log_A(C, lt[w + 1], lo[w + 1]) + (eps[w + 1] + bw[w + 1])[None, :], 1)
    mm = np.sort(fw + bw, 1)
    return mm[:, -1] - mm[:, -2]


def regions(path, gamma, p, start, length):
    """Region table of one sequence from its path: list of (start, end, class, n_windows, posterior f32, scores f32 [C]),
    means as fp64 sums in window order."""
    n = len(path)
    out = []
    if n == 0:
        return out
    a = np.asarray(start, np.int64)
    ln = np.asarray(length, np.int64)
    c = a + ln // 2
    p64 = np.asarray(p, np.float32).astype(np.float64)
    i = 0
    while i < n:
        j = i
        while j + 1 < n and path[j + 1] == path[i]:
            j += 1
        k = int(path[i])
        rs = int(a[0]) if i == 0 else int((c[i - 1] + c[i]) // 2)
        re = int(a[n - 1] + ln[n - 1]) if j == n - 1 else int((c[j] + c[j + 1]) // 2)
        m = j - i + 1
        post = np.float32(np.cumsum(gamma[i:j + 1, k])[-1] / m)
        sc = (np.cumsum(p64[i:j + 1], 0)[-1] / m).astype(np.float32)
        out.append((rs, re, k, m, post, sc))
        i = j + 1
    return out


def decode(probs, offsets, start, length, stride: int, L: float, path_override=None):
    """The whole profile (numpy): dict of posterior [W, C], state [W] and the region_* arrays, as engine.window_regions returns
    them.  path_override: a path [W] to build the region table from (the GPU's), instead of the oracle's Viterbi path."""
    probs = np.asarray(probs, np.float32)
    C = probs.shape[1]
    offsets = np.asarray(offsets, np.int64)
    W = probs.shape[0]
    post = np.zeros((W, C))
    state = np.zeros(W, np.int64)
    best = np.zeros(len(offsets) - 1)
    rows = {k: [] for k in ("contig", "start", "end", "class", "windows", "posterior", "scores")}
    for s in range(len(offsets) - 1):
        a, b = int(offsets[s]), int(offsets[s + 1])
        if b == a:
            continue
        eps = emissions(probs[a:b], stride)
        g = gaps(start[a:b], stride)
        gam = forward_backward(eps, g, C, stride, L)
        path, best[s] = viterbi(eps, g, C, stride, L)
        if path_override is not None:
            path = np.asarray(path_override[a:b], np.int64)
        post[a:b], state[a:b] = gam, path
        for rs, re, k, m, pm, sc in regions(path, gam, probs[a:b], start[a:b], length[a:b]):
            for key, v in zip(("contig", "start", "end", "class", "windows", "posterior", "scores"), (s, rs, re, k, m, pm, sc)):
                rows[key].append(v)
    return {"posterior": post, "state": state, "best": best,
            "region_contig": np.array(rows["contig"], np.int32), "region_start": np.array(rows["start"], np.int64),
            "region_end": np.array(rows["end"], np.int64), "region_class": np.array(rows["class"], np.int32),
            "region_windows": np.array(rows["windows"], np.int32),
            "region_posterior": np.array(rows["posterior"], np.float32),
            "region_scores": np.array(rows["scores"], np.float32).reshape(-1, C)}
