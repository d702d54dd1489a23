"""
fp64 reference of the attributions (include/gnm.h, DESIGN.md "Attributions"): torch.autograd through the unchanged oracle's
pieces (oracle/igloo_model.py), and a NumPy restatement of the backward pass as the kernels decompose it (csrc/attr.cuh).

    attr[t] = d log p_c / d x[t, tok[t]],   x = the one-hot input of the first Conv1D

Max-pool routing: by default F.max_pool1d's, which sends the gradient to the first row of a tie (the rule the kernels follow);
`routes` ([2] arrays [B, 749, 128] of rows 0..7, e.g. the GPU's "route0" / "route1") makes the gradient follow a given routing,
and `masks` (the signs y > 0 of y1, y2, y3) the LeakyReLU branches of a given forward: both derivatives are discontinuous, and
an fp32 forward lands on the other side of a near-tie or of z ~ 0 at a few places per window.  log p_c is differentiated
in a form that keeps its relative precision when p_c saturates (log_p_target), so windows classified confidently as the target
have a reference too.  softmax_fp32 / head_gradient_fp32 restate the float32 head: the forward's softmax and the backward's
first step.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from oracle import igloo_model as M

L_TOK, N_POOL, POOL = M.L_TOK, M.N_POOL, M.POOL


def _igloo(y, w, s, dtype, route=None):
    """IGLOO1D_kernel.call (igloo.py:190-217) with the max-pool either as written (F.max_pool1d's own choice of row, the first
    on ties) or along `route`.  Both take q through the same gather from rows of the same layout, so an explicit route equal
    to F.max_pool1d's gives the same bits on any BLAS (a transposed q would send einsum and its backward through other
    matmul kernels, whose summation order may differ)."""
    P = torch.as_tensor(np.asarray(w[f"ig{s}_random_patches"]).reshape(M.N_PATCH, 4), dtype=torch.long)
    Wf = M._t(w, f"ig{s}_w_mult", dtype)[0] * M._t(w, f"ig{s}_w_summer", dtype).reshape(1, 4, 128)
    mpi = (y[:, P] * Wf).sum(dim=(2, 3)) + M._t(w, f"ig{s}_w_bias", dtype)
    y_proj = y @ M._t(w, f"ig{s}_w_v", dtype)[0]
    if route is None:
        with torch.no_grad():
            _, idx = F.max_pool1d(y_proj.transpose(1, 2), POOL, return_indices=True)     # [B, 128, 749] positions
        route = (idx - POOL * torch.arange(N_POOL)).transpose(1, 2)                    # [B, 749, 128] rows 0..7
    yp = y_proj[:, : N_POOL * POOL].reshape(y.shape[0], N_POOL, POOL, -1)
    q = yp.gather(2, torch.as_tensor(np.asarray(route), dtype=torch.long)[:, :, None, :]).squeeze(2)
    alpha = torch.softmax(mpi @ M._t(w, f"ig{s}_w_qk", dtype), dim=-1)
    return torch.einsum("bg,bgc->bc", alpha, q)


def one_hot(tokens, dtype=torch.float64):
    tok = torch.as_tensor(np.asarray(tokens).astype(np.int64))
    return F.one_hot(M.vocab_tokens(tok), 258)[..., :257].to(dtype)


def _act(z, mask):
    """LeakyReLU; with `mask` (bool [B, L, 128], "y > 0" of some forward), its branch is taken from the mask instead of the
    sign of z -- the value changes only where the signs disagree, i.e. for |z| at rounding level, but the gradient follows
    the given forward's branch (the derivative jumps from 1 to 0.1 at z = 0, like the max-pool's at a tie)."""
    if mask is None:
        return M._lrelu(z)
    return torch.where(torch.as_tensor(np.asarray(mask)), z, z * M.LRELU)


def log_probs_onehot(x, w, routes: Optional[Sequence] = None, dtype=torch.float64, masks: Optional[Sequence] = None):
    """log softmax of the model on one-hot (or relaxed) input x [B, 5997, 257]; masks = [y1 > 0, y2 > 0, y3 > 0] optional."""
    return torch.log_softmax(logits_onehot(x, w, routes, dtype, masks), dim=-1)


def log_p_target(logits, target: int):
    """log p_c from the logits [B, 3], with a gradient that keeps its relative precision when p_c saturates.  log_softmax's
    backward is e_c - p, whose target component 1 - p_c cancels once p_c is near 1 (in fp64 too: p_c == 1.0 from a log-odds
    margin of about 37).  Where c is the argmax this uses log p_c = -log1p(sum_{i != c} exp(l_i - l_c)), whose derivatives are
    sum_{i != c} p_i and -p_i: sums of positive terms.  Elsewhere p_c <= 1/2 and log_softmax loses nothing."""
    lc = logits[:, target: target + 1]
    d = torch.cat([logits[:, :target], logits[:, target + 1:]], dim=1) - lc
    top = d.max(dim=1).values <= 0
    sat = -torch.log1p(torch.exp(d.clamp(max=0)).sum(dim=1))      # the clamp only bites on rows where it is not selected
    return torch.where(top, sat, torch.log_softmax(logits, dim=-1)[:, target])


def logits_onehot(x, w, routes: Optional[Sequence] = None, dtype=torch.float64, masks: Optional[Sequence] = None):
    """the model's three logits on one-hot (or relaxed) input x [B, 5997, 257] (see log_probs_onehot)"""
    ms = masks if masks is not None else (None, None, None)
    xc = F.pad(x.transpose(1, 2), (5, 0))
    k = M._t(w, "c1w", dtype).permute(2, 1, 0).contiguous()
    y1 = _act(F.conv1d(xc, k, M._t(w, "c1b", dtype)).transpose(1, 2), ms[0])
    o0 = _igloo(y1, w, 0, dtype, None if routes is None else routes[0])

    def conv(y, s, mask):
        kk = torch.as_tensor(w[f"c{s}w"], dtype=dtype).permute(2, 1, 0).contiguous()
        z = F.conv1d(F.pad(y.transpose(1, 2), (5, 0)), kk, torch.as_tensor(w[f"c{s}b"], dtype=dtype)).transpose(1, 2)
        return _act(z, mask)

    if masks is None:
        y2 = M.causal_conv(y1, w["c2w"], w["c2b"], dtype)
        y3 = M.causal_conv(y2, w["c3w"], w["c3b"], dtype)
    else:
        y2 = conv(y1, 2, ms[1])
        y3 = conv(y2, 3, ms[2])
    o1 = _igloo(y3, w, 1, dtype, None if routes is None else routes[1])
    return M.head(torch.cat([o0, o1], dim=1), w, dtype, return_logits=True)


def attribution(tokens, w, target: int, routes: Optional[Sequence] = None, dtype=torch.float64,
                masks: Optional[Sequence] = None, logits_at: Optional[np.ndarray] = None) -> np.ndarray:
    """[B, 5997] tokens (0..256) -> [B, 5997] attributions by autograd; `routes` / `masks` make the max-pools / LeakyReLUs
    follow a given forward (e.g. the GPU's: "route0/1", and the signs of y1, y2, y3).  `logits_at` ([B, 3], e.g. the GPU
    forward's) is where log p_c and its gradient are evaluated; the logits' derivatives stay this model's.  For a window
    classified confidently as the target the attributions scale as e^-mu, so a forward's logit-margin error d moves all of
    them by the relative d: an fp32 forward with logits of magnitude ~176 (golden row 16) has d ~ 1e-4."""
    x = one_hot(tokens, dtype).requires_grad_(True)
    lg = logits_onehot(x, w, routes, dtype, masks)
    if logits_at is not None:
        lg = lg - lg.detach() + torch.as_tensor(np.asarray(logits_at), dtype=dtype)
    lp = log_p_target(lg, target).sum()
    (g,) = torch.autograd.grad(lp, x)
    tok = torch.as_tensor(np.asarray(tokens).astype(np.int64))
    return g.gather(2, tok[..., None]).squeeze(2).numpy()


def routing(tokens, w) -> list:
    """fp64 routing of both IGLOO kernels (first row on ties) and the gap between the two largest rows of each pool."""
    with torch.no_grad():
        _, it = M.forward(tokens, w, torch.float64, return_intermediates=True)
    out = []
    for s, y in ((0, it["y1"]), (1, it["y3"])):
        z = (y @ M._t(w, f"ig{s}_w_v", torch.float64)[0])[:, : N_POOL * POOL].reshape(y.shape[0], N_POOL, POOL, -1).numpy()
        r = np.argmax(z, axis=2)                                     # numpy: first maximum
        srt = np.sort(z, axis=2)
        out.append((r.astype(np.uint8), srt[:, :, -1, :] - srt[:, :, -2, :], np.abs(srt[:, :, -1, :])))
    return out


# ----------------------------------------------------------------------------- the kernels' decomposition, in NumPy fp64
def _lrelu_d(y):
    return np.where(y > 0, 1.0, M.LRELU)


def softmax_fp32(logits32) -> np.ndarray:
    """[n, 3] float32 logits -> float32 probabilities as dense3_softmax_kernel (csrc/dense.cuh) computes them: the maximum,
    exp(a_i - m), one reciprocal of (e0 + e1) + e2, three products."""
    a = np.asarray(logits32, dtype=np.float32)
    e = np.exp(a - a.max(axis=1, keepdims=True))
    inv = np.float32(1) / ((e[:, 0] + e[:, 1]) + e[:, 2])
    return e * inv[:, None]


def head_gradient_from_probs32(p32, target: int) -> np.ndarray:
    """g_logits = e_c - p as attr_head_backward_kernel computes it from the forward's float32 probabilities: -p_i off the
    target, and the target's component as the sum of the other two probabilities in ascending i, never as 1 - p_c (which
    cancels in fp32 once p_c is near 1 and is exactly 0 once p_c rounds to 1.0f)."""
    p = np.asarray(p32, dtype=np.float32)
    g = -p
    o = [i for i in range(3) if i != target]
    g[:, target] = p[:, o[0]] + p[:, o[1]]
    return g


def head_gradient_fp32(logits32, target: int) -> np.ndarray:
    """the head's g_logits from float32 logits: the forward's softmax, then the kernel's formula (both in float32)"""
    return head_gradient_from_probs32(softmax_fp32(logits32), target)


def head_gradient_fp64(logits, target: int) -> np.ndarray:
    """e_c - softmax(logits) in fp64 with full relative precision in every component (no 1 - p_c)"""
    a = np.asarray(logits, dtype=np.float64)
    e = np.exp(a - a.max(axis=1, keepdims=True))
    p = e / e.sum(axis=1, keepdims=True)
    g = -p
    g[:, target] = np.delete(p, target, axis=1).sum(axis=1)
    return g


def decomposed(tokens, w, target: int, routes: Optional[Sequence] = None,
               g_logits: Optional[np.ndarray] = None) -> np.ndarray:
    """The backward pass as csrc/attr.cuh computes it, one window at a time, in fp64: head backward, the attention part,
    the sparse value path (per row t: the channels routed to t), the patch path through the position-sorted entries, the
    per-window power of two s_w, conv backward as a causal conv over time-reversed rows against W[j]^T with the mirrored
    lrelu' mask, and the layer-1 formula.  `g_logits` ([B, 3]) replaces the head's gradient e_c - p (by default the fp64
    head_gradient_fp64), e.g. with one computed from float32 probabilities."""
    f64 = torch.float64
    tokens = np.asarray(tokens).astype(np.int64)
    with torch.no_grad():
        _, it = M.forward(tokens, w, f64, return_intermediates=True)
    W = {k: np.asarray(v, dtype=np.float64) for k, v in w.items()}
    if routes is None:
        routes = [r for r, _, _ in routing(tokens, w)]
    y1, y2, y3, h0 = (it[k].numpy() for k in ("y1", "y2", "y3", "h0"))
    bn = {}
    for p in ("bn0", "bn1"):
        bn[p] = W[p + "g"] / np.sqrt(W[p + "v"] + M.BN_EPS)
    out = np.zeros(tokens.shape, dtype=np.float64)
    for b in range(tokens.shape[0]):
        # ---- head
        a0 = h0[b] @ W["d0w"] + W["d0b"]
        h1 = np.maximum(bn["bn0"] * (a0 - W["bn0m"]) + W["bn0b"], 0)
        a1 = h1 @ W["d1w"] + W["d1b"]
        h2 = np.maximum(bn["bn1"] * (a1 - W["bn1m"]) + W["bn1b"], 0)
        lg = h2 @ W["d2w"] + W["d2b"]
        g_lg = head_gradient_fp64(lg[None], target)[0] if g_logits is None else np.asarray(g_logits[b], dtype=np.float64)
        g_a1 = np.where(h2 > 0, W["d2w"] @ g_lg, 0) * bn["bn1"]
        g_a0 = np.where(h1 > 0, W["d1w"] @ g_a1, 0) * bn["bn0"]
        g_h0 = W["d0w"] @ g_a0
        g_y = []
        for s, y in ((0, y1[b]), (1, y3[b])):
            g_o = g_h0[128 * s: 128 * (s + 1)]
            wv = W[f"ig{s}_w_v"][0]
            z = (y @ wv)[: N_POOL * POOL].reshape(N_POOL, POOL, -1)
            q = np.take_along_axis(z, routes[s][b][:, None, :].astype(np.int64), axis=1)[:, 0, :]
            Pt = W[f"ig{s}_random_patches"].reshape(M.N_PATCH, 4).astype(np.int64)
            Wf = W[f"ig{s}_w_mult"][0] * W[f"ig{s}_w_summer"].reshape(1, 4, 128)
            mpi = (y[Pt] * Wf).sum(axis=(1, 2)) + W[f"ig{s}_w_bias"][0]
            lo = mpi @ W[f"ig{s}_w_qk"]
            al = np.exp(lo - lo.max()); al /= al.sum()
            g_al = q @ g_o
            g_logit = al * (g_al - al @ g_al)
            g_mpi = W[f"ig{s}_w_qk"] @ g_logit
            gy = np.zeros((L_TOK, 128))
            g_q = al[:, None] * g_o[None, :]
            for r in range(POOL):                                       # value path, row by row of the pools
                sel = routes[s][b] == r                                 # [749, 128]: channels routed to row 8 p + r
                gy[r: N_POOL * POOL: POOL] += (g_q * sel) @ wv.T
            order = np.argsort(Pt.reshape(-1), kind="stable")           # patch path through the position-sorted entries
            ent_pos = Pt.reshape(-1)[order]
            ent_w = Wf.reshape(-1, 128)[order]
            np.add.at(gy, ent_pos, g_mpi[order // 4][:, None] * ent_w)
            g_y.append(gy)
        g_z3 = g_y[1] * _lrelu_d(y3[b])
        m = np.abs(g_z3).max()
        s_w = 2.0 ** (-np.frexp(m)[1] - 1) if m > 0 else 1.0          # max |g_z3| s_w in [0.25, 0.5)

        def conv_bwd(gz_rev, Wk):                                       # causal conv of the reversed rows against W[j]^T
            pad = np.concatenate([np.zeros((5, 128)), gz_rev])
            return sum(pad[j: j + L_TOK] @ Wk[j].T for j in range(6))

        g_y2 = conv_bwd((s_w * g_z3)[::-1], W["c3w"])[::-1]
        g_z2 = g_y2 * _lrelu_d(y2[b])
        g_y1 = conv_bwd(g_z2[::-1], W["c2w"])[::-1] + s_w * g_y[0]
        g_z1 = g_y1 * _lrelu_d(y1[b])
        W1 = W["c1w"]                                                   # [6, 257, 128]
        tk = np.where(tokens[b] > 256, -1, tokens[b])
        for t in range(L_TOK):
            if tk[t] < 0:
                continue
            u = np.arange(t, min(t + 5, L_TOK - 1) + 1)
            out[b, t] = np.einsum("uc,uc->", g_z1[u], W1[t - u + 5, tk[t]]) / s_w
    return out
