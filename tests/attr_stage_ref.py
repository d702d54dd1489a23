"""
Per-stage fp64 references of the attribution backward pass (csrc/attr.cuh, the kConvBwd epilogue of csrc/conv_t.cuh,
attribute_step in csrc/api.cu), for the stage-precision tests.  Like tests/stage_ref.py, every function takes the input of ONE
stage -- in the GPU tests that kernel's own input, fetched with gnm_debug_fetch -- and returns a stage_ref.Ref (the fp64 value and
the two scales of the stage's contraction), so R.metrics and R.position_regions apply unchanged.

    head_backward   probabilities (fp32), h1, h2                 -> g_out [n, 256]          (unscaled)
    igloo_backward  g_out half, logits, q, routing (+ y3 mask)   -> g_y [n, 5997, 128]      (IGLOO#1: g_z3 = g_y3 * lrelu'(y3))
    conv_backward   gradient rows, W, mask (+ s_w g_y1)          -> sum_j g[s+5-j] W[j]^T * lrelu'(y) at every position s
    layer1          s_w g_z1, tokens, s_w                        -> attr [n, 5997]

The scales chain the absolute values (resp. squares) of every contraction of a stage, so that an error inside any of its sums
is measured against the size of that sum's terms.  `compose` runs the whole pass from fp64 forward intermediates through these
functions; tests/test_attr_stage_recipes_cpu.py shows that it is attr_ref.decomposed to fp64 rounding.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch

import stage_ref as R
from oracle import igloo_model as M

D = torch.float64
L_TOK, N_POOL, POOL = R.L_TOK, R.N_POOL, R.POOL
LRELU = 0.1


def _t(x, dt=D) -> torch.Tensor:
    return torch.as_tensor(np.asarray(x), dtype=dt)


def _bn_scale(w, p, dt=D):
    return _t(w[p + "g"], dt) / torch.sqrt(_t(w[p + "v"], dt) + M.BN_EPS)


def _lrelu_d(mask, dt=D):
    """lrelu' from a mask y > 0 (0.1 in the arithmetic's own precision: torch.where with a Python scalar rounds it to float32)"""
    m = torch.as_tensor(np.asarray(mask))
    return torch.where(m, torch.ones((), dtype=dt), torch.full((), LRELU, dtype=dt))


def head_gradient(probs, target: int, dt=D) -> torch.Tensor:
    """g_logits = e_c - p from the probabilities: -p_i off the target, the sum of the other two on it."""
    p = _t(probs, dt)
    g = -p
    o = [i for i in range(3) if i != target]
    g[:, target] = p[:, o[0]] + p[:, o[1]]
    return g


def head_backward(probs, h1, h2, w, target: int, dt=D) -> R.Ref:
    """g_out = d log p_c / d h0 from the step's probabilities and post-ReLU h1, h2 (attr_head_backward_kernel).  dt: the
    arithmetic (float32 for the CPU emulation of the kernel; the scales are then meaningless)."""
    gl = head_gradient(probs, target, dt)
    h1, h2 = _t(h1, dt), _t(h2, dt)
    d2w, d1w, d0w = _t(w["d2w"], dt), _t(w["d1w"], dt), _t(w["d0w"], dt)
    b1, b0 = _bn_scale(w, "bn1", dt), _bn_scale(w, "bn0", dt)
    m2, m1 = (h2 > 0).to(dt), (h1 > 0).to(dt)
    a1 = (gl @ d2w.T) * m2 * b1
    a0 = (a1 @ d1w.T) * m1 * b0
    val = a0 @ d0w.T
    s1 = (gl.abs() @ d2w.abs().T) * m2 * b1.abs()
    s0 = (s1 @ d1w.abs().T) * m1 * b0.abs()
    q1 = ((gl * gl) @ (d2w * d2w).T) * m2 * b1 * b1
    q0 = (q1 @ (d1w * d1w).T) * m1 * b0 * b0
    return R.Ref(val, s0 @ d0w.abs().T, torch.sqrt(q0 @ (d0w * d0w).T))


def _patch_entries(w, s, dt=D):
    """(position, patch, folded weight row) of every patch entry, sorted by position (the gather's slot order)."""
    P = np.asarray(w[f"ig{s}_random_patches"]).reshape(-1).astype(np.int64)
    Wf = (_t(w[f"ig{s}_w_mult"], dt)[0] * _t(w[f"ig{s}_w_summer"], dt).reshape(1, 4, 128)).reshape(-1, 128)
    order = np.argsort(P, kind="stable")
    return torch.as_tensor(P[order]), torch.as_tensor(order // 4), Wf[torch.as_tensor(order)]


def igloo_backward(g_out, logits, q, route, w, s: int, y_mask=None, dt=D, mutant: str = "") -> R.Ref:
    """g_y of IGLOO kernel s (attr_igloo_prep_kernel, the g_mpi sgemm, attr_igloo_backward_kernel) from this kernel's 128
    columns of g_out [n, 128], its logits [n, >= 749], its q [n, 749, 128] and routing [n, 749, 128] (rows 0..7):
        alpha = softmax(logits), g_alpha = q g_out, g_logit = alpha (g_alpha - <alpha, g_alpha>), g_mpi = w_qk g_logit,
        g_y[t] = sum over the (p, c) routed to t of alpha[p] g_out[c] w_v[:, c] + sum over the patch entries on t of g_mpi Wf.
    y_mask (IGLOO#1: y3 > 0, [n, 5997, 128]) multiplies by lrelu'(y3), giving g_z3.  dt as for head_backward; mutant (CPU
    emulation only): "no patch path", or "first routed channel" (the value path keeps one channel per row)."""
    g_o, q = _t(g_out, dt), _t(q, dt)
    al = torch.softmax(_t(logits, dt)[:, :N_POOL], dim=-1)
    wv = _t(w[f"ig{s}_w_v"], dt).reshape(128, 128)
    wqk = _t(w[f"ig{s}_w_qk"], dt)                                           # [2100, 749]
    g_al = torch.einsum("bpc,bc->bp", q, g_o)
    g_al_abs = torch.einsum("bpc,bc->bp", q.abs(), g_o.abs())
    g_al_sq = torch.einsum("bpc,bc->bp", q * q, g_o * g_o)
    dot = (al * g_al).sum(1, keepdim=True)
    g_logit = al * (g_al - dot)
    gl_abs = al * (g_al_abs + (al * g_al_abs).sum(1, keepdim=True))
    gl_sq = al * al * (g_al_sq + (al * al * g_al_sq).sum(1, keepdim=True))
    g_mpi, gm_abs, gm_sq = g_logit @ wqk.T, gl_abs @ wqk.abs().T, gl_sq @ (wqk * wqk).T
    n = g_o.shape[0]
    g_q = al[:, :, None] * g_o[:, None, :]                                   # [n, 749, 128]
    rt = torch.as_tensor(np.asarray(route).astype(np.int64))
    val, sab, ssq = (torch.zeros(n, L_TOK, 128, dtype=dt) for _ in range(3))
    for r in range(POOL):                                                    # value path, row r of every pool
        sel = (rt == r).to(dt)
        if mutant == "first routed channel":
            sel = sel * (torch.cumsum(sel, dim=2) == 1).to(dt)
        gq = g_q * sel
        val[:, r: N_POOL * POOL: POOL] += gq @ wv.T
        sab[:, r: N_POOL * POOL: POOL] += gq.abs() @ wv.abs().T
        ssq[:, r: N_POOL * POOL: POOL] += (gq * gq) @ (wv * wv).T
    pos, patch, ent = _patch_entries(w, s, dt)                               # patch path
    if mutant == "no patch path":
        ent = ent * 0
    val.index_add_(1, pos, g_mpi[:, patch, None] * ent[None])
    sab.index_add_(1, pos, gm_abs[:, patch, None] * ent.abs()[None])
    ssq.index_add_(1, pos, gm_sq[:, patch, None] * (ent * ent)[None])
    if y_mask is not None:
        d = _lrelu_d(y_mask, dt)
        val, sab, ssq = val * d, sab * d, ssq * d * d
    return R.Ref(val, sab, torch.sqrt(ssq))


def conv_backward(g, W, mask, add=None, add_scale=None, out_scale=None) -> R.Ref:
    """The backward of a causal Conv1D + LeakyReLU (conv_t_attr_kernel<kConvBwd>), in natural position order:
        out[s] = (out_scale * sum_j g[s+5-j] W[j]^T + add_scale * add[s]) * lrelu'(y[s])
    with g [n, 5997, 128] the gradient rows the conv reads, W [6, in, out] the forward's kernel, mask = y > 0 [n, 5997, 128],
    add (conv2: IGLOO#0's g_y1) times the per-window add_scale [n] (s_w), out_scale [n] (1 / s2 for conv2) per window."""
    g = _t(g)
    WT = _t(W).transpose(1, 2)
    conv = lambda x, k: R._causal(x.flip(1), k).flip(1)                     # noqa: E731
    val, sab, ssq = conv(g, WT), conv(g.abs(), WT.abs()), conv(g * g, WT * WT)
    if out_scale is not None:
        o = _t(out_scale).reshape(-1, 1, 1)
        val, sab, ssq = val * o, sab * o.abs(), ssq * o * o
    if add is not None:
        a = _t(add) * _t(add_scale).reshape(-1, 1, 1)
        val, sab, ssq = val + a, sab + a.abs(), ssq + a * a
    d = _lrelu_d(mask)
    return R.Ref(val * d, sab * d, torch.sqrt(ssq) * d)


def layer1(g_z1, tokens, w, s_w, dt=D, mutant: str = "") -> R.Ref:
    """attr[t] = (1 / s_w) sum_{u=t}^{min(t+5, 5996)} <g_z1[u], W1[t-u+5, tok[t], :]> (layer1_attr_kernel), g_z1 = s_w times
    the gradient at layer 1's pre-activation; tokens 0..256.  dt as for head_backward; mutant (CPU emulation only):
    "g_z1 in fp16" (the rows read at half precision)."""
    g = _t(g_z1, dt)
    if mutant == "g_z1 in fp16":
        g = g.half().to(dt)
    W1 = _t(w["c1w"], dt)                                                   # [6, 257, 128]
    tok = torch.as_tensor(np.asarray(tokens).astype(np.int64))
    n = g.shape[0]
    val, sab, ssq = (torch.zeros(n, L_TOK, dtype=dt) for _ in range(3))
    for j in range(6):                                                      # u = t + 5 - j
        sh = 5 - j
        wr = W1[j][tok[:, : L_TOK - sh]]                                     # [n, L - sh, 128]
        gu = g[:, sh:]
        val[:, : L_TOK - sh] += (gu * wr).sum(-1)
        sab[:, : L_TOK - sh] += (gu.abs() * wr.abs()).sum(-1)
        ssq[:, : L_TOK - sh] += (gu * gu * wr * wr).sum(-1)
    inv = 1.0 / _t(s_w, dt).reshape(-1, 1)
    return R.Ref(val * inv, sab * inv.abs(), torch.sqrt(ssq) * inv.abs())


def pow2_scale(gmax, top: int) -> np.ndarray:
    """attr_scale_of: the power of two s with max |g| s in [2^(top-1), 2^top) per window (1 for an all-zero gradient);
    s_w is top = -1 ([0.25, 0.5)), s2 top = 1 ([1, 2))."""
    m = np.asarray(gmax, dtype=np.float64)
    e = np.frexp(m)[1]
    return np.where(m > 0, np.ldexp(1.0, np.clip(top - e, -120, 120)), 1.0)


def compose(tokens, w, target: int, routes: Optional[Sequence] = None) -> np.ndarray:
    """The whole backward pass from the fp64 forward, stage by stage through the functions above (s_w and s2 as the kernels
    pick them); attr_ref.decomposed to fp64 rounding."""
    import attr_ref as A
    tokens = np.asarray(tokens).astype(np.int64)
    with torch.no_grad():
        _, it = M.forward(tokens, w, D, return_intermediates=True)
    if routes is None:
        routes = [r for r, _, _ in A.routing(tokens, w)]
    h1 = R.dense_bn_relu(it["h0"], w, 0).value
    h2 = R.dense_bn_relu(h1, w, 1).value
    probs = R.head_softmax(h2, w).value
    g_out = head_backward(probs, h1, h2, w, target).value
    y1, y2, y3 = it["y1"], it["y2"], it["y3"]
    lg = [it[f"ig{s}"]["mpi"] @ _t(w[f"ig{s}_w_qk"]) for s in (0, 1)]
    qs = [R.wv_pool(y, w[f"ig{s}_w_v"]).value for s, y in ((0, y1), (1, y3))]
    g_z3 = igloo_backward(g_out[:, 128:], lg[1], qs[1], routes[1], w, 1, y3 > 0).value
    s_w = torch.as_tensor(pow2_scale(g_z3.abs().amax(dim=(1, 2)).numpy(), -1))
    g_z2 = conv_backward(g_z3 * s_w.reshape(-1, 1, 1), w["c3w"], y2 > 0).value              # s_w g_z2
    s2 = torch.as_tensor(pow2_scale(g_z2.abs().amax(dim=(1, 2)).numpy(), 1))
    g_y1 = igloo_backward(g_out[:, :128], lg[0], qs[0], routes[0], w, 0).value
    g_z1 = conv_backward(g_z2 * s2.reshape(-1, 1, 1), w["c2w"], y1 > 0, g_y1, s_w, 1.0 / s2).value
    return layer1(g_z1, tokens, w, s_w).value.numpy()
