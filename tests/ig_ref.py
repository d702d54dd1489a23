"""
fp64 reference of integrated gradients (include/gnm.h, DESIGN.md "Integrated gradients"), built on attr_ref.logits_onehot at
relaxed one-hot inputs on the straight line from a baseline x' to the window x:

    x_k = x' + alpha_k (x - x'),  alpha_k = (k + 1/2) / m          (midpoint rule, k = 0..m-1)
    zero baseline: x' = 0                  row_k[t] = g_k[t, tok[t]]
    N baseline:    x' = e_0 at every t     row_k[t] = g_k[t, tok[t]] - g_k[t, 0]   (0 where tok[t] = 0)
    IG[t] = (1/m) sum_k row_k[t],          g_k = d log p_c / d x at x_k

Each row's three logit gradients are taken once (logit_jacobian); the gradient of log p_c is their combination with the head's
g_logits = e_c - p at the row's logits (attr_ref.head_gradient_fp64, no 1 - p_c).  So one Jacobian serves every target, any
given logits (`logits_at`, e.g. the GPU forward's, from its h2) and every head-sharpened weight set (d2w, d2b times k scales
the logits by k, and the gradient of log p_c by k at the sharpened probabilities).  `routes` / `masks` make each row follow a
given forward's max-pool routing and LeakyReLU branches, as in attr_ref.attribution, and `head_masks` ([h1 > 0, h2 > 0])
its head's ReLU branches: at interpolated inputs a head unit sits at ~0 now and then, where an fp32 forward and fp64 can take
different sides.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

import attr_ref as A
from oracle import igloo_model as M

BASELINES = ("zero", "N")


def alphas(m: int) -> np.ndarray:
    return (np.arange(m) + 0.5) / m


def interp_onehot(tokens, alpha, baseline: str, dtype=torch.float64):
    """[R, 5997] tokens, alpha [R] -> x' + alpha (x - x') [R, 5997, 257]"""
    x = A.one_hot(tokens, dtype)
    a = torch.as_tensor(np.asarray(alpha, dtype=np.float64), dtype=dtype).reshape(-1, 1, 1)
    if baseline == "zero":
        return a * x
    base = torch.zeros_like(x)
    base[..., 0] = 1
    return base + a * (x - base)


def _select(g, tokens, baseline: str) -> np.ndarray:
    """g [R, 5997, 257] -> the IG row value per position: g[t, tok] (zero) or g[t, tok] - g[t, 0] (N, 0 at token 0)"""
    tok = torch.as_tensor(np.asarray(tokens).astype(np.int64))
    v = g.gather(2, tok[..., None]).squeeze(2)
    if baseline == "N":
        v = torch.where(tok == 0, torch.zeros_like(v), v - g[..., 0])
    return v.numpy()


def _head(h0, w, head_masks):
    """oracle_model.head's logits with the two ReLUs' branches taken from head_masks ([h1 > 0, h2 > 0])"""
    dt = torch.float64

    def bn(x, p):
        return M._t(w, p + "g", dt) * (x - M._t(w, p + "m", dt)) / torch.sqrt(M._t(w, p + "v", dt) + M.BN_EPS) + M._t(w, p + "b", dt)

    def relu(z, m):
        return torch.where(torch.as_tensor(np.asarray(m)), z, torch.zeros_like(z))
    h1 = relu(bn(h0 @ M._t(w, "d0w", dt) + M._t(w, "d0b", dt), "bn0"), head_masks[0])
    h2 = relu(bn(h1 @ M._t(w, "d1w", dt) + M._t(w, "d1b", dt), "bn1"), head_masks[1])
    return h2 @ M._t(w, "d2w", dt) + M._t(w, "d2b", dt)


def logits_onehot(x, w, routes=None, masks=None, head_masks=None):
    """attr_ref.logits_onehot, and with head_masks the head's ReLU branches of a given forward too"""
    if head_masks is None:
        return A.logits_onehot(x, w, routes, torch.float64, masks)
    ms = masks if masks is not None else (None, None, None)
    xc = F.pad(x.transpose(1, 2), (5, 0))
    k = M._t(w, "c1w", torch.float64).permute(2, 1, 0).contiguous()
    y1 = A._act(F.conv1d(xc, k, M._t(w, "c1b", torch.float64)).transpose(1, 2), ms[0])
    o0 = A._igloo(y1, w, 0, torch.float64, None if routes is None else routes[0])

    def conv(y, s, mask):
        kk = torch.as_tensor(w[f"c{s}w"], dtype=torch.float64).permute(2, 1, 0).contiguous()
        z = F.conv1d(F.pad(y.transpose(1, 2), (5, 0)), kk, torch.as_tensor(w[f"c{s}b"], dtype=torch.float64)).transpose(1, 2)
        return A._act(z, mask)
    y3 = conv(conv(y1, 2, ms[1]), 3, ms[2])
    o1 = A._igloo(y3, w, 1, torch.float64, None if routes is None else routes[1])
    return _head(torch.cat([o0, o1], dim=1), w, head_masks)


def logit_jacobian(tokens, w, alpha, baseline: str, routes: Optional[Sequence] = None, masks: Optional[Sequence] = None,
                   batch: int = 8, head_masks: Optional[Sequence] = None):
    """rows tokens [R, 5997] at alpha [R] -> (fp64 logits [R, 3], J [R, 3, 5997]: the IG row value of d logit_i / d x)"""
    tokens = np.asarray(tokens)
    alpha = np.broadcast_to(np.asarray(alpha, dtype=np.float64), (len(tokens),))
    lg_out, j_out = [], []
    for s in range(0, len(tokens), batch):
        sl = slice(s, s + batch)
        x = interp_onehot(tokens[sl], alpha[sl], baseline).requires_grad_(True)
        lg = logits_onehot(x, w, None if routes is None else [r[sl] for r in routes],
                           None if masks is None else [m[sl] for m in masks],
                           None if head_masks is None else [m[sl] for m in head_masks])
        J = []
        for i in range(3):
            (g,) = torch.autograd.grad(lg[:, i].sum(), x, retain_graph=i < 2)
            J.append(_select(g, tokens[sl], baseline))
        lg_out.append(lg.detach().numpy())
        j_out.append(np.stack(J, axis=1))
    return np.concatenate(lg_out), np.concatenate(j_out)


def rows_from_jacobian(logits, J, target: int, scale: float = 1.0) -> np.ndarray:
    """[R, 5997] gradients of log p_c (IG row values) at `scale` x the given logits, for weights whose head is scaled by `scale`"""
    G = A.head_gradient_fp64(scale * np.asarray(logits, dtype=np.float64), target) * scale
    return np.einsum("ri,rit->rt", G, J)


def log_p(logits, target: int, scale: float = 1.0) -> np.ndarray:
    """log p_c without cancellation (attr_ref.log_p_target) at `scale` x logits [R, 3]"""
    return A.log_p_target(torch.as_tensor(scale * np.asarray(logits, dtype=np.float64)), target).numpy()


def endpoint_logits(tokens, w, baseline: str) -> tuple:
    """fp64 logits at x (alpha = 1) [B, 3] and at the baseline x' (alpha = 0) [3]"""
    tokens = np.asarray(tokens)
    with torch.no_grad():
        lx = A.logits_onehot(interp_onehot(tokens, np.ones(len(tokens)), baseline), w).numpy()
        lb = A.logits_onehot(interp_onehot(tokens[:1], np.zeros(1), baseline), w).numpy()[0]
    return lx, lb


def integrated_gradients(tokens, w, target: int, steps: int, baseline: str, routes: Optional[Sequence] = None,
                         masks: Optional[Sequence] = None, logits_at: Optional[np.ndarray] = None):
    """[B, 5997] tokens -> (IG [B, 5997], rows [B, m, 5997]) at the midpoint nodes.  routes / masks / logits_at, when given,
    are per ROW (row w m + k = window w at alpha_k), e.g. the GPU's debug buffers after an IG call."""
    tokens = np.asarray(tokens)
    B, m = len(tokens), int(steps)
    rt = np.repeat(tokens, m, axis=0)
    al = np.tile(alphas(m), B)
    lg, J = logit_jacobian(rt, w, al, baseline, routes, masks)
    rows = rows_from_jacobian(lg if logits_at is None else logits_at, J, target).reshape(B, m, -1)
    return rows.mean(axis=1), rows


def layer1_preact(tokens, w, alpha, baseline: str) -> np.ndarray:
    """The interpolated layer-1 pre-activation as the kernel states it (encode.cuh), in fp64:
    b1 + alpha S_tok + (1 - alpha) S_base, S_tok[t] = sum_{j: t-5+j >= 0} W1[j, tok[t-5+j]], S_base = 0 (zero) or
    sum_{j: t-5+j >= 0} W1[j, 0] (N).  tokens [B, 5997], alpha [B] -> [B, 5997, 128]"""
    W1 = np.asarray(w["c1w"], dtype=np.float64)
    b1 = np.asarray(w["c1b"], dtype=np.float64)
    tokens = np.asarray(tokens).astype(np.int64)
    B, L = tokens.shape
    s_tok = np.zeros((B, L, W1.shape[2]))
    s_base = np.zeros((L, W1.shape[2]))
    for j in range(6):
        sh = 5 - j                                                   # tap j reads token t - sh
        s_tok[:, sh:] += W1[j][tokens[:, : L - sh]]
        s_base[sh:] += W1[j, 0]
    a = np.asarray(alpha, dtype=np.float64).reshape(-1, 1, 1)
    pre = b1 + a * s_tok
    if baseline == "N":
        pre = pre + (1 - a) * s_base
    return pre


def conv1_preact(x, w) -> np.ndarray:
    """the oracle's Conv1D #1 (causal padding) on a one-hot or relaxed input x [B, 5997, 257], fp64, before the LeakyReLU"""
    xc = F.pad(x.transpose(1, 2), (5, 0))
    k = M._t(w, "c1w", torch.float64).permute(2, 1, 0).contiguous()
    return F.conv1d(xc, k, M._t(w, "c1b", torch.float64)).transpose(1, 2).numpy()
