"""
fp64 oracle of the novelty attributions (include/gnm.h "Novelty attributions", DESIGN.md "Head novelty") and the a-priori
bound the H100 tests hold the GPU's seed to.

For a window's encoder output h1, its target class c and the head's model (center, P lower triangular, m):

    r = P (h1 - center) - m_c,   D_c = ||r||^2 / 512,   g_h1 = dD_c / dh1 = (2 / 512) P^T r

The gradient's sensitivity to h1 is Sigma^-1 (kappa up to 5e4 on real embeddings), so an fp64 run from the tokens, whose h1
differs from the GPU's by fp32 rounding, is no bar for the whole path.  The tests check the two stages separately:
- the seed: g_h1 against fp64 on the GPU's own h1 (grad_bound);
- the encoder backward: each attribution row against the fp64 vector-Jacobian product sum_j g_h1,gpu[j] h1(x)[j], along the
  GPU forward's max-pool routing, LeakyReLU branches and h1 > 0 mask (encoder_vjp).
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch

import attr_ref as A
import ig_ref as I
from novelty_ref import DIM, TINY32, U, U32, gamma
from oracle import igloo_model as M


def residual(x, center, P, m, target):
    """fp64 r [n, 512] = P (x - center) - m_target."""
    x = np.asarray(x, np.float64)
    Y = (x - np.asarray(center, np.float64)) @ np.asarray(P, np.float64).T
    return Y - np.asarray(m, np.float64)[np.asarray(target)]


def grad(x, center, P, m, target):
    """fp64 g_h1 [n, 512] = (2 / 512) P^T r."""
    return (2.0 / DIM) * residual(x, center, P, m, target) @ np.asarray(P, np.float64)


def grad_bound(x, center, P, m, target):
    """(g [n, 512], bound [n, 512]): g from the fp64 oracle, and a bound on |g_device - g| for a device that forms Y, r and
    P^T r in fp64 (any fixed order) and stores g in fp32.  With a = |x - center|:
      dY = gamma_514 |P| a            (Y = P (x - center): 512 products and the subtraction)
      dr = dY + u |r|                 (r = Y - m_c)
      |dg| <= (2 / 512) (|P^T| dr + gamma_513 |P^T| |r|)
    doubled because the oracle is an fp64 computation too, then 2^-24 of the value for the fp32 store and 2^-150 absolute."""
    x = np.asarray(x, np.float64)
    center, P = np.asarray(center, np.float64), np.asarray(P, np.float64)
    a = np.abs(x - center)
    r = residual(x, center, P, m, target)
    g = (2.0 / DIM) * r @ P
    dY = gamma(DIM + 2) * (a @ np.abs(P).T)
    dr = dY + U * np.abs(r)
    b64 = (2.0 / DIM) * (dr @ np.abs(P) + gamma(DIM + 1) * (np.abs(r) @ np.abs(P)))
    return g, 2 * b64 + U32 * (np.abs(g) + 2 * b64) + TINY32


def grad_ratio(g_dev, g, bound) -> float:
    """max |g_dev - g| / bound (0 / 0 read as 0)."""
    err = np.abs(np.asarray(g_dev, np.float64) - g)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(r.max())


# ------------------------------------------------------------------------------------------------ emulated errors (CPU tests)
def grad_other_order(x, center, P, m, target):
    """fp64 g_h1 with every sum in another order: Y and P^T r summed from the last index down, one column at a time."""
    x = np.asarray(x, np.float64)
    a = (x - np.asarray(center, np.float64))[:, ::-1]
    P = np.asarray(P, np.float64)
    Y = np.stack([np.einsum("nk,k->n", a, P[i, ::-1]) for i in range(DIM)], 1)
    r = Y - np.asarray(m, np.float64)[np.asarray(target)]
    Pr = P[::-1]
    g = np.stack([np.einsum("ni,i->n", r[:, ::-1], Pr[:, j]) for j in range(DIM)], 1)
    return ((2.0 / DIM) * g).astype(np.float32)


def grad_fp32_residual(x, center, P, m, target):
    """the error of forming r in fp32: r rounded to fp32, then P^T r in fp64."""
    r = residual(x, center, P, m, target).astype(np.float32).astype(np.float64)
    return ((2.0 / DIM) * r @ np.asarray(P, np.float64)).astype(np.float32)


def grad_no_diagonal(x, center, P, m, target):
    """the error of dropping the i = j term from P^T r (a tile loop that starts one row below the diagonal)."""
    P = np.asarray(P, np.float64)
    r = residual(x, center, P, m, target)
    return ((2.0 / DIM) * r @ np.tril(P, -1)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ encoder backward (fp64)
def h1_onehot(x, w, routes: Optional[Sequence] = None, masks: Optional[Sequence] = None, h1_mask=None):
    """the encoder output h1 = relu(bn0(h0 d0w + d0b)) [B, 512] on one-hot (or relaxed) input x, along a given forward's
    max-pool routing, LeakyReLU branches and, with h1_mask, its ReLU branches (attr_ref.logits_onehot's pieces)."""
    dt = torch.float64
    ms = masks if masks is not None else (None, None, None)
    xc = torch.nn.functional.pad(x.transpose(1, 2), (5, 0))
    k = M._t(w, "c1w", dt).permute(2, 1, 0).contiguous()
    y1 = A._act(torch.nn.functional.conv1d(xc, k, M._t(w, "c1b", dt)).transpose(1, 2), ms[0])
    o0 = A._igloo(y1, w, 0, dt, None if routes is None else routes[0])

    def conv(y, s, mask):
        kk = torch.as_tensor(w[f"c{s}w"], dtype=dt).permute(2, 1, 0).contiguous()
        z = torch.nn.functional.conv1d(torch.nn.functional.pad(y.transpose(1, 2), (5, 0)), kk,
                                       torch.as_tensor(w[f"c{s}b"], dtype=dt)).transpose(1, 2)
        return A._act(z, mask)
    y3 = conv(conv(y1, 2, ms[1]), 3, ms[2])
    o1 = A._igloo(y3, w, 1, dt, None if routes is None else routes[1])
    h0 = torch.cat([o0, o1], dim=1)
    z = M._t(w, "bn0g", dt) * (h0 @ M._t(w, "d0w", dt) + M._t(w, "d0b", dt) - M._t(w, "bn0m", dt)) \
        / torch.sqrt(M._t(w, "bn0v", dt) + M.BN_EPS) + M._t(w, "bn0b", dt)
    if h1_mask is None:
        return torch.relu(z)
    return torch.where(torch.as_tensor(np.asarray(h1_mask)), z, torch.zeros_like(z))


def encoder_vjp(tokens, w, g_h1, alpha=None, baseline: str = "zero", routes: Optional[Sequence] = None,
                masks: Optional[Sequence] = None, h1_mask=None, batch: int = 8) -> np.ndarray:
    """rows tokens [R, 5997] (at alpha [R], default 1: the window itself), seeds g_h1 [R, 512] -> [R, 5997]: the row value
    (g[t, tok[t]], or g[t, tok[t]] - g[t, 0] for the N baseline) of d (sum_j g_h1[j] h1(x)[j]) / d x in fp64."""
    tokens = np.asarray(tokens)
    alpha = np.broadcast_to(np.asarray(1.0 if alpha is None else alpha, dtype=np.float64), (len(tokens),))
    out = []
    for s in range(0, len(tokens), batch):
        sl = slice(s, s + batch)
        x = I.interp_onehot(tokens[sl], alpha[sl], baseline).requires_grad_(True)
        h = h1_onehot(x, w, None if routes is None else [r[sl] for r in routes],
                      None if masks is None else [mm[sl] for mm in masks], None if h1_mask is None else h1_mask[sl])
        (g,) = torch.autograd.grad((h * torch.as_tensor(np.asarray(g_h1[sl], np.float64))).sum(), x)
        out.append(I._select(g, tokens[sl], baseline))
    return np.concatenate(out)
