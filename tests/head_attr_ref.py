"""
fp64 reference of head attributions (include/gnm.h, DESIGN.md "Head attributions"): the model with a C-class head in place of
the shipped tail is the shipped encoder with the head's d1w .. d2b under the shipped layer names (weights.HEAD_KEYS), so
ig_ref.logits_onehot gives its C logits on one-hot or interpolated input, following a given forward's max-pool routing,
LeakyReLU branches and head ReLU branches ([h1 > 0, hh > 0]).

Each row's C logit gradients are taken once (logit_jacobian); the gradient of log p_c is their combination with
g_logits = e_c - p at given logits (attr_ref.head_gradient_fp64, no 1 - p_c), so one Jacobian serves every target, the GPU
forward's logits, and every sharpened head (d2w, d2b times k multiply the logits by k and the gradient of log p_c by k at the
sharpened probabilities).
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch

import attr_ref as A
import ig_ref as I


def with_head(w: dict, head_arrays: dict) -> dict:
    """the shipped weights with the head's layers in place of the shipped tail"""
    out = dict(w)
    out.update({k: np.asarray(v, dtype=np.float32) for k, v in head_arrays.items()})
    return out


def logit_jacobian(tokens, w, alpha=None, baseline: str = "zero", routes: Optional[Sequence] = None,
                   masks: Optional[Sequence] = None, head_masks: Optional[Sequence] = None, batch: int = 8):
    """rows tokens [R, 5997] at alpha [R] (default 1: the window itself) -> (fp64 logits [R, C], J [R, C, 5997]: the row value
    of d logit_i / d x, g[t, tok[t]] or, for the N baseline, g[t, tok[t]] - g[t, 0])"""
    tokens = np.asarray(tokens)
    alpha = np.broadcast_to(np.asarray(1.0 if alpha is None else alpha, dtype=np.float64), (len(tokens),))
    lg_out, j_out = [], []
    for s in range(0, len(tokens), batch):
        sl = slice(s, s + batch)
        x = I.interp_onehot(tokens[sl], alpha[sl], baseline).requires_grad_(True)
        lg = I.logits_onehot(x, w, None if routes is None else [r[sl] for r in routes],
                             None if masks is None else [m[sl] for m in masks],
                             None if head_masks is None else [m[sl] for m in head_masks])
        C = lg.shape[1]
        J = []
        for i in range(C):
            (g,) = torch.autograd.grad(lg[:, i].sum(), x, retain_graph=i < C - 1)
            J.append(I._select(g, tokens[sl], baseline))
        lg_out.append(lg.detach().numpy())
        j_out.append(np.stack(J, axis=1))
    return np.concatenate(lg_out), np.concatenate(j_out)


def rows_from_jacobian(logits, J, target: int, scale: float = 1.0) -> np.ndarray:
    """[R, 5997] gradients of log p_c at `scale` x the given logits [R, C], for a head whose d2w, d2b are scaled by `scale`"""
    G = A.head_gradient_fp64(scale * np.asarray(logits, dtype=np.float64), target) * scale
    return np.einsum("ri,rit->rt", G, J)


def log_p(logits, target: int, scale: float = 1.0) -> np.ndarray:
    """log p_c without cancellation (attr_ref.log_p_target) at `scale` x logits [R, C]"""
    return A.log_p_target(torch.as_tensor(scale * np.asarray(logits, dtype=np.float64)), target).numpy()
