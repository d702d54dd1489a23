"""
CPU restatement (PyTorch, fp32 or fp64) of the reference's encoder sub-model, create_encoder() (genomad/neural_network/model.py:14-31):
the IGLOO block of oracle.igloo_model.forward followed by Dense(512) + BatchNorm + ReLU (model.py:28-30), 512 values per window.
Built on the oracle without changing it: forward() gives h0, and dense0() is the same operations as the first layer of
oracle.igloo_model.head.  Pinned to the reference's own encoder by tests/golden/reference_encoder_golden.npz
(make_reference_encoder_golden.py; tests/test_embed_cpu.py).
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import igloo_model as M


def dense0(h0: torch.Tensor, w, dtype):
    """Dense(512) + BatchNorm(eps = 1e-3, inference form) + ReLU on h0 [B, 256]."""
    def bn(x, p):
        return (M._t(w, p + "g", dtype) * (x - M._t(w, p + "m", dtype))
                / torch.sqrt(M._t(w, p + "v", dtype) + M.BN_EPS) + M._t(w, p + "b", dtype))
    return torch.relu(bn(h0 @ M._t(w, "d0w", dtype) + M._t(w, "d0b", dtype), "bn0"))


@torch.no_grad()
def encoder(tokens, w, dtype=torch.float32) -> np.ndarray:
    """tokens [B, 5997] -> the encoder output [B, 512]."""
    _, im = M.forward(tokens, w, dtype, return_intermediates=True)
    return dense0(im["h0"], w, dtype).numpy()
