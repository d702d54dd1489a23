"""
CPU restatement (PyTorch, fp32 or fp64) of the geNomad IGLOO1D classifier.
TEST INFRASTRUCTURE (see oracle/__init__.py).

Pinning status.  STRUCTURE PINNED, TensorFlow's arithmetic unpinned: TF / Keras / h5py cannot be installed in the build
container and the reference has no model tests, but the reference's own model definition (genomad/neural_network/model.py and
igloo.py, imported by path) runs on a NumPy stand-in for the ~25 TF / Keras calls it makes (tests/golden/keras_shim.py).  Its
outputs for 24 windows -- create_classifier() -> load_weights(nn_classifier.h5) -> predict, shipped weights and synthetic O(1)
IGLOO weights -- are committed (tests/golden/reference_graph_golden.npz, generator make_reference_graph_golden.py) and this
restatement agrees with them to 5e-14 in fp64 (tests/test_oracle_golden.py::test_oracle_model_matches_reference_graph).  The
semantics of the library calls themselves (causal Conv1D, gather_nd, MaxPool1D, BatchNormalization(eps=1e-3) ...) are the
documented ones, restated in that stand-in.  What is here follows the reference source text:

  one-hot                 genomad/neural_network/model.py:9-11
  encoder graph           genomad/neural_network/model.py:14-31
  classifier head         genomad/neural_network/model.py:34-45
  IGLOO1D_Block wiring    genomad/neural_network/igloo.py:30-83   (two IGLOO kernels: on conv #1 and conv #3 outputs)
  IGLOO1D_kernel.call     genomad/neural_network/igloo.py:190-217
  weight <-> layer order  Keras legacy-H5 loader maps by order; see `__weight_order__` in the npz

and the Keras defaults the source relies on: Conv1D is cross-correlation with kernel
layout [k, in, out], bias, "causal" = k-1 zeros on the left; LeakyReLU(negative_slope=0.1);
BatchNormalization(epsilon=1e-3) in inference form; MaxPool1D(pool=8, stride=8, "valid");
Dense = x @ W + b; softmax over the last axis; Dropout/SpatialDropout1D = identity.

Two formulations are provided and tested against each other:
  * forward_as_written : op-for-op (one-hot tensor -> conv1d; transpose/gather_nd/multiply/
                         reshape/matmul for the patches) -- this is also the timed CPU baseline
  * forward            : closed form (embedding-sum conv #1, folded patch weights)
"""
from __future__ import annotations

from typing import Callable, Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

L_TOK = 5997
N_PATCH = 2100
POOL = 8
N_POOL = L_TOK // POOL  # 749
BN_EPS = 1e-3
LRELU = 0.1

ENC = "/model/"
KEYS = {
    "c1w": ENC + "conv1d/kernel:0", "c1b": ENC + "conv1d/bias:0",
    "c2w": ENC + "conv1d_1/kernel:0", "c2b": ENC + "conv1d_1/bias:0",
    "c3w": ENC + "conv1d_2/kernel:0", "c3b": ENC + "conv1d_2/bias:0",
    "d0w": ENC + "dense/kernel:0", "d0b": ENC + "dense/bias:0",
    "bn0g": ENC + "batch_normalization/gamma:0", "bn0b": ENC + "batch_normalization/beta:0",
    "bn0m": ENC + "batch_normalization/moving_mean:0", "bn0v": ENC + "batch_normalization/moving_variance:0",
    "d1w": "/dense_1/dense_1/kernel:0", "d1b": "/dense_1/dense_1/bias:0",
    "bn1g": "/batch_normalization_1/batch_normalization_1/gamma:0",
    "bn1b": "/batch_normalization_1/batch_normalization_1/beta:0",
    "bn1m": "/batch_normalization_1/batch_normalization_1/moving_mean:0",
    "bn1v": "/batch_normalization_1/batch_normalization_1/moving_variance:0",
    "d2w": "/dense_2/dense_2/kernel:0", "d2b": "/dense_2/dense_2/bias:0",
}
for _s, _g in ((0, "igloo1d_kernel"), (1, "igloo1d_kernel_1")):
    for _w in ("w_mult", "w_summer", "w_bias", "w_qk", "w_v", "random_patches"):
        KEYS[f"ig{_s}_{_w}"] = f"{ENC}{_g}/{_w}:0"


def load_npz_weights(path) -> Dict[str, np.ndarray]:
    """Return {short_name: ndarray} from the npz written by tools/export_weights.py."""
    z = np.load(path)
    return {k: np.array(z[v]) for k, v in KEYS.items()}


def synthetic_igloo_weights(w: Dict[str, np.ndarray], seed: int = 7, scale: float = 1.0) -> Dict[str, np.ndarray]:
    """
    The shipped patch/attention weights are ~1e-32 (numerically dead: the softmax is exactly
    uniform), so a wrong gather cannot be seen through them.  This returns a copy in which
    w_mult, w_summer, w_bias, w_qk of both IGLOO kernels are redrawn at O(1) scale so the
    attention logits are O(1), and the patch indices are redrawn to include positions 0 and
    5996 and repeated positions across patches.  Conv / w_v / head weights are kept.
    """
    rng = np.random.default_rng(seed)
    out = dict(w)
    for s in (0, 1):
        out[f"ig{s}_w_mult"] = rng.uniform(-0.5, 0.5, (1, N_PATCH, 4, 128)).astype(np.float32) * scale
        out[f"ig{s}_w_summer"] = rng.uniform(-0.5, 0.5, (1, 512, 1)).astype(np.float32)
        out[f"ig{s}_w_bias"] = rng.uniform(-0.5, 0.5, (1, N_PATCH)).astype(np.float32)
        out[f"ig{s}_w_qk"] = rng.uniform(-0.25, 0.25, (N_PATCH, N_POOL)).astype(np.float32)
        p = np.sort(np.stack([rng.choice(L_TOK, 4, replace=False) for _ in range(N_PATCH)]), axis=1)
        p[0] = [0, 1, 2, 5996]
        p[1] = [0, 7, 8, 5996]
        p[2] = [5993, 5994, 5995, 5996]
        p[3:40, 1] = 3000  # one position shared by many patches
        p[3:40] = np.sort(p[3:40], axis=1)
        out[f"ig{s}_random_patches"] = p.astype(np.int32).reshape(N_PATCH, 4, 1)
    return out


def _t(w, k, dtype):
    return torch.as_tensor(np.asarray(w[k]), dtype=dtype)


def _lrelu(x):
    return torch.where(x > 0, x, x * LRELU)


# ----------------------------------------------------------------------------- pieces
def vocab_tokens(tok: torch.Tensor) -> torch.Tensor:
    """Tokens as int64 with every value above 256 replaced by 257: tf.one_hot(x, 257) gives such a token an all-zero row,
    and index 257 selects the zero row that `conv1_*` append to the 257 real ones."""
    t = tok.long()
    return torch.where(t > 256, torch.full_like(t, 257), t)


def conv1_as_written(tok: torch.Tensor, w, dtype):
    """tf.one_hot(257) -> Conv1D(128, 6, causal) -> LeakyReLU   (model.py:11, igloo.py:45-48)"""
    oh = F.one_hot(vocab_tokens(tok), 258)[..., :257].to(dtype)     # [B, L, 257]; tokens > 256: zero rows
    x = F.pad(oh.transpose(1, 2), (5, 0))                            # causal: 5 zero rows on the left
    k = _t(w, "c1w", dtype).permute(2, 1, 0).contiguous()            # [k,in,out] -> [out,in,k]
    return _lrelu(F.conv1d(x, k, _t(w, "c1b", dtype))).transpose(1, 2)


def conv1_embedding(tok: torch.Tensor, w, dtype):
    """y1[t] = lrelu(b + sum_j W1[j, tok[t-5+j]]), taps added in order j = 0..5; padded taps and tokens > 256 add nothing."""
    W = F.pad(_t(w, "c1w", dtype), (0, 0, 0, 1))                     # [6, 258, 128]: row 257 = 0
    B, L = tok.shape
    acc = torch.zeros(B, L, 128, dtype=dtype)
    t = vocab_tokens(tok)
    for j in range(6):
        sh = 5 - j                                                   # tap j reads tok[t - sh]
        acc[:, sh:, :] += W[j][t[:, : L - sh]]
    return _lrelu(acc + _t(w, "c1b", dtype))


def causal_conv(y: torch.Tensor, kernel: np.ndarray, bias: np.ndarray, dtype,
                round_a: Optional[Callable] = None, round_w: Optional[Callable] = None):
    """Conv1D(128, 6, causal) + LeakyReLU (igloo.py:64-67). round_* optionally emulate reduced-precision operands."""
    k = torch.as_tensor(kernel, dtype=dtype)
    if round_w is not None:
        k = round_w(k)
    if round_a is not None:
        y = round_a(y)
    x = F.pad(y.transpose(1, 2), (5, 0))
    out = F.conv1d(x, k.permute(2, 1, 0).contiguous(), torch.as_tensor(bias, dtype=dtype))
    return _lrelu(out).transpose(1, 2)


def igloo_as_written(y: torch.Tensor, w, s: int, dtype):
    """IGLOO1D_kernel.call transcribed op for op (igloo.py:190-217)."""
    patches = torch.as_tensor(np.asarray(w[f"ig{s}_random_patches"]), dtype=torch.long)  # [2100,4,1]
    M = y.permute(1, 2, 0)                                           # tf.transpose(y,[1,2,0]) -> [L, C, B]
    M = M[patches[..., 0]]                                           # tf.gather_nd -> [2100,4,C,B]
    mpi = M.permute(3, 0, 1, 2)                                      # [B,2100,4,C]
    mpi = _t(w, f"ig{s}_w_mult", dtype) * mpi
    mpi = mpi.reshape(-1, N_PATCH, 4 * y.shape[2])
    mpi = torch.matmul(mpi, _t(w, f"ig{s}_w_summer", dtype)).squeeze(-1)
    mpi = mpi + _t(w, f"ig{s}_w_bias", dtype)
    y_proj = torch.matmul(y, _t(w, f"ig{s}_w_v", dtype))             # [B,L,C]
    y_proj = F.max_pool1d(y_proj.transpose(1, 2), POOL).transpose(1, 2)   # valid, stride 8 -> [B,749,C]
    alpha = torch.softmax(torch.matmul(mpi, _t(w, f"ig{s}_w_qk", dtype)), dim=-1)
    return torch.matmul(alpha.unsqueeze(1), y_proj).squeeze(1)       # [B,C]


def igloo_closed(y: torch.Tensor, w, s: int, dtype, wv_fn: Optional[Callable] = None, return_parts=False):
    """
    mpi[p] = sum_k sum_c y[P[p,k],c] * Wm[p,k,c] * Ws[128k+c] + Wb[p];  q = maxpool8(y @ Wv);
    out = softmax(mpi @ Wqk) @ q.   wv_fn(y, Wv) optionally replaces the projection (precision studies).
    """
    P = torch.as_tensor(np.asarray(w[f"ig{s}_random_patches"]).reshape(N_PATCH, 4), dtype=torch.long)
    Wf = _t(w, f"ig{s}_w_mult", dtype)[0] * _t(w, f"ig{s}_w_summer", dtype).reshape(1, 4, 128)
    g = y[:, P]                                                      # [B,2100,4,128]
    mpi = (g * Wf).sum(dim=(2, 3)) + _t(w, f"ig{s}_w_bias", dtype)
    Wv = _t(w, f"ig{s}_w_v", dtype)[0]
    z = wv_fn(y, Wv) if wv_fn is not None else y @ Wv
    q = z[:, : N_POOL * POOL].reshape(y.shape[0], N_POOL, POOL, -1).amax(dim=2)
    logits = mpi @ _t(w, f"ig{s}_w_qk", dtype)
    alpha = torch.softmax(logits, dim=-1)
    out = torch.einsum("bg,bgc->bc", alpha, q)
    if return_parts:
        return out, dict(mpi=mpi, q=q, logits=logits, alpha=alpha)
    return out


def head(h0: torch.Tensor, w, dtype, return_logits=False):
    """Dense512+BN+ReLU (model.py:28-30), Dense512+BN+ReLU, Dense3+softmax (model.py:40-44)."""
    def bn(x, p):
        return (_t(w, p + "g", dtype) * (x - _t(w, p + "m", dtype))
                / torch.sqrt(_t(w, p + "v", dtype) + BN_EPS) + _t(w, p + "b", dtype))
    h1 = torch.relu(bn(h0 @ _t(w, "d0w", dtype) + _t(w, "d0b", dtype), "bn0"))
    h2 = torch.relu(bn(h1 @ _t(w, "d1w", dtype) + _t(w, "d1b", dtype), "bn1"))
    logits = h2 @ _t(w, "d2w", dtype) + _t(w, "d2b", dtype)
    if return_logits:
        return logits
    return torch.softmax(logits, dim=-1)


# ----------------------------------------------------------------------------- whole model
@torch.no_grad()
def forward_as_written(tokens, w, dtype=torch.float32) -> np.ndarray:
    """Op-for-op graph the reference executes per batch (nn_classification.py:317). tokens [B,5997] ints."""
    tok = torch.as_tensor(np.asarray(tokens).astype(np.int64))
    y1 = conv1_as_written(tok, w, dtype)
    o0 = igloo_as_written(y1, w, 0, dtype)
    y2 = causal_conv(y1, w["c2w"], w["c2b"], dtype)
    y3 = causal_conv(y2, w["c3w"], w["c3b"], dtype)
    o1 = igloo_as_written(y3, w, 1, dtype)
    return head(torch.cat([o0, o1], dim=1), w, dtype).numpy()


@torch.no_grad()
def forward(tokens, w, dtype=torch.float32, round_a=None, round_w=None, wv_fn=None,
            return_intermediates: bool = False):
    """Closed-form restatement; optional operand-rounding hooks for conv2/conv3 and w_v."""
    tok = torch.as_tensor(np.asarray(tokens).astype(np.int64))
    y1 = conv1_embedding(tok, w, dtype)
    o0, p0 = igloo_closed(y1, w, 0, dtype, wv_fn, return_parts=True)
    y2 = causal_conv(y1, w["c2w"], w["c2b"], dtype, round_a, round_w)
    y3 = causal_conv(y2, w["c3w"], w["c3b"], dtype, round_a, round_w)
    o1, p1 = igloo_closed(y3, w, 1, dtype, wv_fn, return_parts=True)
    h0 = torch.cat([o0, o1], dim=1)
    probs = head(h0, w, dtype).numpy()
    if return_intermediates:
        return probs, dict(y1=y1, y2=y2, y3=y3, h0=h0, ig0=p0, ig1=p1)
    return probs
