"""
Per-stage fp64 references of the classifier, for the stage-precision tests.

Every function takes the input of ONE stage -- in the GPU tests the kernel's own input, fetched with gnm_debug_fetch -- and returns
a ``Ref``: the fp64 value of the stage's output and two per-output scales of its contraction,

    s_abs = sum |terms|          (bound of any rounding of the terms; the max metric divides by it)
    s_rms = sqrt(sum terms^2)    (the size of the terms; the RMS metric divides by its RMS)

so an error measured against ``value`` is the error of that kernel alone, not drift carried in from upstream stages.  The
stages follow oracle/igloo_model.py (closed form); LeakyReLU, ReLU and max-pooling do not enlarge an error, so their scales are
those of the contraction in front of them.

``metrics`` turns (GPU output, Ref) into the two numbers the bars in ``BARS`` apply to:
    rms = RMS(err) / RMS(s_rms)                 over all outputs -- catches a change of recipe (a lost correction pass);
    max = max |err| / (s_abs + floor)           per region -- catches a bug confined to a few outputs (padding, tails,
                                                window-group edges).
"""
from __future__ import annotations

from typing import Dict, NamedTuple, Optional

import numpy as np
import torch
import torch.nn.functional as F

D = torch.float64
L_TOK, N_POOL, POOL = 5997, 749, 8


class Ref(NamedTuple):
    value: torch.Tensor
    s_abs: torch.Tensor
    s_rms: torch.Tensor


# (rms bar, max bar) per stage.  The tensor-core bars come from tests/test_stage_recipes.py, which emulates each recipe from its
# packing code and asserts that the recipe passes with >= 2x margin and that every mutant (a dropped correction pass, a single
# pass, corrections into a reduced-precision accumulator, small-weight operand planes) fails by >= 2x.  The fp32 CUDA-core stages
# (layer 1, attention, softmax and the conv_impl = 1 validation kernels) are held to fp32 rounding level.
BARS: Dict[str, tuple] = {
    "conv_tc": (4e-5, 1.2e-4),       # conv2 / conv3 on tensor cores: fp16 main pass + 2 e4m3 correction passes
    "conv_fp32": (4e-6, 1e-5),       # conv2 / conv3, fp32 validation kernels (conv_impl = 1): 768 sequential fp32 FMAs
    "y1": (2e-7, 2e-6),              # layer 1: fp32 sum of 6 table rows + bias, stored as hi16 + lo16
    "wv": (1e-5, 4e-5),              # w_v + maxpool8: fp16 x 3 passes (fp32 FFMA for conv_impl = 1)
    "gather": (3e-6, 2e-5),          # patch gather + bias: fp16 hi/lo x hi/lo (fp32 FFMA for fuse_gather = 0)
    "tf32x3": (2e-5, 2e-5),          # logits and the two Dense(512) layers: 3 x TF32 (fp32 FFMA for conv_impl = 1).  The H100
                                     # measures ~3e-6 rms for the logits, 10x the fp64-summed emulation and 7x the dense layers.
                                     # Not explained by a measurement; a model whose accumulator truncates after every K = 8
                                     # step gives 3.6e-6 for the logits' 352-product split-K partials (tests/test_stage_recipes.py)
    "attention": (1e-5, 5e-5),       # softmax over 749 logits + weighted sum of q, fp32 (h0[:128] also carries logits0's error)
    "probs": (2e-6, 1e-5),           # Dense(3) + softmax, fp32; absolute error of the probabilities
    # attribution backward pass (tests/attr_stage_ref.py); the bars come from tests/test_attr_stage_recipes_cpu.py, which emulates
    # each stage and a mutant of each.  conv_bwd_tc: the conv recipe over gradient rows whose per-window scale puts the maximum
    # in [1, 2): entries more than ~2^7 below it keep a normal lo8 no longer, so the per-output max is wider than conv_tc's
    "conv_bwd_tc": (4e-5, 4e-4),     # conv3 / conv2 backward on tensor cores, operand-row output (conv3) or fp32 rows (conv2)
    "attr_head": (1e-5, 1e-5),       # g_out: Dense(3), Dense(512) and Dense(512) backward, fp32
    "attr_igloo": (1e-5, 5e-5),      # g_y / g_z3: softmax, g_alpha, the g_mpi sgemm, value and patch paths, fp32
    "attr_layer1": (1e-5, 1e-5),     # attr: 6 table rows x 128 channels per position, fp32
    "attr_gz3_rows": (1e-4, 2e-3),   # IGLOO#1 + pack: s_w g_z3 stored as hi16 + lo8, max in [0.25, 0.5) (the max bar is
                                     # wider than the emulation's 2x for the 1.1e-3 the H100 measures; only the rms bar
                                     # separates the recipe from its mutant, rows without lo8)
}


def _t(x) -> torch.Tensor:
    return torch.as_tensor(np.asarray(x), dtype=D)


def _causal(x: torch.Tensor, W: torch.Tensor) -> torch.Tensor:
    """x [B, L, Cin], W [6, Cin, Cout] -> [B, L, Cout]: Keras causal Conv1D without bias (5 zero rows on the left)."""
    xx = F.pad(x.transpose(1, 2), (5, 0))
    return F.conv1d(xx, W.permute(2, 1, 0).contiguous()).transpose(1, 2)


def _lrelu(x):
    return torch.where(x > 0, x, 0.1 * x)


def _pool(z):
    return z[:, : N_POOL * POOL].reshape(z.shape[0], N_POOL, POOL, -1).amax(dim=2)


def conv1(tokens: np.ndarray, w) -> Ref:
    """Layer 1 (one-hot -> causal Conv1D -> LeakyReLU) from the tokens: y1[t] = lrelu(b + sum_j W1[j, tok[t-5+j]]); a token
    above 256 is an all-zero one-hot row (tf.one_hot(x, 257)) and adds nothing."""
    W = F.pad(_t(w["c1w"]), (0, 0, 0, 1))                               # [6, 258, 128]: row 257 = 0
    t = torch.as_tensor(np.asarray(tokens).astype(np.int64))
    t = torch.where(t > 256, 257, t)
    B, L = t.shape
    acc, sab, s2 = (torch.zeros(B, L, 128, dtype=D) for _ in range(3))
    for j in range(6):
        sh = 5 - j
        g = W[j][t[:, : L - sh]]
        acc[:, sh:] += g
        sab[:, sh:] += g.abs()
        s2[:, sh:] += g * g
    b = _t(w["c1b"])
    return Ref(_lrelu(acc + b), sab + b.abs(), torch.sqrt(s2 + b * b))


def conv(y: torch.Tensor, kernel, bias) -> Ref:
    """conv2 / conv3: causal Conv1D(128, 6) + LeakyReLU of the activations y [B, 5997, 128]."""
    y = y.to(D)
    W, b = _t(kernel), _t(bias)
    val = _lrelu(_causal(y, W) + b)
    return Ref(val, _causal(y.abs(), W.abs()) + b.abs(), torch.sqrt(_causal(y * y, W * W) + b * b))


def wv_pool(y: torch.Tensor, w_v) -> Ref:
    """q = maxpool8(y @ w_v); the max of perturbed values is within the largest perturbation, so the scales are pooled too."""
    y = y.to(D)
    Wv = _t(w_v).reshape(128, 128)
    return Ref(_pool(y @ Wv), _pool(y.abs() @ Wv.abs()), torch.sqrt(_pool((y * y) @ (Wv * Wv))))


def gather(y: torch.Tensor, w, s: int, chunk: int = 8) -> Ref:
    """mpi[p] = sum_k sum_c y[P[p,k], c] Wm[p,k,c] Ws[128k + c] + Wb[p] (the folded patch weights of the IGLOO kernel)."""
    y = y.to(D)
    P = torch.as_tensor(np.asarray(w[f"ig{s}_random_patches"]).reshape(-1, 4), dtype=torch.long)
    Wf = _t(w[f"ig{s}_w_mult"])[0] * _t(w[f"ig{s}_w_summer"]).reshape(1, 4, 128)
    b = _t(w[f"ig{s}_w_bias"]).reshape(-1)
    out = [[], [], []]
    for i in range(0, y.shape[0], chunk):
        t = y[i:i + chunk][:, P] * Wf
        out[0].append(t.sum(dim=(2, 3)) + b)
        out[1].append(t.abs().sum(dim=(2, 3)) + b.abs())
        out[2].append(torch.sqrt((t * t).sum(dim=(2, 3)) + b * b))
    return Ref(*(torch.cat(o) for o in out))


def matmul(a: torch.Tensor, B) -> Ref:
    """a @ B (the attention logits mpi @ w_qk)."""
    a, B = a.to(D), _t(B)
    return Ref(a @ B, a.abs() @ B.abs(), torch.sqrt((a * a) @ (B * B)))


def attention(logits: torch.Tensor, q: torch.Tensor) -> Ref:
    """out[c] = sum_g softmax(logits)[g] q[g, c] -- one 128-wide half of h0.  A weighted mean: both scales are sum alpha |q|
    (sqrt(sum (alpha q)^2) would shrink with the number of pooled positions, not the error)."""
    alpha = torch.softmax(logits.to(D)[:, :N_POOL], dim=-1)
    q = q.to(D)
    s = torch.einsum("bg,bgc->bc", alpha, q.abs())
    return Ref(torch.einsum("bg,bgc->bc", alpha, q), s, s)


def dense_bn_relu(h: torch.Tensor, w, layer: int) -> Ref:
    """relu(BatchNorm(h @ W + b)), Keras inference form x * inv + (beta - mean * inv), inv = gamma / sqrt(var + 1e-3)."""
    h = h.to(D)
    W, b = _t(w[f"d{layer}w"]), _t(w[f"d{layer}b"])
    p = f"bn{layer}"
    inv = _t(w[p + "g"]) / torch.sqrt(_t(w[p + "v"]) + 1e-3)
    shift = _t(w[p + "b"]) - _t(w[p + "m"]) * inv
    val = torch.relu((h @ W + b) * inv + shift)
    s_abs = inv.abs() * (h.abs() @ W.abs() + b.abs()) + shift.abs()
    s_rms = torch.sqrt(inv * inv * ((h * h) @ (W * W) + b * b) + shift * shift)
    return Ref(val, s_abs, s_rms)


def head_softmax(h2: torch.Tensor, w) -> Ref:
    """Dense(3) + softmax; probabilities are compared in absolute terms (scale 1)."""
    val = torch.softmax(h2.to(D) @ _t(w["d2w"]) + _t(w["d2b"]), dim=-1)
    one = torch.ones_like(val)
    return Ref(val, one, one)


# ------------------------------------------------------------------------------------------ metrics
def position_regions(n: int, pooled: bool = False, windows: Optional[list] = None, tile: Optional[int] = None) -> Dict[str, tuple]:
    """Index sets (window slice or indices, position slice) where kernels tend to go wrong: the causal zero fill (positions 0-5),
    the last, partial 256-position conv unit (5888-5996), the last 24-position IGLOO band (5976-5996), and the windows on both
    sides of the 8-window groups of the fused IGLOO kernel (8k - 1, 8k, 8k + 1).  pooled: the same regions in max-pool groups.
    windows: the batch indices of the rows actually compared (a sample of an n-window batch); the window regions then index
    into that sample.  tile: also the windows on both sides of every `tile`-row M tile edge of the tail GEMMs (tile k - 1,
    tile k, tile k + 1) and, when the last M tile is partial, the windows of that tile."""
    f = (lambda a, b: slice(a // POOL, min(N_POOL, (b + POOL) // POOL))) if pooled else (lambda a, b: slice(a, b + 1))

    def rows(edges):
        return sorted(edges) if windows is None else [r for r, i in enumerate(windows) if i in edges]
    edge = rows({i for k in range(8, n + 1, 8) for i in (k - 1, k, k + 1) if i < n})
    regions = {"all": (slice(None), slice(None)), "pos 0-5": (slice(None), f(0, 5)),
               "pos 5888-5996": (slice(None), f(5888, 5996)), "pos 5976-5996": (slice(None), f(5976, 5996))}
    if edge:
        regions["win 8k+-1"] = (edge, slice(None))
    if tile:
        t_edge = rows({i for k in range(tile, n, tile) for i in (k - 1, k, k + 1) if i < n})
        if t_edge:
            regions[f"win {tile}k+-1"] = (t_edge, slice(None))
        last = rows(set(range(n // tile * tile, n)))
        if n % tile and last:
            regions["win last tile"] = (last, slice(None))
    return regions


def metrics(got: torch.Tensor, ref: Ref, regions: Optional[Dict[str, tuple]] = None) -> Dict[str, float]:
    """{"rms": RMS(err) / RMS(s_rms), "max": max over all outputs, "max <region>": max per region} of the normalised error."""
    err = got.to(D).cpu() - ref.value
    out = {"rms": float(err.pow(2).mean().sqrt() / ref.s_rms.pow(2).mean().sqrt().clamp_min(1e-300))}
    floor = 1e-6 * float(ref.s_abs.max()) + 1e-300          # outputs whose terms all vanish: an absolute floor
    nerr = err.abs() / (ref.s_abs + floor)
    out["max"] = float(nerr.max())
    for name, (wi, pi) in (regions or {}).items():
        if name != "all":
            out["max " + name] = float(nerr[wi][:, pi].max()) if nerr.dim() > 2 else float(nerr[wi].max())
    return out
