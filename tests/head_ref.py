"""
fp64 NumPy statement of the classifier-head semantics of include/gnm.h (gnm_head_forward, gnm_head_train_*): inference, the
training-mode forward, its backward, Adam, the moving statistics and the dropout hash.  The GPU tests compare against it; the
CPU tests check the backward against finite differences.
"""
import numpy as np

EPS_BN = 1e-3
KEEP = 0.8
THRESHOLD = 858993460            # ceil(0.2 * 2^32)
M32 = 0xFFFFFFFF


def mix32(x):
    x = np.asarray(x, dtype=np.uint64) & M32
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x7FEB352D)) & np.uint64(M32)
    x ^= x >> np.uint64(15)
    x = (x * np.uint64(0x846CA68B)) & np.uint64(M32)
    x ^= x >> np.uint64(16)
    return x


def key(seed: int) -> int:
    return (int(seed) * 0x9E3779B1 + 0x7F4A7C15) & M32


def keep_mask(seed: int, step: int, B: int, width: int = 512) -> np.ndarray:
    """bool [B, width]: keep(seed, step, row, col)."""
    s = mix32(np.uint64(key(seed) ^ (int(step) & M32)))
    r = mix32((s + np.arange(B, dtype=np.uint64)) & np.uint64(M32))
    h = mix32((r[:, None] + np.arange(width, dtype=np.uint64)[None, :]) & np.uint64(M32))
    return h >= THRESHOLD


def softmax(l):
    m = l.max(1, keepdims=True)
    e = np.exp(l - m)
    return e / e.sum(1, keepdims=True)


def xent(logits, labels):
    """Per row -log softmax(logits)[y] and its gradient softmax(logits) - onehot(y) in fp64, each to full relative precision:
    the loss is (max - l_y) + log1p(sum_{c != a} e^(l_c - max)), a the argmax, and the target component -sum_{c != y} p_c.
    p_y - 1 and log(sum e^(l - max)) would cancel once the margin reaches about 37, where p_y == 1.0 in fp64."""
    l = np.asarray(logits, np.float64)
    r, y = np.arange(len(l)), np.asarray(labels)
    m = l.max(1)
    e = np.exp(l - m[:, None])
    cls = np.arange(l.shape[1])[None, :]
    s = e.sum(1)
    g = e / s[:, None]
    g[r, y] = -np.where(cls == y[:, None], 0.0, e).sum(1) / s
    nll = (m - l[r, y]) + np.log1p(np.where(cls == l.argmax(1)[:, None], 0.0, e).sum(1))
    return nll, g


def _butterfly(v):
    """The xor-shuffle sum of 32 float32 lanes (lanes past the row's classes hold 0), as every lane of the warp ends it."""
    lanes = np.zeros((v.shape[0], 32), np.float32)
    lanes[:, :v.shape[1]] = v
    for off in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, np.arange(32) ^ off]
    return lanes[:, 0]


def xent_fp32(logits32, labels, cw, B: int):
    """(row loss, dZ2) in float32 in head_softmax_xent_kernel's order: m = max, e = exp(l - m), a = the lowest class at m,
    sa / sy = butterfly sums of e without class a / class y, s = 1 + sa; dZ2 = w (e / s) / B off the label and
    w (-(sy / s)) / B at it; loss = w ((m - l_y) + log1p(sa)).  NumPy's float32 exp and log1p stand in for expf and log1pf."""
    l = np.asarray(logits32, np.float32)
    r, y = np.arange(len(l)), np.asarray(labels)
    cls = np.arange(l.shape[1])[None, :]
    m = l.max(1)
    e = np.exp(l - m[:, None])
    a = (l == m[:, None]).argmax(1)
    sa = _butterfly(np.where(cls == a[:, None], np.float32(0), e))
    sy = _butterfly(np.where(cls == y[:, None], np.float32(0), e))
    s = np.float32(1) + sa
    w = np.asarray(cw, np.float32)[y]
    q = e / s[:, None]
    q[r, y] = -(sy / s)
    return w * ((m - l[r, y]) + np.log1p(sa)), w[:, None] * q / np.float32(B)


def xent_fp32_cancelling(logits32, labels, cw, B: int):
    """The same from the formula the kernel used before: dZ2 = w (e / s - onehot(y)) / B, loss = w -((l_y - m) - log(s)) with
    s the butterfly sum of every e.  Both cancel once p_y is near 1."""
    l = np.asarray(logits32, np.float32)
    r, y = np.arange(len(l)), np.asarray(labels)
    m = l.max(1)
    e = np.exp(l - m[:, None])
    s = _butterfly(e)
    w = np.asarray(cw, np.float32)[y]
    q = e / s[:, None]
    q[r, y] -= np.float32(1)
    return w * -((l[r, y] - m) - np.log(s)), w[:, None] * q / np.float32(B)


def infer(a, X) -> np.ndarray:
    """Head in inference mode: float64 probabilities [n, C]."""
    f = {k: np.asarray(v, np.float64) for k, v in a.items()}
    z = np.asarray(X, np.float64) @ f["d1w"] + f["d1b"]
    y = (z - f["bn1m"]) / np.sqrt(f["bn1v"] + EPS_BN) * f["bn1g"] + f["bn1b"]
    return softmax(np.maximum(y, 0) @ f["d2w"] + f["d2b"])


U32 = 2.0 ** -24                 # unit roundoff of fp32 (round to nearest)
TF32_MASK = np.uint32(0xFFFFE000)


def fold32(a):
    """(scale, shift) float32 [512] as gnm_head_create's fold_bn rounds them, in its operation order:
    inv = gamma * (1 / sqrt(var + 1e-3f)); shift = beta - mean * inv, every step in fp32 (no contraction on the host)."""
    f32 = np.float32
    g, b, m, v = (np.asarray(a[k], f32) for k in ("bn1g", "bn1b", "bn1m", "bn1v"))
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        inv = g * (f32(1) / np.sqrt(v + f32(1e-3)))
        return inv, b - m * inv


def _logits64(a, X, scale, shift):
    f = {k: np.asarray(a[k], np.float64) for k in ("d1w", "d1b", "d2w", "d2b")}
    z = np.asarray(X, np.float64) @ f["d1w"] + f["d1b"]
    y = z * np.asarray(scale, np.float64) + np.asarray(shift, np.float64)
    h = np.maximum(y, 0)
    return dict(z=z, y=y, h=h, logits=h @ f["d2w"] + f["d2b"])


def logits_exact(a, X) -> np.ndarray:
    """fp64 logits of the exact head (infer's): BN as (z - mean) / sqrt(var + 1e-3) * gamma + beta."""
    f = {k: np.asarray(v, np.float64) for k, v in a.items()}
    inv = f["bn1g"] / np.sqrt(f["bn1v"] + EPS_BN)
    return _logits64(a, X, inv, f["bn1b"] - f["bn1m"] * inv)["logits"]


def folded(a, X) -> dict:
    """fp64 evaluation of the head as the library evaluates it: fold32's float32 scale / shift, everything after them in fp64.
    Returns z, y (BN output), h (ReLU), logits [n, C] and logp [n, C] (log_softmax without cancellation)."""
    sc, sh = fold32(a)
    r = _logits64(a, X, sc, sh)
    r["logp"] = log_softmax(r["logits"])
    return r


def infer_folded(a, X) -> np.ndarray:
    """Probabilities [n, C] of folded(): the reference of gnm_head_forward's kernels, apart from the fold they share."""
    return np.exp(folded(a, X)["logp"])


def log_softmax(l) -> np.ndarray:
    """log p = (l - max) - log1p(sum_{c != argmax} e^(l_c - max)) in fp64: full relative precision for every class."""
    l = np.asarray(l, np.float64)
    m = l.max(1, keepdims=True)
    e = np.exp(l - m)
    a = l.argmax(1)
    e[np.arange(len(l)), a] = 0.0
    return (l - m) - np.log1p(e.sum(1, keepdims=True))


def fold_bound(a, X) -> np.ndarray:
    """Bound [n, C] on |logits of folded() - logits_exact()|: the error of fold_bn's float32 scale and shift, carried in fp64.
    Per unit j, with inv the exact gamma / sqrt(var + 1e-3) and d = 4u (u = 2^-24) the relative error of the rounded inv
    (var + 1e-3f: u, plus 1e-3f's own representation error, halved by sqrt; sqrt: u; 1 / s: u; gamma * r: u):
        |scale - inv|           <= |inv| d
        |shift - (beta - m inv)| <= |m inv| (d + u) + |shift| u        (mean * inv rounded, then the subtraction)
        |dy|                    <= |z inv| d + |m inv| (d + u) + |shift| u
    ReLU is 1-Lipschitz, so |d logit_c| <= sum_j |dy_j| |W2_jc|.  |m inv| >> |beta| makes the shift cancel: the fold loses
    |m inv| u absolutely, where the unfolded form (z - m) inv loses only |z - m| inv u; Keras' inference form shares this."""
    f = {k: np.asarray(v, np.float64) for k, v in a.items()}
    inv = f["bn1g"] / np.sqrt(f["bn1v"] + EPS_BN)
    _, sh = fold32(a)
    z = np.asarray(X, np.float64) @ f["d1w"] + f["d1b"]
    d = 4 * U32
    dy = np.abs(z * inv) * d + np.abs(f["bn1m"] * inv) * (d + U32) + np.abs(sh.astype(np.float64)) * U32
    return dy @ np.abs(f["d2w"])


def split_tf32(x):
    """float32 x -> (hi, lo), both float32 with the low 13 mantissa bits clear: hi = x truncated to TF32, lo = (x - hi) truncated
    (x - hi is exact in fp32), the bits of head_split_tf32_kernel and split_dense_t."""
    x = np.ascontiguousarray(x, np.float32)
    hi = (x.view(np.uint32) & TF32_MASK).view(np.float32)
    r = np.ascontiguousarray(x - hi)
    return hi, (r.view(np.uint32) & TF32_MASK).view(np.float32)


# fp32 accumulations of gnm_head_forward's kernels (api.cu, logits_tc.cuh, dense.cuh, head.cuh)
TC_SPLITS, TC_CHUNK, TC_KSTEP = 8, 32, 8          # dense_1 on the tensor cores: K = 512 in 8 splits of 2 chunks of 32
TC_MMA_PER_SPLIT = (512 // TC_SPLITS // TC_KSTEP) * 3   # 24 wgmma (K = 8, tf32) per accumulator chain: 3 passes per K step
TC_MMA_ERR = 4                                    # one wgmma's error, in u (Sum |acc| + |its 8 products|), see kernel_bound


def kernel_bound(a, X, route: str) -> dict:
    """Per-row error bounds of gnm_head_forward against folded() (same scale / shift), for route "tc" (conv_impl 0: 3 x TF32 on
    the tensor cores) or "ffma" (conv_impl 1).  u = 2^-24; S_j = sum_k |x_k| |W1_kj|; every bound is on an absolute error and
    first order in u (second-order terms are covered by using |value| + bound wherever a computed value is bounded).

    z = x W1 + b1.
      tc:   x = xh + xl + xr and w = wh + wl + wr (xh, xl the TF32 halves, xr what they leave, |xr| < 2^-21 |x|); the kernel
            forms xh wh + xl wh + xh wl, so each product loses xh wr + xl (wl + wr) + xr w, summed in absolute value over k
            (three fp64 products of |.| matrices).  A lo half that is an fp32 subnormal is counted as lost as well, in case the
            tensor core flushes it.  The products of TF32 values are exact.  Each split's accumulator takes 24 wgmma (K = 8):
            each is bounded by 4u (|acc| + sum of its products' magnitudes) -- 2u for a truncating normalisation plus ~2u for
            aligning 9 terms to the largest with 3 guard bits -- and both are <= S_j, so 96 u S_j; the 8 split partials are added
            in fp32 (7 u S_j), then b1 (u (S_j + |b1_j|)).
      ffma: 512 fmaf in k order (sgemm_epi_kernel): gamma_512 S_j, gamma_n = n u / (1 - n u); then b1 as above.
    y = z scale + shift (one FFMA, or a multiply and an add): |dy| <= |scale| |dz| + u (|scale| (|z| + |dz|) + |y| + |scale| |dz|).
    h = relu(y): 1-Lipschitz, |dh| <= |dy|.
    logit_c = sum_j h_j W2_jc + b2_c (head_softmax_kernel: 16 fmaf per lane in k order, a 5-level butterfly, then + b2):
            |dl_c| <= sum_j |dh_j| |W2_jc| + 21 u sum_j (|h_j| + |dh_j|) |W2_jc| + u (|l_c| + sum_j (|h_j| + |dh_j|) |W2_jc|).
    log p_c = l_c - m - log s (max m, s = sum_i e^(l_i - m)), computed as e_c = expf(l_c - m) (the subtraction: u |l_c - m|;
    expf: 2 ulp <= 4u), s by C - 1 adds (C u), p_c = e_c * (1 / s) (2u):
            |d log p_c| <= |dl_c| + max_i |dl_i| + sm_c,   sm_c = u |l_c - m| + 6u + C u + sum_i p_i (4u + u |l_i - m|).
    Returns dict(ref=folded(a, X), dz, dy, dl [n, C], dlogp [n, C])."""
    r = folded(a, X)
    u = U32
    X32 = np.asarray(X, np.float32)
    W32 = np.asarray(a["d1w"], np.float32)
    X64, W64 = X32.astype(np.float64), W32.astype(np.float64)
    S = np.abs(X64) @ np.abs(W64)
    b1 = np.abs(np.asarray(a["d1b"], np.float64))
    if route == "tc":
        (xh, xl), (wh, wl) = split_tf32(X32), split_tf32(W32)
        xh, xl, wh, wl = (v.astype(np.float64) for v in (xh, xl, wh, wl))
        xr, wr = X64 - xh - xl, W64 - wh - wl
        sub = lambda v: np.where((v != 0) & (np.abs(v) < 2.0 ** -126), np.abs(v), 0.0)
        drop = np.abs(xh) @ np.abs(wr) + np.abs(xl) @ np.abs(wl + wr) + np.abs(xr) @ np.abs(W64)      # <= 2^-19 S
        drop = drop + sub(xl) @ np.abs(wh) + np.abs(xh) @ sub(wl)
        dz = drop + (TC_MMA_PER_SPLIT * TC_MMA_ERR + TC_SPLITS - 1) * u * S + u * (S + b1)
    elif route == "ffma":
        n_k = X64.shape[1]
        dz = n_k * u / (1 - n_k * u) * S + u * (S + b1)
    else:
        raise ValueError(route)
    sc = np.abs(fold32(a)[0].astype(np.float64))
    dy = sc * dz + u * (sc * (np.abs(r["z"]) + dz) + np.abs(r["y"]) + sc * dz)
    W2 = np.abs(np.asarray(a["d2w"], np.float64))
    hw = (np.abs(r["h"]) + dy) @ W2
    dl = dy @ W2 + 21 * u * hw + u * (np.abs(r["logits"]) + hw)
    l = r["logits"]
    lm = np.abs(l - l.max(1, keepdims=True))
    C = l.shape[1]
    p = np.exp(r["logp"])
    sm = u * lm + (6 + C) * u + (p * (4 * u + u * lm)).sum(1, keepdims=True)
    return dict(ref=r, dz=dz, dy=dy, dl=dl, dlogp=dl + dl.max(1, keepdims=True) + sm)


def _rz32(x64):
    """fp64 -> fp32 rounded toward zero."""
    f = np.asarray(x64, np.float64).astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(x64)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f


def _fma32(a, b, c):
    """fmaf emulated in fp64: the product of two fp32 values is exact there; one more rounding of the sum (off by at most one
    fp32 ulp in a double-rounding tie, far inside every bound it is used against)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def emulate_forward(a, X, route: str, drop_pass: bool = False) -> dict:
    """NumPy emulation of gnm_head_forward in fp32: dense_1 (route "tc": the three TF32 passes, 8-product groups summed exactly
    and added to a round-toward-zero fp32 accumulator per wgmma, split partials added in fp32; "ffma": 512 sequential fmaf),
    + b1, the FFMA epilogue with fold32's scale / shift, ReLU, and head_softmax_kernel's lanes, butterfly and bias.
    drop_pass=True leaves out the xl wh pass (a mutant the bound must catch).  Returns z, y, h, logits (float32)."""
    X32 = np.asarray(X, np.float32)
    W32 = np.asarray(a["d1w"], np.float32)
    n, K = X32.shape
    if route == "tc":
        (xh, xl), (wh, wl) = split_tf32(X32), split_tf32(W32)
        xh, xl, wh, wl = (v.astype(np.float64) for v in (xh, xl, wh, wl))
        passes = [(xh, wh), (xh, wl)] if drop_pass else [(xh, wh), (xl, wh), (xh, wl)]
        per = K // TC_SPLITS
        acc = None
        for s in range(TC_SPLITS):
            part = np.zeros((n, W32.shape[1]), np.float32)
            for k0 in range(s * per, (s + 1) * per, TC_KSTEP):
                ks = slice(k0, k0 + TC_KSTEP)
                for A, B in passes:
                    part = _rz32(part.astype(np.float64) + A[:, ks] @ B[ks])
            acc = part if acc is None else (acc + part).astype(np.float32)
        z = acc
    else:
        z = np.zeros((n, W32.shape[1]), np.float32)
        for k in range(K):
            z = _fma32(X32[:, k:k + 1], W32[k][None, :], z)
    z = (z + np.asarray(a["d1b"], np.float32)).astype(np.float32)
    sc, sh = fold32(a)
    y = _fma32(z, sc, sh)
    h = np.maximum(y, np.float32(0))
    W2 = np.asarray(a["d2w"], np.float32)
    C = W2.shape[1]
    lanes = np.zeros((n, 32, C), np.float32)
    for i in range(K // 32):
        k = np.arange(32) + 32 * i
        lanes = _fma32(h[:, k, None], W2[k][None, :, :], lanes)
    for off in (16, 8, 4, 2, 1):
        lanes = (lanes + lanes[:, np.arange(32) ^ off]).astype(np.float32)
    logits = (lanes[:, 0] + np.asarray(a["d2b"], np.float32)).astype(np.float32)
    return dict(z=z, y=y, h=h, logits=logits)


def forward(p, X, labels, cw, mask):
    """Training-mode forward: (loss, cache).  p: d1w, d1b, bn1g, bn1b, d2w, d2b; mask bool [B, 512]."""
    f = {k: np.asarray(v, np.float64) for k, v in p.items()}
    X = np.asarray(X, np.float64)
    B = X.shape[0]
    z = X @ f["d1w"] + f["d1b"]
    mu = z.mean(0)
    var = ((z - mu) ** 2).mean(0)
    inv = 1.0 / np.sqrt(var + EPS_BN)
    xh = (z - mu) * inv
    y = f["bn1g"] * xh + f["bn1b"]
    h = np.maximum(y, 0) * mask / KEEP
    logits = h @ f["d2w"] + f["d2b"]
    nll, g_logits = xent(logits, labels)
    w = np.asarray(cw, np.float64)[labels]
    loss = float((w * nll).sum() / B)
    return loss, dict(X=X, z=z, mu=mu, var=var, inv=inv, xh=xh, y=y, h=h, logits=logits, nll=nll, g_logits=g_logits, w=w,
                      labels=labels, mask=mask, f=f)


def backward(c):
    """Gradients of the loss with respect to d1w, d1b, bn1g, bn1b, d2w, d2b."""
    B = c["X"].shape[0]
    dz2 = c["w"][:, None] * c["g_logits"] / B
    g = {"d2w": c["h"].T @ dz2, "d2b": dz2.sum(0)}
    dh = dz2 @ c["f"]["d2w"].T
    dy = dh * c["mask"] / KEEP * (c["y"] > 0)
    g["bn1b"] = dy.sum(0)
    g["bn1g"] = (dy * c["xh"]).sum(0)
    dz = c["f"]["bn1g"] * c["inv"] * (dy - g["bn1b"] / B - c["xh"] * g["bn1g"] / B)
    g["d1b"] = dz.sum(0)
    g["d1w"] = c["X"].T @ dz
    return g


def adam(p, g, m, v, t: int, lr: float = 1e-3, b1: float = 0.9, b2: float = 0.999, eps: float = 1e-7):
    """One Keras 3 Adam update in fp64: returns (p, m, v)."""
    p, g, m, v = (np.asarray(x, np.float64) for x in (p, g, m, v))
    m = m + (g - m) * (1 - b1)
    v = v + (g * g - v) * (1 - b2)
    alpha = lr * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
    return p - (m * alpha) / (np.sqrt(v) + eps), m, v


def moving(mean, var, mu, var_b):
    return 0.99 * np.asarray(mean, np.float64) + 0.01 * mu, 0.99 * np.asarray(var, np.float64) + 0.01 * var_b


def random_head(C: int, seed: int):
    """A head with non-trivial values in every array (float32), for the inference and training tests."""
    from genomad_b200 import weights as W
    a = W.initial_head(C, seed)
    rng = np.random.default_rng(seed + 1000)
    a["d1b"] = rng.normal(0, 0.1, 512).astype(np.float32)
    a["bn1g"] = rng.uniform(0.5, 1.5, 512).astype(np.float32)
    a["bn1b"] = rng.normal(0, 0.1, 512).astype(np.float32)
    a["bn1m"] = rng.normal(0, 0.2, 512).astype(np.float32)
    a["bn1v"] = rng.uniform(0.5, 2.0, 512).astype(np.float32)
    a["d2b"] = rng.normal(0, 0.1, C).astype(np.float32)
    return a


def bn_regime_head(X, C: int, seed: int, ratio: float = 1.0, var=None, gamma_log2=(0.0, 0.0), spread: float = 4.0):
    """random_head with BN statistics of a chosen regime that still fit the data X [n, 512]: per unit, moving variance `var`
    (uniform in [0.5, 2] when None), moving mean = ratio * sqrt(var + 1e-3) with a random sign, gamma = +-2^t with t spread
    evenly over gamma_log2.  Each dense_1 column is scaled by a power of two so that z's spread over X is about
    sqrt(var + 1e-3), and b1 puts z's mean at the moving mean, so the normalised values are O(1) as after real training and
    the fold cancels |mean * inv| ~ ratio |gamma|.  dense_2 is scaled by a power of two so the logits spread over ~`spread`."""
    a = random_head(C, seed)
    rng = np.random.default_rng(seed + 2000)
    z0 = np.asarray(X, np.float64) @ a["d1w"].astype(np.float64)
    mu_d, sd_d = z0.mean(0), np.maximum(z0.std(0), 1e-30)
    v = rng.uniform(0.5, 2.0, 512) if var is None else np.full(512, float(var))
    std = np.sqrt(v + EPS_BN)
    e = np.round(np.log2(std / sd_d))
    a["d1w"] = (a["d1w"] * np.exp2(e)[None, :].astype(np.float32)).astype(np.float32)
    m = ratio * std * rng.choice([-1.0, 1.0], 512)
    a["d1b"] = (m - mu_d * np.exp2(e)).astype(np.float32)
    a["bn1m"], a["bn1v"] = m.astype(np.float32), v.astype(np.float32)
    t = rng.permutation(np.linspace(gamma_log2[0], gamma_log2[1], 512))
    a["bn1g"] = (np.exp2(t) * rng.choice([-1.0, 1.0], 512)).astype(np.float32)
    l = folded(a, X)["logits"]
    k = np.round(np.log2(spread / max(float(l.std(0).mean()), 1e-30)))
    a["d2w"] = (a["d2w"] * np.float32(2.0 ** k)).astype(np.float32)
    a["d2b"] = (a["d2b"] * np.float32(2.0 ** k)).astype(np.float32)
    return a


def sharpen(a, k: int):
    """d2w and d2b times 2^k: every logit is multiplied by 2^k exactly, in fp32 as in fp64 (h does not change)."""
    out = dict(a)
    out["d2w"] = (a["d2w"] * np.float32(2.0 ** k)).astype(np.float32)
    out["d2b"] = (a["d2b"] * np.float32(2.0 ** k)).astype(np.float32)
    return out


def check_probs(logp_ref, dlogp, probs):
    """The assertions of a head's probabilities against folded(): returns (worst |d log p| / bound over classes whose fp64
    probability is a normal fp32 -- per row, [n]) after asserting that
      * no probability is NaN;
      * |log p - log p64| <= dlogp wherever p64 >= 2^-126;
      * p == 0 only where p64 could lie below half the smallest fp32 subnormal (log p64 - dlogp < log 2^-150);
      * the argmax is fp64's wherever the fp64 margin log p_1 - log p_2 exceeds dlogp_1 + dlogp_2 (then the fp32 values are
        ordered too)."""
    p = np.asarray(probs, np.float64)
    assert not np.isnan(p).any(), "a probability is NaN"
    normal = logp_ref >= np.log(2.0 ** -126)
    with np.errstate(divide="ignore"):
        lg = np.log(p)
    ratio = np.where(normal, np.abs(lg - logp_ref) / dlogp, 0.0)
    bad = np.argwhere(ratio > 1)
    assert not len(bad), f"{len(bad)} probabilities off by more than the bound, first row/class {bad[0]}: " \
                         f"log p {lg[tuple(bad[0])]!r}, fp64 {logp_ref[tuple(bad[0])]!r}, bound {dlogp[tuple(bad[0])]:.3e}"
    zero = p == 0
    assert (logp_ref[zero] - dlogp[zero] < np.log(2.0 ** -150)).all(), "a probability of fp32's range came out as 0"
    order = np.argsort(-logp_ref, axis=1)
    r = np.arange(len(p))
    top, second = order[:, 0], order[:, 1]
    margin = logp_ref[r, top] - logp_ref[r, second]
    sure = margin > dlogp[r, top] + dlogp[r, second]
    assert (p[sure].argmax(1) == top[sure]).all(), "argmax differs from fp64 where the margin exceeds the bound"
    return ratio.max(1)
