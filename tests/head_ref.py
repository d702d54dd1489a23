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
