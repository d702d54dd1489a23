"""
CPU checks of the first step of the attribution pass, the head's g_logits = e_c - p from the forward's float32 probabilities
(attr_head_backward_kernel, restated by tests/attr_ref.py head_gradient_fp32), and of the fp64 reference where p_c saturates.
When the window is classified confidently as the target, 1 - p_c cancels in float32 (values just below 1 are 2^-24 apart) and
is exactly 0 once p_c rounds to 1.0f; the kernel takes the target's component as the sum of the other two probabilities.
"""
import numpy as np
import pytest
import torch

from oracle import igloo_model as M
from oracle import tokenizer as T
import attr_ref as A

ULP = 2.0 ** -24
FP32_NORMAL = 2.0 ** -126


def _sweep(target, n=4001, seed=0):
    """float32 logit triples with log-odds margin mu = l_c - max_{i != c} l_i from -120 to 120, the third logit 0..30 below
    the second and a common shift.  All values are multiples of 2^-12 below 2^9, so every difference the softmax forms is
    exact in float32 and the sweep measures the head formula, not the rounding of its input."""
    rng = np.random.default_rng(seed + target)
    q = lambda v: np.round(v * 4096.0) / 4096.0                     # noqa: E731
    mu = q(np.linspace(-120.0, 120.0, n))
    gap = q(rng.uniform(0.0, 30.0, n))
    shift = q(rng.uniform(-20.0, 20.0, n))
    o = [i for i in range(3) if i != target]
    lg = np.empty((n, 3))
    lg[:, target] = shift + mu
    lg[:, o[0]] = shift
    lg[:, o[1]] = shift - gap
    lg[n // 2:, [o[0], o[1]]] = lg[n // 2:, [o[1], o[0]]]           # either off-target class the larger one
    lg32 = lg.astype(np.float32)
    assert np.array_equal(lg32.astype(np.float64), lg)
    return lg32, mu


@pytest.mark.parametrize("target", [0, 1, 2])
def test_head_gradient_fp32_over_the_margin_sweep(target):
    lg32, mu = _sweep(target)
    ref = A.head_gradient_fp64(lg32.astype(np.float64), target)
    got = A.head_gradient_fp32(lg32, target).astype(np.float64)
    p64 = np.exp(lg32 - lg32.max(axis=1, keepdims=True).astype(np.float64))
    p64 /= p64.sum(axis=1, keepdims=True)
    normal = np.delete(p64, target, axis=1).min(axis=1) >= FP32_NORMAL     # off-target probabilities fp32-normal
    scale = np.abs(ref).max(axis=1)
    err = np.abs(got - ref).max(axis=1) / scale
    assert normal[mu > 0].any() and normal[mu < 0].any() and (mu[normal] > 60).any()
    print(f"\ntarget {target}: fixed head formula {err[normal].max() / ULP:.2f} ulp of max |g| over {normal.sum()} triples "
          f"(mu {mu[normal].min():.0f} .. {mu[normal].max():.0f})")
    assert err[normal].max() <= 6 * ULP                                      # exp, sum, reciprocal, product, sum
    assert np.all(np.isfinite(got))
    # e_c - p from the same float32 probabilities: cancels, so the sweep reaches the regime the formula is for
    p32 = A.softmax_fp32(lg32).astype(np.float64)
    old = np.eye(3)[target] - p32
    err_old = np.abs(old - ref).max(axis=1) / scale
    print(f"target {target}: e_c - p: worst {err_old[normal].max():.2e}; first mu above 1e-4: "
          f"{mu[normal & (err_old > 1e-4)].min():.1f}")
    assert err_old[normal].max() > 1e-4
    # off-target probabilities all round to 0 from mu ~ 104 on: the gradient is exactly 0, not NaN
    dead = mu >= 110
    assert dead.any() and np.all(got[dead] == 0)


def test_log_p_target_gradient_keeps_precision_at_saturation():
    """the fp64 reference's log p_c: its gradient is e_c - softmax with every component to fp64 relative precision, for
    margins far past the point where p_c == 1.0 in fp64 (mu ~ 37), and log_softmax's below the argmax"""
    rng = np.random.default_rng(4)
    for target in range(3):
        n = 2001
        lg = rng.uniform(-5.0, 5.0, (n, 3))
        o = [i for i in range(3) if i != target]
        lg[:, target] = lg[:, o].max(axis=1) + np.linspace(-600.0, 600.0, n)
        x = torch.tensor(lg, dtype=torch.float64, requires_grad=True)
        (g,) = torch.autograd.grad(A.log_p_target(x, target).sum(), x)
        ref = A.head_gradient_fp64(lg, target)
        err = np.abs(g.numpy() - ref) / np.maximum(np.abs(ref), 1e-300)
        assert np.all(np.isfinite(g.numpy()))
        assert err.max() <= 1e-13, err.max()


@pytest.fixture(scope="module")
def weights(weights_npz):
    w = M.load_npz_weights(weights_npz)
    return {"shipped": w, "synthetic": M.synthetic_igloo_weights(w)}


@pytest.fixture(scope="module")
def golden_tokens(golden_dir):
    return T.tokenize_windows(np.load(golden_dir / "reference_graph_golden.npz")["windows"])


# golden windows classified confidently as the target: (weights, row, target, log-odds margin)
CONFIDENT = [("shipped", 16, 2, 9.1), ("shipped", 21, 1, 12.1), ("synthetic", 21, 1, 20.3)]


@pytest.mark.parametrize("variant,row,target,mu", CONFIDENT)
def test_head_gradient_from_fp32_probabilities_on_confident_windows(weights, golden_tokens, variant, row, target, mu):
    """The backward as the kernels decompose it, with the head's gradient taken from the float32-rounded fp64 probabilities:
    the kernel's formula stays within 1e-6 of autograd, e_c - fl32(p) does not stay within 1e-4."""
    w = weights[variant]
    tok = golden_tokens[row: row + 1]
    with torch.no_grad():
        _, it = M.forward(tok, w, torch.float64, return_intermediates=True)
        lg = M.head(it["h0"], w, torch.float64, return_logits=True).numpy()
    assert abs(lg[0, target] - np.delete(lg[0], target).max() - mu) < 0.05
    p32 = (np.exp(lg - lg.max()) / np.exp(lg - lg.max()).sum()).astype(np.float32)
    ref = A.attribution(tok, w, target)
    scale = np.abs(ref).max()
    fixed = A.decomposed(tok, w, target, g_logits=A.head_gradient_from_probs32(p32, target))
    old = A.decomposed(tok, w, target, g_logits=np.eye(3)[target] - p32.astype(np.float64))
    e_fixed, e_old = np.abs(fixed - ref).max() / scale, np.abs(old - ref).max() / scale
    print(f"\n{variant} row {row} target {target} (p_c = {p32[0, target]!r}): sum of the others {e_fixed:.1e}, "
          f"e_c - p {e_old:.1e}")
    assert e_fixed <= 1e-6
    assert e_old > 1e-4


def test_reference_at_given_logits(weights, golden_tokens):
    """attribution(logits_at=) evaluates log p_c at the given logits and keeps the model's derivatives of the logits: at the
    model's own fp64 logits it is the plain reference bit for bit, and at logits whose log-odds are moved by ~1e-4 (an fp32
    forward's error on these windows) it is the decomposition with that head gradient.  On row 16, classified confidently as
    virus (mu 9.1), the attributions move by about as much as the log-odds; on row 21 (virus at mu -12.1) they hardly move."""
    w = weights["shipped"]
    tok = golden_tokens[[16, 21]]
    with torch.no_grad():
        _, it = M.forward(tok, w, torch.float64, return_intermediates=True)
        lg = M.head(it["h0"], w, torch.float64, return_logits=True).numpy()
    ref = A.attribution(tok, w, 2)
    assert np.array_equal(A.attribution(tok, w, 2, logits_at=lg), ref)
    moved = lg + np.array([[1e-4, -1e-4, 0.0], [0.0, 2e-4, -1e-4]])
    got = A.attribution(tok, w, 2, logits_at=moved)
    dec = A.decomposed(tok, w, 2, g_logits=A.head_gradient_fp64(moved, 2))
    scale = np.abs(got).max(axis=1)
    assert (np.abs(dec - got).max(axis=1) / scale).max() < 1e-12
    shift = np.abs(got - ref).max(axis=1) / scale
    assert 5e-5 < shift[0] < 2e-4 and shift[1] < 1e-6, shift


def test_reference_keeps_the_gradient_where_p_is_one_in_fp64(weights, golden_tokens):
    """Head-sharpened weights (d2w, d2b times 4: every logit times 4 exactly) on shipped row 21: margin ~48, p_c == 1.0 even
    in fp64.  Autograd through log_p_target still matches the decomposition (with the fp64 head gradient) to 1e-12."""
    w = dict(weights["shipped"])
    w["d2w"], w["d2b"] = w["d2w"] * np.float32(4), w["d2b"] * np.float32(4)
    tok = golden_tokens[21:22]
    assert M.forward(tok, w, torch.float64)[0, 1] == 1.0
    ref = A.attribution(tok, w, 1)
    got = A.decomposed(tok, w, 1)
    assert np.abs(ref).max() > 0
    assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-12
