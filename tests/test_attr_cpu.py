"""
CPU checks of the attribution reference (tests/attr_ref.py) and of the kernels' decomposition of the backward pass, in fp64:
autograd against central finite differences on the one-hot relaxation, the first-row rule on the exact max-pool ties of N runs,
and the NumPy restatement of csrc/attr.cuh against autograd.
"""
import numpy as np
import pytest
import torch

from oracle import igloo_model as M
from oracle import tokenizer as T
import attr_ref as A


@pytest.fixture(scope="module")
def weights(weights_npz):
    w = M.load_npz_weights(weights_npz)
    return {"shipped": w, "synthetic": M.synthetic_igloo_weights(w)}


def _windows(golden_dir):
    g = np.load(golden_dir / "reference_graph_golden.npz")
    rng = np.random.default_rng(11)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    rand = acgt[rng.integers(0, 4, 6000)]
    tail = acgt[rng.integers(0, 4, 6000)].copy()
    tail[3000:] = ord("N")                                          # a 3 kb N tail
    runs = acgt[rng.integers(0, 4, 6000)].copy()
    runs[1000:1400] = ord("N"); runs[4000:4100] = ord("N")
    alln = np.full(6000, ord("N"), dtype=np.uint8)
    asc = np.stack([g["windows"][0], rand, tail, runs, alln])
    return T.tokenize_windows(asc)


@pytest.fixture(scope="module")
def tokens(golden_dir):
    return _windows(golden_dir)


def test_log_probs_onehot_is_the_oracle(weights, tokens):
    for w in weights.values():
        lp = A.log_probs_onehot(A.one_hot(tokens[:2]), w).detach().numpy()
        ref = np.log(M.forward_as_written(tokens[:2], w, torch.float64))
        np.testing.assert_allclose(lp, ref, rtol=0, atol=1e-12)


@pytest.mark.parametrize("variant", ["shipped", "synthetic"])
@pytest.mark.parametrize("window", [1, 0])
def test_autograd_matches_finite_differences(weights, tokens, variant, window):
    """Central differences on x[t, tok[t]] at 48 positions of a window (random ACGT, golden), at positions whose touched
    pools have no near-tie: a perturbation at t reaches y1 at t..t+5 and y3 at t..t+15, i.e. pools t//8 .. t//8 + 2."""
    w = weights[variant]
    tok = tokens[window: window + 1]
    attr = A.attribution(tok, w, 2)[0]
    rts = A.routing(tok, w)
    rng = np.random.default_rng(5 + window)
    cand = rng.permutation(A.L_TOK - 24)[:400] + 8
    gaps0, gaps1 = rts[0][1][0], rts[1][1][0]

    def clear(t):
        lo, hi = t // 8 - 1, min(A.N_POOL, t // 8 + 3)
        return min(gaps0[lo:hi].min(), gaps1[lo:hi].min()) > 1e-6

    pos = np.array([t for t in cand if clear(t)][:48])
    assert len(pos) == 48
    eps = 1e-5
    x = A.one_hot(tok).repeat(2 * len(pos), 1, 1)
    for i, t in enumerate(pos):
        x[2 * i, t, tok[0, t]] += eps
        x[2 * i + 1, t, tok[0, t]] -= eps
    with torch.no_grad():
        lp = A.log_probs_onehot(x, w)[:, 2].numpy()
    fd = (lp[0::2] - lp[1::2]) / (2 * eps)
    scale = np.abs(attr).max()
    err = np.abs(fd - attr[pos]).max() / scale
    print(f"\n{variant} window {window}: finite differences vs autograd at {len(pos)} positions: {err:.1e} of max |attr|")
    assert err < 1e-6


def test_ties_in_n_runs_route_to_the_first_row(weights, tokens):
    """All-N window and a 3 kb N tail: every pool inside the run is an exact tie, and autograd sends the gradient to row 0."""
    w = weights["shipped"]
    tok = tokens[[4, 2]]
    routes = A.routing(tok, w)
    for s in (0, 1):
        r, gap, _ = routes[s]
        inner = np.s_[:, 3000 // 8 + 4:, :]                       # pools well inside the tail (window 2) / all-N (window 4)
        assert np.all(gap[0][8:] == 0) and np.all(gap[1][3000 // 8 + 4:] == 0)
        assert np.all(r[inner] == 0)
    # autograd's max_pool1d routing is the explicit first-row routing: same attributions bit for bit
    a_default = A.attribution(tok, w, 1)
    a_routed = A.attribution(tok, w, 1, routes=[routes[0][0], routes[1][0]])
    assert np.array_equal(a_default, a_routed)
    # and a different routing inside the ties changes the result, so the rule is observable
    other = [routes[0][0].copy(), routes[1][0].copy()]
    other[1][1, 3000 // 8 + 4:, :] = 7
    assert not np.array_equal(A.attribution(tok[1:], w, 1, routes=[other[0][1:], other[1][1:]]), a_default[1:])


@pytest.mark.parametrize("variant", ["shipped", "synthetic"])
def test_decomposition_matches_autograd(weights, tokens, variant):
    w = weights[variant]
    rng = np.random.default_rng(2)
    rand_tok = rng.integers(0, 257, (1, A.L_TOK))
    for tok, target in ((tokens[[0, 2]], 0), (tokens[[3, 4]], 2), (rand_tok, 1)):
        ref = A.attribution(tok, w, target)
        got = A.decomposed(tok, w, target)
        err = np.abs(got - ref).max(axis=1) / np.abs(ref).max(axis=1)
        assert err.max() < 1e-12, err


def test_joined_row_sign_is_the_hi16_sign():
    """The kernels take lrelu' from the sign of a row's hi16 plane; the GPU tests read the LeakyReLU branches of the forward
    from the joined rows gnm_debug_fetch returns ((hi16 + lo16) / 32, or (hi16 + lo8 / 128) / 32 for conv2's output).  The two
    predicates are the same: lo is the rounded remainder Y - hi16, so hi16 > 0 gives a positive sum, and hi16 = +-0 means
    |Y| rounded to zero in fp16 (|Y| <= 2^-25), where the remainder rounds to zero too (in fp16, and in e4m3 after the 2^7
    scale: 2^-18 is below its smallest subnormal 2^-9)."""
    rng = np.random.default_rng(3)
    Y = np.concatenate([rng.standard_normal(200000) * 10.0 ** rng.uniform(-12, 2, 200000),
                        [0.0, -0.0, 2.0 ** -25, -2.0 ** -25, 2.0 ** -24, 2.0 ** -26, 3e-8, -3e-8]]).astype(np.float32)
    hi = Y.astype(np.float16).astype(np.float32)
    lo16 = (Y - hi).astype(np.float16).astype(np.float32)
    lo8 = torch.from_numpy((Y - hi) * 128.0).to(torch.float8_e4m3fn).to(torch.float32).numpy() / 128.0
    assert np.array_equal((hi + lo16) > 0, hi > 0)
    assert np.array_equal((hi + lo8) > 0, hi > 0)
