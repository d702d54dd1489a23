"""
Arbitrary token input (no GPU): what gnm_forward_tokens must compute for token windows that are not a tokenization, and why
layer 1's triple-table shortcut needs a consistency check there.

The reference model's first op is tf.one_hot(x, depth=257), which takes any integer: a token in [0, 256] selects its row, any
other value gives an all-zero row.  tests/golden/reference_tokens_golden.npz holds the reference graph's outputs
(make_reference_tokens_golden.py) on 16 token windows: random tokens, tokenizations with inconsistent 4-mers (everywhere, or
only at the window start, the 256-position segment seam and the window end) and windows carrying 257 .. 65535.
"""
import numpy as np
import pytest
import torch

import stage_ref as R
from oracle import igloo_model as M
from oracle import tokenizer as T


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(golden_dir / "reference_tokens_golden.npz")


@pytest.fixture(scope="module")
def shipped(weights_npz):
    return M.load_npz_weights(weights_npz)


def test_golden_token_windows_cover_the_cases(golden):
    tok = golden["tokens"].astype(np.int64)
    assert tok.shape == (16, 5997) and golden["tokens"].dtype == np.uint16
    assert np.array_equal(golden["in_range"], (tok <= 256).all(1))
    assert golden["in_range"].sum() >= 8 and (~golden["in_range"]).sum() >= 4
    big = np.unique(tok[tok > 256])
    assert {257, 4096, 32767, 32768, 65535} <= set(big.tolist())


def test_oracle_matches_reference_graph_on_arbitrary_tokens(golden, shipped):
    """The oracle (closed form, fp64 and fp32) against the reference's own model graph, shipped and synthetic IGLOO weights; the
    op-for-op formulation (one-hot tensor -> conv1d) agrees too, on windows with and without out-of-range tokens."""
    tok = golden["tokens"]
    for key, ww in (("shipped", shipped), ("synthetic", M.synthetic_igloo_weights(shipped))):
        o64 = np.concatenate([M.forward(tok[i:i + 8], ww, torch.float64) for i in range(0, 16, 8)])
        o32 = np.concatenate([M.forward(tok[i:i + 8], ww, torch.float32) for i in range(0, 16, 8)])
        d64, d32 = np.abs(o64 - golden[key + "_fp64"]).max(), np.abs(o32 - golden[key]).max()
        print(f"{key}: fp64 max |dp| {d64:.2e}, fp32 max |dp| {d32:.2e}")
        assert d64 <= 1e-11, (key, d64)
        assert d32 <= 5e-5 and np.abs(o32 - golden[key + "_fp64"]).max() <= 5e-5, (key, d32)
        assert np.array_equal(o32.argmax(1), golden[key + "_fp64"].argmax(1))
        pick = [0, 8, 10]                                          # uniform; sprinkled > 256; all 65535
        assert np.abs(M.forward_as_written(tok[pick], ww, torch.float64) - o64[pick]).max() < 1e-12


def test_layer1_matches_reference_graph(golden, shipped):
    """Layer 1 alone: the reference graph's activations after one-hot -> Conv1D -> LeakyReLU (fp64), the oracle's closed form,
    the op-for-op form and the stage reference R.conv1 all agree; a window of 65535s is the bias alone."""
    tok = golden["tokens"]
    pos = golden["l1_pos"]
    t = torch.as_tensor(tok.astype(np.int64))
    y_closed = M.conv1_embedding(t, shipped, torch.float64)
    y_written = M.conv1_as_written(t, shipped, torch.float64)
    ref = R.conv1(tok, shipped)
    g = torch.as_tensor(golden["l1_shipped_fp64"])
    assert float((y_closed[:, pos, ::4] - g).abs().max()) < 1e-13
    assert float((y_written - y_closed).abs().max()) < 1e-13
    assert float((ref.value - y_closed).abs().max()) < 1e-14
    b = torch.as_tensor(shipped["c1b"], dtype=torch.float64)
    assert torch.equal(y_closed[10], torch.where(b > 0, b, 0.1 * b).expand(5997, 128))


# ------------------------------------------------------------------------------------------ layer 1's table rule
def _vocab(tok):
    """The kernels' token handling: int, > 256 -> -1 (a zero row, like the causal padding)."""
    t = np.asarray(tok).astype(np.int64)
    return np.where(t > 256, -1, t)


def _triple_tables(W):
    """A and B "triple" tables exactly as gnm_create builds them (csrc/api.cu): (W[3h][k0] + W[3h+1][k1]) + W[3h+2][k2] in fp32,
    k0 = 1 + (code >> 4), k1 = 1 + ((code >> 2) & 255), k2 = 1 + (code & 255)."""
    code = np.arange(4096)
    k0, k1, k2 = 1 + (code >> 4), 1 + ((code >> 2) & 255), 1 + (code & 255)
    return [(W[3 * h][k0] + W[3 * h + 1][k1]) + W[3 * h + 2][k2] for h in (0, 1)]


def _consistent(t0, t1, t2):
    """The fixed rule: the three tokens are the overlapping 4-mers of one all-ACGT 6-base word."""
    return ((t0 > 0) & (t1 > 0) & (t2 > 0) & (((t0 - 1) & 15) == ((t2 - 1) >> 4))
            & (t1 - 1 == ((((t0 - 1) & 63) << 2) | (((t2 - 1) >> 2) & 3))))


def _outer_only(t0, t1, t2):
    """The rule the kernels used before arbitrary tokens were handled: outer tokens of the half > 0."""
    return (t0 > 0) & (t2 > 0)


def _layer1_preact(tok, W, tri, rule):
    """Emulation of embed_conv1_kernel / layer1_wv_kernel: per position the fp32 sum A + B, each half either its triple row (when
    `rule` says so) or the three-row fallback (row(j0) + row(j0+1)) + row(j0+2); padded / out-of-range taps add 0.
    rule None: always the fallback (the six-row sum).  Returns (pre-activation [n, 5997, 128] fp32, triple hits [n, 5997, 2])."""
    t = _vocab(tok)
    n, L = t.shape
    tp = np.concatenate([np.full((n, 5), -1), t], axis=1)           # tp[:, i + j] = token of tap j at position i
    taps = [tp[:, j:j + L] for j in range(6)]
    Wz = np.concatenate([W, np.zeros((6, 1, W.shape[2]), np.float32)], axis=1)   # index -1 -> the zero row 257

    def row(j, k):
        return Wz[j][np.where(k < 0, 257, k)]
    halves, hits = [], []
    for h in (0, 1):
        a, b, c = taps[3 * h], taps[3 * h + 1], taps[3 * h + 2]
        fb = (row(3 * h, a) + row(3 * h + 1, b)) + row(3 * h + 2, c)
        hit = np.zeros_like(a, dtype=bool) if rule is None else rule(a, b, c)
        code = np.where(hit, ((a - 1) << 4) | ((c - 1) & 15), 0)
        halves.append(np.where(hit[..., None], tri[h][code], fb))
        hits.append(hit)
    return halves[0] + halves[1], np.stack(hits, -1)


def test_layer1_table_rule_is_the_six_row_sum(golden, shipped):
    """The fixed rule gives bitwise the six-row sum on every golden window (in range or not), and on tokenizer output it takes the
    triple rows exactly where the old rule did (the shortcut is kept for real sequences).  The old rule, which looked only at
    the outer tokens of each half, is wrong on arbitrary in-range tokens (the mutant check): it read the row of another 6-base
    word, off by O(0.1) in the pre-activation."""
    W = np.asarray(shipped["c1w"], np.float32)
    tri = _triple_tables(W)
    tok = golden["tokens"]
    six, _ = _layer1_preact(tok, W, tri, None)
    fixed, hit = _layer1_preact(tok, W, tri, _consistent)
    assert np.array_equal(fixed.view(np.uint32), six.view(np.uint32))
    assert hit.any()

    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tools"))
    import precision_study
    tk = T.tokenize_windows(precision_study.make_windows(8, seed=3))
    six_t, _ = _layer1_preact(tk, W, tri, None)
    fixed_t, hit_fixed = _layer1_preact(tk, W, tri, _consistent)
    old_t, hit_old = _layer1_preact(tk, W, tri, _outer_only)
    assert np.array_equal(hit_fixed, hit_old) and hit_fixed.mean() > 0.5
    assert np.array_equal(fixed_t.view(np.uint32), six_t.view(np.uint32))
    assert np.array_equal(old_t.view(np.uint32), six_t.view(np.uint32))

    inr = golden["in_range"]
    old, _ = _layer1_preact(tok[inr], W, tri, _outer_only)
    err = np.abs(old - six[inr]).max(axis=2)                         # per position: max over channels
    kinds = golden["kinds"][inr]
    for k, e in zip(kinds, err):
        print(f"old rule, {k}: max |error| {e.max():.3f}, positions off {np.mean(e > 0):.1%}")
    assert np.median(err[kinds == "uniform [0, 256]"]) > 0.1
    for k in ("tokenization, odd positions random", "tokenization, seams random"):
        assert (err[kinds == k] > 1e-3).any(axis=1).all(), k
    assert (err[kinds == "tokenization, seams random"][:, 20:240] == 0).all()     # consistent away from the seams
