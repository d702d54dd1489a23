"""
CPU tests of integrated gradients' definition and fp64 reference (tests/ig_ref.py), no GPU:
- the kernel's interpolated layer-1 formula (encode.cuh), restated in NumPy, against the oracle's Conv1D #1 on the relaxed
  one-hot input x' + alpha (x - x'), for both baselines;
- S_base of the N baseline is the all-N window's layer-1 pre-activation, and alpha = 1 is the window's own;
- N-baseline IG is 0 at token-0 positions, and IG rows are the one-hot gradient at the node;
- the fp64 completeness gap at the largest m of the convergence study, on a golden window the study did not use, stays
  within a bound derived from the study's recorded gaps (profiles/integrated_gradients_h100.json);
- no spills in the new kernels (ptxas report of the library build).
"""
import json
import re
from pathlib import Path

import numpy as np
import pytest
import torch

import attr_ref as A
import ig_ref as I
from oracle import igloo_model as M
from oracle import tokenizer as T

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def w(weights_npz):
    return M.load_npz_weights(weights_npz)


@pytest.fixture(scope="module")
def tok_all(golden_dir):
    return T.tokenize_windows(np.load(golden_dir / "reference_graph_golden.npz")["windows"])


@pytest.fixture(scope="module")
def tok(golden_dir):
    asc = np.load(golden_dir / "reference_graph_golden.npz")["windows"][:2].copy()
    asc[1, 1000:1700] = ord("N")
    asc[1, 5000] = ord("R")
    return T.tokenize_windows(asc)


@pytest.mark.parametrize("baseline", I.BASELINES)
def test_layer1_formula_is_conv1_on_the_interpolated_input(w, tok, baseline):
    al = np.array([0.0, 0.3125, 0.9, 1.0])
    t = np.repeat(tok[1:], len(al), axis=0)
    x = I.interp_onehot(t, al, baseline)
    ref = I.conv1_preact(x, w)
    got = I.layer1_preact(t, w, al, baseline)
    scale = np.abs(ref).max()
    assert np.abs(got - ref).max() <= 1e-12 * scale


def test_base_sum_is_the_all_n_window(w, tok):
    alln = np.zeros_like(tok[:1])                                       # token 0 everywhere
    s_base_n = I.layer1_preact(tok[:1], w, np.zeros(1), "N")             # alpha 0: b1 + S_base
    own = I.layer1_preact(alln, w, np.ones(1), "zero")                  # the all-N window's own pre-activation
    assert np.array_equal(s_base_n, own)
    assert np.array_equal(I.layer1_preact(tok, w, np.ones(2), "N"), I.layer1_preact(tok, w, np.ones(2), "zero"))
    zero = I.layer1_preact(tok[:1], w, np.zeros(1), "zero")
    assert np.array_equal(zero, np.broadcast_to(np.asarray(w["c1b"], np.float64), zero.shape))


def test_rows_are_the_gradient_at_the_node(w, tok):
    """At alpha = 1 a zero-baseline row is gradient x input (attr_ref.attribution); an N-baseline row at any node is
    g[t, tok] - g[t, 0] of the full autograd gradient of log p_c there."""
    target = 2
    lg, J = I.logit_jacobian(tok, w, np.ones(2), "zero")
    row = I.rows_from_jacobian(lg, J, target)
    ref = A.attribution(tok, w, target)
    assert np.abs(row - ref).max() <= 1e-12 * np.abs(ref).max()
    lg, J = I.logit_jacobian(tok[1:], w, np.array([0.4]), "N")
    row = I.rows_from_jacobian(lg, J, target)[0]
    x = I.interp_onehot(tok[1:], np.array([0.4]), "N").requires_grad_(True)
    (g,) = torch.autograd.grad(A.log_p_target(A.logits_onehot(x, w), target).sum(), x)
    g = g[0].numpy()
    t1 = tok[1].astype(np.int64)
    ref = np.where(t1 == 0, 0.0, g[np.arange(len(t1)), t1] - g[:, 0])
    assert np.abs(row - ref).max() <= 1e-12 * np.abs(ref).max()


def test_n_baseline_is_zero_at_token_0(w, tok):
    ig, rows = I.integrated_gradients(tok[1:], w, 1, 2, "N")
    assert np.any(tok[1] == 0)
    assert np.all(ig[0][tok[1] == 0] == 0) and np.all(rows[0][:, tok[1] == 0] == 0)
    assert np.abs(ig[0][tok[1] != 0]).max() > 0


HELD_OUT = 2                  # a golden window the convergence study did not use
MARGIN = 2.0                  # the study's worst gap, times this, is the bound for a window outside the study


def test_completeness_within_recorded_bound(w, tok_all):
    """The fp64 gap |sum IG - (log p(x) - log p(x'))| at the largest m of the convergence study, on a golden window the study
    did not use (shipped weights, every target, both baselines), stays within MARGIN x the worst gap the study recorded for
    the unsharpened weight sets at that m (profiles/integrated_gradients_h100.json, the raw output of
    tools/ig_convergence.py).  The bound is derived here from the recorded cases, not stored."""
    conv = json.loads((ROOT / "profiles" / "integrated_gradients_h100.json").read_text())["convergence"]
    assert HELD_OUT not in conv["rows"]
    m = max(conv["steps"])
    t0 = tok_all[HELD_OUT: HELD_OUT + 1]
    for baseline in I.BASELINES:
        bound = MARGIN * max(c["gap"] for c in conv["cases"] if c["k"] == 1 and c["steps"] == m and c["baseline"] == baseline)
        lx, lb = I.endpoint_logits(t0, w, baseline)
        lg, J = I.logit_jacobian(np.repeat(t0, m, axis=0), w, I.alphas(m), baseline)
        for target in range(3):
            ig_sum = I.rows_from_jacobian(lg, J, target).mean(axis=0).sum()
            gap = abs(ig_sum - (I.log_p(lx, target) - I.log_p(lb[None], target)[0])[0])
            print(f"\n{baseline} target {target}: fp64 gap at m = {m}: {gap:.2e} (bound {bound:.2e})")
            assert gap <= bound, (baseline, target)


KERNELS = ["_ZN3gnm21embed_conv1_ig_kernelEPKhPKfS3_S3_PhiiPNS_12DeviceStatusE",
           "_ZN3gnm16layer1_ig_kernelEPKhPKfS3_S3_iiPf",
           "_ZN3gnm16ig_reduce_kernelEPKfiPf",
           "_ZN3gnm14ig_logp_kernelEPKfiiiPf"]


@pytest.mark.parametrize("mangled", KERNELS)
def test_ig_kernels_do_not_spill(mangled):
    from genomad_b200 import build as B
    B.build()
    log = (B.PKG / "build.log").read_text()
    m = re.search(r"Function properties for " + re.escape(mangled) + r"\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads", log)
    assert m, f"no ptxas resource report for {mangled} in build.log"
    assert tuple(map(int, m.groups())) == (0, 0, 0), mangled
