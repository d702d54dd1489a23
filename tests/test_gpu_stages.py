"""
Stage-by-stage precision of the CUDA path (run with `-m gpu -s` on an H100 for the tables).

Each stage's output, fetched with gnm_debug_fetch, is compared with an fp64 CPU evaluation of that stage on the kernel's OWN input
(tests/stage_ref.py), so what is measured is that kernel's error alone, and is held to the bars that tests/test_stage_recipes.py
derives from an emulation of each recipe and its mutants.  Stops: debug_stop = 2 leaves y1 in buf0 and y2 in buf1 (and q0, mpi0),
debug_stop = 3 leaves y3 in buf0, a full step leaves q1, mpi1, the logits of IGLOO#1, h0, h1, h2 and the probabilities.

The matrix: shipped weights, synthetic O(1) IGLOO weights, a set whose three conv layers reach |y| ~ 3.2 (the top of the range
the activation planes support), conv3 and w_v weight-scale sweeps (2^-8 .. 2^2) and weights on both sides of the conv operand
scaling rule's switch points; batches of 1, 7, 9 and 24 windows (max_batch 9: not a multiple of the fused IGLOO kernel's 8-window groups); the
tensor-core path and the fp32 validation kernels (conv_impl), fused and separate patch gather (fuse_gather) and layer 1 (fuse_l1).
"""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import stage_ref as R
from oracle import igloo_model as M
from oracle import tokenizer as T

pytestmark = pytest.mark.gpu


def _windows(n, seed):
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tools"))
    import precision_study
    return precision_study.make_windows(n, seed)


@pytest.fixture(scope="module")
def shipped(weights_npz):
    return M.load_npz_weights(weights_npz)


def _scaled(w, **factors):
    out = dict(w)
    for k, f in factors.items():
        out[k] = (np.asarray(w[k], np.float64) * f).astype(np.float32)
    return out


def _fetch(w, a, max_batch, opts, stops=(2, 3, 0)):
    """Run the windows through a fresh handle with the given options; the fetched buffers as fp64 CPU tensors."""
    from genomad_b200 import engine
    n = len(a)
    c = engine.Classifier(w, device=0, max_batch=max_batch)
    got = {}
    try:
        for k, v in opts.items():
            c.set_option(k, v)
        da = torch.from_numpy(a).cuda()
        for stop in stops:
            c.set_option("debug_stop", stop)
            probs = c.predict_ascii(da)
            c.check_status()

            def f(name):
                return c.debug_fetch(name, n).double().cpu()
            if stop == 2:
                got.update(y1=f("buf0"), y2=f("buf1"), q0=f("q0"), mpi0=f("mpi0"))
            elif stop == 3:
                got.update(y2_3=f("buf1"), y3=f("buf0"))
            else:
                got.update(y3_0=f("buf0"), q1=f("q1"), mpi1=f("mpi1"), logits=f("logits")[:, :R.N_POOL], h0=f("h0"),
                           h1=f("h1"), h2=f("h2"), probs=probs.double().cpu())
    finally:
        c.close()
    return got


def _check(label, w, a, got, conv_impl=0, tokens=None, regions=None, rows=None):
    """Every stage present in `got` against its bar; prints one table row per stage, returns the misses.  tokens: layer 1's
    input when it is not the tokenization of the windows `a`; regions: (positions, pooled positions) region sets of
    R.position_regions when `got` holds a sample of a larger batch; rows: window regions (R.position_regions' "win ..."
    entries) for the stages with one row per window (mpi, logits1, h0, h1, h2, probs).  `got` may hold the tail alone (q0, mpi0,
    q1, mpi1 and the tail buffers, no activations): the tail stages are then checked on their own inputs."""
    n = len(a)
    reg, preg = regions or (R.position_regions(n), R.position_regions(n, pooled=True))
    rows = rows or {}
    conv_bar = "conv_fp32" if conv_impl else "conv_tc"
    checks = []
    if "y1" in got:
        checks += [("y1", "y1", got["y1"], R.conv1(T.tokenize_windows(a) if tokens is None else tokens, w), reg),
                   ("y2 (conv2)", conv_bar, got["y2"], R.conv(got["y1"], w["c2w"], w["c2b"]), reg),
                   ("q0 (w_v#0)", "wv", got["q0"], R.wv_pool(got["y1"], w["ig0_w_v"]), preg),
                   ("mpi0", "gather", got["mpi0"], R.gather(got["y1"], w, 0), rows)]
    if "y3" in got:
        checks += [("y3 (conv3)", conv_bar, got["y3"], R.conv(got["y2_3"], w["c3w"], w["c3b"]), reg)]
        if "y2" in got:
            assert torch.equal(got["y2"], got["y2_3"]), "conv2 is not deterministic across steps"
    if "q1" in got and "y3" in got:
        assert torch.equal(got["y3"], got["y3_0"]), "conv3 is not deterministic across steps"
        checks += [("q1 (w_v#1)", "wv", got["q1"], R.wv_pool(got["y3"], w["ig1_w_v"]), preg),
                   ("mpi1", "gather", got["mpi1"], R.gather(got["y3"], w, 1), rows)]
    if "h1" in got:
        logits0 = got["mpi0"] @ torch.as_tensor(w["ig0_w_qk"], dtype=R.D)        # not fetchable: fp64 from the kernel's mpi0
        checks += [("logits1", "tf32x3", got["logits"], R.matmul(got["mpi1"], w["ig1_w_qk"]), rows),
                   ("h0[:128]", "attention", got["h0"][:, :128], R.attention(logits0, got["q0"]), rows),
                   ("h0[128:]", "attention", got["h0"][:, 128:], R.attention(got["logits"], got["q1"]), rows),
                   ("h1 (dense0)", "tf32x3", got["h1"], R.dense_bn_relu(got["h0"], w, 0), rows),
                   ("h2 (dense1)", "tf32x3", got["h2"], R.dense_bn_relu(got["h1"], w, 1), rows),
                   ("probs", "probs", got["probs"], R.head_softmax(got["h2"], w), rows)]
    bad = []
    for stage, key, g, ref, regions in checks:
        if float(ref.s_abs.max()) < 1e-20:
            # the shipped patch / attention weights (~1e-32): mpi and the logits sit below fp32's normal range, numerically dead
            print(f"| {label} | {stage} | skipped (dead weights: sum |terms| < 1e-20) | | | | | |")
            continue
        m = R.metrics(g, ref, regions)
        rms_bar, max_bar = R.BARS[key]
        ok = m["rms"] <= rms_bar and m["max"] <= max_bar
        per_region = ", ".join(f"{k[4:]} {v:.1e}" for k, v in m.items() if k.startswith("max ")) or "-"
        print(f"| {label} | {stage} | {m['rms']:.2e} | {rms_bar:.0e} | {m['max']:.2e} | {max_bar:.1e} | {per_region} | "
              f"{'ok' if ok else 'MISS'} |")
        if not ok:
            bad.append((label, stage, m))
    return bad


HEADER = ("\n| configuration | stage | rms err / rms scale | bar | max err / sum abs terms | bar | max per region | |"
          "\n|---|---|---|---|---|---|---|---|")


# ------------------------------------------------------------------------------------------ shipped / synthetic weights x paths
PATHS = {"tc fused (default)": ({}, 0), "tc fuse_l1": ({"fuse_l1": 1}, 0), "tc fuse_gather=0": ({"fuse_gather": 0}, 0),
         "fp32 validation (conv_impl=1)": ({"conv_impl": 1}, 1)}


@pytest.mark.parametrize("weights", ["shipped", "synthetic"])
@pytest.mark.parametrize("path", list(PATHS))
def test_stages_24_windows(shipped, weights, path):
    w = shipped if weights == "shipped" else M.synthetic_igloo_weights(shipped)
    opts, impl = PATHS[path]
    a = _windows(24, seed=5)
    print(HEADER)
    assert not _check(f"{weights}, n=24, {path}", w, a, _fetch(w, a, 24, opts), impl)


@pytest.mark.parametrize("n", [1, 7, 9])
def test_stages_small_batches(shipped, n):
    """max_batch 9: the last 8-window group of the fused IGLOO kernel is partial; n = 1 and 7 leave one group partly empty."""
    w = M.synthetic_igloo_weights(shipped)
    a = _windows(9, seed=13)[:n]
    print(HEADER)
    bad = []
    for path in ("tc fused (default)", "tc fuse_gather=0", "tc fuse_l1"):
        bad += _check(f"synthetic, n={n}, max_batch=9, {path}", w, a, _fetch(w, a, 9, PATHS[path][0]))
    assert not bad


# ------------------------------------------------------------------------------------------ range edge
def test_stages_at_the_top_of_the_activation_range(shipped):
    """conv1, conv2 and conv3 weights and biases scaled (LeakyReLU is positively homogeneous, so each layer's output scales
    exactly) until every layer's max |y| is ~3.2 on the test windows: the hi8 plane is near its e4m3 limit (|y| = 3.5)."""
    a = _windows(16, seed=29)
    base = M.synthetic_igloo_weights(shipped)
    _, it = M.forward(T.tokenize_windows(a), base, torch.float32, return_intermediates=True)
    g1, g2, g3 = (3.2 / float(it[k].abs().max()) for k in ("y1", "y2", "y3"))
    w = _scaled(base, c1w=g1, c1b=g1, c2w=g2 / g1, c2b=g2, c3w=g3 / g2, c3b=g3)
    got = _fetch(w, a, 16, {})
    assert 3.0 < float(got["y1"].abs().max()) < 3.5 and 3.0 < float(got["y2"].abs().max()) < 3.5
    print(HEADER)
    assert not _check("range edge |y| ~ 3.2", w, a, got)


# ------------------------------------------------------------------------------------------ operand scaling rule
@pytest.mark.parametrize("k", [-8, -6, -4, -2, 0, 1, 2])
def test_conv3_weight_scale_sweep(shipped, k):
    """conv3 weights and bias x 2^k (y3 scales with them; its hi16 + lo16 planes keep the output's precision).  Swept on conv3
    rather than conv2: conv2 writes hi16 + lo8, and a y2 scaled down by 2^k loses precision in its e4m3 lo8 plane on its own,
    whatever the weights, which would hide the operand scaling rule under the output's storage error.  The packing code is the
    same for both layers; conv2's weights are exercised at the rule's switch points below.  With the old
    rule (d <= 16, hi = fp16(W)) conv3 lost its Ahi * Wlo correction for small weights: on an H100 the y3 error was 1.3e-4 at
    k = -8 and 3.8e-5 at k = -6, against 8.4e-6 with the current rule at every k."""
    f = 2.0 ** k
    w = _scaled(M.synthetic_igloo_weights(shipped), c3w=f, c3b=f)
    a = _windows(8, seed=31)
    print(HEADER)
    assert not _check(f"conv3 x 2^{k}", w, a, _fetch(w, a, 8, {}, stops=(2, 3)))


@pytest.mark.parametrize("k", [-8, -6, -4, -2, 0, 2])
def test_wv_weight_scale_sweep(shipped, k):
    """Both IGLOO kernels' w_v x 2^k, through all three w_v paths (fused IGLOO kernel, conv_t_kernel<true>, fused layer 1).
    gnm_create splits w_v * 2^e into its fp16 halves, max |w_v| * 2^e in [2^13, 2^14); unscaled, the lo halves of small
    weights were fp16 subnormals and q lost its Ahi * Wlo correction."""
    w = _scaled(M.synthetic_igloo_weights(shipped), ig0_w_v=2.0 ** k, ig1_w_v=2.0 ** k)
    a = _windows(8, seed=47)
    print(HEADER)
    bad = []
    for path in ("tc fused (default)", "tc fuse_gather=0", "tc fuse_l1"):
        bad += _check(f"w_v x 2^{k}, {path}", w, a, _fetch(w, a, 8, PATHS[path][0]))
    assert not bad


@pytest.mark.parametrize("j", [-2, 0])
@pytest.mark.parametrize("side", [-1, 1])
def test_conv_weights_at_the_scaling_rule_switch(shipped, j, side):
    """max |W| of conv2 and conv3 just below / just above 0.78 * 2^j, where the exponent d of the operand scaling changes."""
    target = 0.78 * 2.0 ** j * (1 + side * 2.0 ** -10)
    w = _scaled(shipped, c2w=target / float(np.abs(shipped["c2w"]).max()), c3w=target / float(np.abs(shipped["c3w"]).max()))
    a = _windows(8, seed=37)
    print(HEADER)
    assert not _check(f"wmax = 0.78 * 2^{j} * (1 {'+' if side > 0 else '-'} 2^-10)", w, a, _fetch(w, a, 8, {}, stops=(2, 3)))


# ------------------------------------------------------------------------------------------ overflow flag per stage
def _y_max(w, a):
    _, it = M.forward(T.tokenize_windows(a), w, torch.float32, return_intermediates=True)
    return float(it["y2"].abs().max()), float(it["y3"].abs().max())


@pytest.mark.parametrize("layer, limit", [("conv2", 3.5), ("conv3", 2047.0)])
def test_overflow_flag_names_the_stage(shipped, layer, limit):
    """Weights and bias of one conv layer scaled so that its max |y| lands 3% above / below the limit of the planes it writes
    (conv2: hi8 = e4m3(4 * 32 y) saturates above 3.5; conv3: fp16(32 y) overflows above 2047).  Above: the library reports
    "activation range exceeded in <layer>"; below: nothing is reported and the stage still meets its bar."""
    from genomad_b200 import engine
    a = _windows(8, seed=43)
    y2max, y3max = _y_max(shipped, a)
    for over in (True, False):
        if layer == "conv2":
            g = limit * (1.03 if over else 0.97) / y2max
            w = _scaled(shipped, c2w=g, c2b=g, c3w=1 / g)
        else:
            g = limit * (1.03 if over else 0.97) / y3max
            w = _scaled(shipped, c3w=g, c3b=g)
        c = engine.Classifier(w, device=0, max_batch=8)
        try:
            c.set_option("debug_stop", 3)
            c.predict_ascii(torch.from_numpy(a).cuda())
            if over:
                with pytest.raises(engine.GnmError, match=f"activation range exceeded in {layer}"):
                    c.check_status()
                continue
            c.check_status()
        finally:
            c.close()
        got = _fetch(w, a, 8, {}, stops=(2, 3))
        print(HEADER)
        assert not _check(f"{layer} max |y| = 0.97 x {limit}", w, a, got)
