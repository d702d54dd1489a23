"""
Every stage against fp64 at the batch sizes where the kernels' tiles end, and bitwise batch invariance with live IGLOO weights
(run with `-m gpu -s` on an H100 for the tables).

Almost every launch of a step takes its grid from the window count n, and each kernel has its own tile edge: logits_tc_kernel
(the IGLOO logits and both Dense(512) layers) runs ceil(n / 128) M tiles and guards rows past n in its epilogue; the split-K
reducers read partial z at z * n * ldc; wv_gather_kernel works on 8-window groups with a CTA split cached per group count
(api.cu wv_split); conv_t_kernel and layer1_wv_kernel run n * 24 / n * 63 units on persistent CTAs; the fp32 validation path
(conv_impl = 1) switches launch_sgemm from 32-row to 64-row tiles at 64 rows.  The shapes below put a partial tile or group on
each of those edges (tests/test_batch_shapes_cpu.py reads the tile sizes from the sources and checks that they still do):

    n = max_batch   last logits / head M tile   last wv group      paths
    129             1 row (2nd tile)            1 window           default, fuse_gather = 0, fuse_l1 = 1
    200             72 rows                     8 (25 groups)      default, fuse_gather = 0
    383             127 rows                    7 windows          default, fuse_gather = 0, fuse_l1 = 1
    1000            104 rows (8th tile)         8 (125 groups)     default, fuse_gather = 0
    63 / 64 / 65    sgemm 32-row / 64-row tiles                    conv_impl = 1

Synthetic O(1) IGLOO weights throughout: with the shipped ones (~1e-32) mpi and the attention logits underflow and softmax is
uniform, so a wrong or stale row in the logits GEMM or the attention kernel would change no probability.  The tail stages (one
row per window, ~2 MFLOP of fp64 reference each) are checked on every row; the streaming stages (activations, q, mpi) on the
sampled rows of `sample_rows`, fetched on the GPU and indexed there (tests/test_gpu_tokens_batch1024.py).
"""
import sys
import time
from pathlib import Path

import numpy as np
import pytest
import torch

import stage_ref as R
import test_gpu_attr_stages as GA
import test_gpu_ig as GI
import test_gpu_stages as GS
import test_gpu_tokens_batch1024 as GT
from oracle import igloo_model as M
from oracle import tokenizer as T

pytestmark = pytest.mark.gpu

TILE = 128                                   # kLgBM: rows per M tile of logits_tc_kernel
GROUP = 8                                    # kBandWins: windows per group of wv_gather_kernel
TC_SHAPES = (129, 200, 383, 1000)            # max_batch = n, tensor-core path
FUSE_L1_SHAPES = (129, 383)
FFMA_SHAPES = (63, 64, 65)                   # max_batch = n, conv_impl = 1: both sides of launch_sgemm's 64-row switch
MULTI_STEP = ((200, 401), (129, 265), (1000, 1129))      # (max_batch, n): steps 200 200 1, 129 129 7, 1000 129
INVARIANCE_BATCHES = (1, 8, 9, 129, 200, 383, 1000, 1024)
POOL = 1100
SINGLES = (0, 127, 128, 999, 1099)
ATTR_CTX, ATTR_CHUNK = 256, 200
ATTR_SAMPLE = [126, 127, 128, 129, 130, 199]
IG_WINDOWS, IG_STEPS, IG_CHECK = 13, 16, (0, 8, 12)      # 208 rows: window 8's rows are 128-143
TARGET = 2
TC_PATHS = {"tc fused (default)": {}, "tc fuse_gather=0": {"fuse_gather": 0}, "tc fuse_l1": {"fuse_l1": 1}}
FFMA_PATH = ("fp32 validation (conv_impl=1)", {"conv_impl": 1})


def sample_rows(n):
    """The streaming stages' rows of an n-window step: the first window groups, both sides of the first two M tile edges and of
    the last one, and the last window groups."""
    last = (n - 1) // TILE * TILE
    rows = {0, 1, 7, 8, 9, 127, 128, 129, 255, 256, 257, last - 1, last, n - 9, n - 8, n - 2, n - 1}
    return sorted(i for i in rows if 0 <= i < n)


def head_tile(n, conv_impl):
    """Rows per M tile of the head GEMMs: logits_tc_kernel's 128, or launch_sgemm's 32 / 64 on the fp32 validation path."""
    return TILE if not conv_impl else 32 if n < 64 else 64


def paths(n):
    if n in FFMA_SHAPES:
        return [FFMA_PATH]
    return [(p, o) for p, o in TC_PATHS.items() if p != "tc fuse_l1" or n in FUSE_L1_SHAPES]


@pytest.fixture(scope="module", autouse=True)
def _report_cost():
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    GT.STATS["device_used_peak"] = 0
    yield
    print(f"\n{Path(__file__).name}: {time.time() - t0:.0f} s; peak torch allocation "
          f"{torch.cuda.max_memory_allocated() / 2**30:.2f} GiB; peak device memory in use "
          f"{GT.STATS['device_used_peak'] / 2**30:.2f} GiB")


@pytest.fixture(scope="module")
def syn(weights_npz):
    return M.synthetic_igloo_weights(M.load_npz_weights(weights_npz))


@pytest.fixture(scope="module")
def pool():
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tools"))
    import precision_study
    return precision_study.make_windows(max(n for _, n in MULTI_STEP), seed=71)


def _classifier(w, max_batch):
    from genomad_b200 import engine
    return engine.Classifier(w, device=0, max_batch=max_batch)


def _fetch_step(c, m, idx):
    """After a full step of m windows: y2 / y3 and q1 / mpi1 of the rows idx, and q0, mpi0, q1, mpi1 and the tail buffers of
    every row (fp64, host)."""
    ix, every = torch.as_tensor(idx, device="cuda"), torch.arange(m, device="cuda")
    y3 = GT._take(c, "buf0", m, ix)
    samp = dict(y2_3=GT._take(c, "buf1", m, ix), y3=y3, y3_0=y3, q1=GT._take(c, "q1", m, ix), mpi1=GT._take(c, "mpi1", m, ix))
    tail = {k: GT._take(c, k, m, every) for k in ("q0", "mpi0", "q1", "mpi1", "h0", "h1", "h2")}
    tail["logits"] = GT._take(c, "logits", m, every)[:, :R.N_POOL]
    return GT._f64(samp), GT._f64(tail)


def _check_step(label, w, a, samp, tail, idx, conv_impl=0):
    """The streaming stages of the sampled rows and the tail stages of every row against their bars, with the region maxima
    of the 8-window groups, the M tile edges and the last, partial M tile; returns the misses."""
    n, t = len(a), head_tile(len(a), conv_impl)
    reg = R.position_regions(n, windows=idx, tile=t)
    preg = R.position_regions(n, pooled=True, windows=idx, tile=t)
    win = {k: v for k, v in reg.items() if k.startswith("win")}
    every = {k: v for k, v in R.position_regions(n, tile=t).items() if k.startswith("win")}
    for k in ("q1", "mpi1") + (("q0", "mpi0") if "q0" in samp else ()):
        assert torch.equal(samp[k], tail[k][idx]), f"{label}: {k} differs between the debug stops"
    return (GS._check(f"{label}, sampled rows", w, a[idx], samp, conv_impl, regions=(reg, preg), rows=win) +
            GS._check(f"{label}, every row", w, a, tail, conv_impl, rows=every))


# ------------------------------------------------------------------------------------------ a. stages at tile-edge shapes
@pytest.mark.parametrize("n", TC_SHAPES + FFMA_SHAPES)
def test_stages_at_tile_edges(syn, pool, n):
    a = pool[:n]
    idx = sample_rows(n)
    ix = torch.as_tensor(idx, device="cuda")
    da = torch.from_numpy(a).cuda()
    c = _classifier(syn, n)
    bad = []
    print(GS.HEADER)
    try:
        for path, opts in paths(n):
            for k, v in {**GT.DEFAULTS, **opts}.items():
                c.set_option(k, v)
            samp = {}
            try:
                for stop in (2, 3):
                    c.set_option("debug_stop", stop)
                    c.predict_ascii(da)
                    c.check_status()
                    if stop == 2:
                        samp.update(y1=GT._take(c, "buf0", n, ix), y2=GT._take(c, "buf1", n, ix), q0=GT._take(c, "q0", n, ix),
                                    mpi0=GT._take(c, "mpi0", n, ix))
                    else:
                        samp.update(y3=GT._take(c, "buf0", n, ix))
            finally:
                c.set_option("debug_stop", 0)
            probs = c.predict_ascii(da)
            c.check_status()
            s0, tail = _fetch_step(c, n, idx)
            assert torch.equal(samp["y3"].double(), s0["y3"]), f"{path}: conv3 is not deterministic across steps"
            samp = {**GT._f64(samp), **{k: v for k, v in s0.items() if k != "y3"}}
            tail["probs"] = probs.double().cpu()
            bad += _check_step(f"n={n}, {path}", syn, a, samp, tail, idx, opts.get("conv_impl", 0))
    finally:
        c.close()
    assert not bad, bad


# ------------------------------------------------------------------------------------------ b. multi-step calls, short last step
@pytest.mark.parametrize("max_batch, n", MULTI_STEP)
def test_multistep_call_ending_in_a_short_step(syn, pool, max_batch, n):
    """Every step's probabilities are bitwise those of a one-step call on its windows, the fetched buffers are the last step's
    (bitwise those of a one-step call on it, and within their bars against references built from its inputs), and a repeat of
    the call is bitwise the first.  The short step's one-step call comes first, so the multi-step call starts on a window-group
    count other than the one wv_gather_kernel's CTA split was last made for, and its last step changes that count again."""
    a = pool[:n]
    da = torch.from_numpy(a).cuda()
    steps = [(o, min(n, o + max_batch)) for o in range(0, n, max_batch)]
    lo, hi = steps[-1]
    m = hi - lo
    idx = sample_rows(m)
    c = _classifier(syn, max_batch)
    bad = []
    print(GS.HEADER)
    try:
        for overlap in (0, 1):
            for k, v in {**GT.DEFAULTS, "tail_overlap": overlap}.items():
                c.set_option(k, v)
            p_short = c.predict_ascii(da[lo:hi])
            c.check_status()
            one_samp, one_tail = _fetch_step(c, m, idx)
            p = c.predict_ascii(da)
            c.check_status()
            samp, tail = _fetch_step(c, m, idx)
            GT._assert_bitwise(samp, one_samp, f"tail_overlap {overlap}: multi-step vs one-step call of the last step")
            GT._assert_bitwise(tail, one_tail, f"tail_overlap {overlap}: multi-step vs one-step call of the last step")
            tail["probs"] = p[lo:hi].double().cpu()
            bad += _check_step(f"{n} windows, max_batch {max_batch}, tail_overlap {overlap}, last step ({m} windows)", syn,
                               a[lo:hi], samp, tail, idx)
            assert torch.equal(p[lo:hi], p_short), f"tail_overlap {overlap}: last step"
            for i, (s, e) in enumerate(steps[:-1]):
                assert torch.equal(p[s:e], c.predict_ascii(da[s:e])), f"tail_overlap {overlap}: step {i}"
            assert torch.equal(c.predict_ascii(da), p), f"tail_overlap {overlap}: the repeated call"
            c.check_status()
    finally:
        c.close()
    assert not bad, bad


# ------------------------------------------------------------------------------------------ c. bitwise batch invariance
@pytest.mark.parametrize("path", ["tc fused (default)", "tc fuse_gather=0"])
def test_batch_invariance_with_live_weights(syn, pool, path):
    """Each window's probabilities (predict_ascii, predict_tokens, embed_ascii) and embeddings are bitwise the same at every
    max_batch, in a permuted pool and in single-window calls, and the embeddings are bitwise the h1 of their step.  Each handle
    runs its single-window calls first, so every later call starts on another window-group count.  The default path is
    compared with itself only: fuse_gather = 0 sums mpi in another order (test_gpu_tokens_batch1024._assert_paths_bitwise)."""
    a = pool[:POOL]
    da = torch.from_numpy(a).cuda()
    tok = GT._cuda_tokens(T.tokenize_windows(a))
    perm = torch.from_numpy(np.random.default_rng(3).permutation(POOL)).cuda()
    ref = None
    for mb in INVARIANCE_BATCHES:
        c = _classifier(syn, mb)
        try:
            for k, v in {**GT.DEFAULTS, **TC_PATHS[path]}.items():
                c.set_option(k, v)
            single = {}
            for i in SINGLES:
                p1, e1 = c.embed_ascii(da[i:i + 1])
                assert torch.equal(e1, c.debug_fetch("h1", 1)), f"max_batch {mb}: window {i}'s embedding is not its h1"
                assert torch.equal(c.predict_ascii(da[i:i + 1]), p1), f"max_batch {mb}: window {i}"
                single[i] = (p1, e1)
            p = c.predict_ascii(da)
            pe, e = c.embed_ascii(da)
            last = (POOL - 1) // mb * mb
            assert torch.equal(e[last:], c.debug_fetch("h1", POOL - last)), f"max_batch {mb}: embeddings vs the last step's h1"
            pp, ep = c.embed_ascii(da[perm])
            pt = c.predict_tokens(tok)
            c.check_status()
        finally:
            c.close()
        assert torch.equal(pe, p) and torch.equal(pt, p), f"max_batch {mb}: embed_ascii / predict_tokens vs predict_ascii"
        assert torch.equal(pp, p[perm]) and torch.equal(ep, e[perm]), f"max_batch {mb}: permuted pool"
        for i, (p1, e1) in single.items():
            assert torch.equal(p1, p[i:i + 1]) and torch.equal(e1, e[i:i + 1]), f"max_batch {mb}: single-window call {i}"
        if ref is None:
            ref = (p, e)
        else:
            rows = (p != ref[0]).any(dim=1) | (e != ref[1]).any(dim=1)
            assert not bool(rows.any()), f"max_batch {mb} vs {INVARIANCE_BATCHES[0]}: windows {rows.nonzero().flatten().tolist()[:10]}"


# ------------------------------------------------------------------------------------------ d. attribution chunks across a tile
def _attribute_sample(c, asc, target, idx):
    """attribute_ascii on one chunk, with the forward and backward buffers of the rows idx (test_gpu_attr_stages._attribute,
    fetched on the GPU and sampled there)"""
    n = len(asc)
    assert n <= c.attr_max_batch
    a = torch.from_numpy(asc).cuda()
    ix = torch.as_tensor(idx, device="cuda")
    c.predict_ascii(a)
    c.check_status()
    logits1 = GT._take(c, "logits", n, ix)[:, :R.N_POOL].double()
    probs, attr = c.attribute_ascii(a, target)
    c.check_status()
    got = {k: GT._take(c, k, n, ix).double() for k in ("h1", "h2", "q0", "q1", "mpi1", "h0", "attr_y1", "buf1", "buf0",
                                                        "attr_g_out", "attr_s_w", "attr_s2", "attr_gz3", "attr_gz2",
                                                        "attr_gy1", "attr_gz1")}
    got.update(logits1=logits1, logits0=GT._take(c, "logits", n, ix)[:, :R.N_POOL].double(), probs=probs[ix].double().cpu(),
               attr=attr[ix].double().cpu(), route0=GT._take(c, "route0", n, ix).numpy(),
               route1=GT._take(c, "route1", n, ix).numpy(), last0=0)
    return got, probs, attr


def test_attribution_chunks_across_a_tile(syn, pool):
    """Gradient x input on a 200-window chunk (two M tiles): every backward stage of the windows around window 128 within its
    bar, attributions within 1e-4 of fp64, and bitwise those of chunks of 64 and 8 windows.  Integrated gradients of 13
    windows x 16 steps (208 rows, window 8 on rows 128-143): bitwise those of one window per call, and windows 0, 8 and 12
    within test_gpu_ig's bar of fp64."""
    asc = pool[:ATTR_CHUNK]
    a = torch.from_numpy(asc).cuda()
    ig_asc = pool[:IG_WINDOWS]
    c = _classifier(syn, ATTR_CTX)
    try:
        c._attr_ctx(ATTR_CTX)
        got, probs, attr = _attribute_sample(c, asc, TARGET, ATTR_SAMPLE)
        ig = GI._gpu_ig(c, ig_asc, TARGET, IG_STEPS, "zero")
        dig = torch.from_numpy(ig_asc).cuda()
        for i in range(IG_WINDOWS):
            p1, l1, x1 = (v.cpu().numpy() for v in c.integrated_gradients_ascii(dig[i:i + 1], TARGET, IG_STEPS, "zero"))
            assert (np.array_equal(p1, ig[0][i:i + 1]) and np.array_equal(l1, ig[1][i:i + 1]) and
                    np.array_equal(x1, ig[2][i:i + 1])), f"integrated gradients of window {i}: one call vs 13 windows"
        c.check_status()
    finally:
        c.close()
    for mb in (64, 8):
        c = _classifier(syn, mb)
        try:
            c._attr_ctx(mb)
            p2, x2 = c.attribute_ascii(a, TARGET)
            c.check_status()
        finally:
            c.close()
        assert torch.equal(p2, probs) and torch.equal(x2, attr), f"chunks of {mb} vs one chunk of {ATTR_CHUNK}"
    print(GA.HEADER)
    sel = asc[ATTR_SAMPLE]
    bad = GA._check(f"{ATTR_CHUNK}-window chunk, windows {ATTR_SAMPLE}", syn, sel, TARGET, got)
    err = GA._attr_vs_fp64(syn, sel, TARGET, got)
    print(f"\nattributions vs fp64, windows {ATTR_SAMPLE}: " + " ".join(f"{e:.1e}" for e in err))
    assert not bad, bad
    assert err.max() <= 1e-4, err
    _, _, x, routes, masks, h2 = ig
    rows = np.concatenate([np.arange(i * IG_STEPS, (i + 1) * IG_STEPS) for i in IG_CHECK])
    _, J = GI._reference(T.tokenize_windows(ig_asc[list(IG_CHECK)]), syn, IG_STEPS, "zero", [r[rows] for r in routes],
                         [k[rows] for k in masks])
    logits = h2[rows] @ syn["d2w"].astype(np.float64) + syn["d2b"].astype(np.float64)
    e, _, _ = GI._check(x[list(IG_CHECK)], J, logits, TARGET, IG_STEPS)
    print(f"\nintegrated gradients, windows {IG_CHECK} of {IG_WINDOWS} x {IG_STEPS} steps: error / bar "
          + " ".join(f"{v:.2f}" for v in e))
    assert e.max() <= 1.0, e
