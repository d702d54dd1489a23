"""
Every stage against fp64 on arbitrary token input, and at the production batch of 1024 windows (run with `-m gpu -s` for the
tables).

gnm_forward_tokens is nn_model.predict on a token batch, whose first op is tf.one_hot(x, 257): any uint16 is valid input, a token
above 256 contributes nothing, and tokens need not be the overlapping 4-mers a tokenizer produces.  The golden token windows
(tests/golden/reference_tokens_golden.npz, from the reference's own model graph) go through every layer-1 / w_v / gather path.

At batch 1024 the activation buffers pass byte offsets 2^31 and 2^32 (one window is 5997 x 768 B, so at windows 466 and 932),
each persistent CTA of the conv kernels works through ~186 units instead of ~4, and multi-step calls alternate two buffer sets.
A whole-batch fp64 reference would be 6 GB per activation and ~1 TFLOP per conv layer on the CPU, so each buffer is fetched on
the GPU, the sampled windows are indexed there and only they are copied to the host; the references are computed for them
alone.  Synthetic O(1) IGLOO weights keep the patch gather and the attention logits live.
"""
import sys
import time
from pathlib import Path

import numpy as np
import pytest
import torch

import stage_ref as R
from oracle import igloo_model as M
from oracle import tokenizer as T
from test_gpu_stages import HEADER, _check

pytestmark = pytest.mark.gpu

N = 1024
SAMPLE = [0, 1, 7, 8, 9, 465, 466, 467, 468, 511, 512, 931, 932, 933, 934, 1015, 1016, 1023]
ROW_BYTES = 5997 * 768                       # one window of activations (four planes)
PATHS = {"tc fused (default)": {}, "tc fuse_l1": {"fuse_l1": 1}, "tc fuse_gather=0": {"fuse_gather": 0}}
SAME_ALL_PATHS = ("y1", "y2", "y2_3", "y3", "y3_0", "q0", "q1")
DEFAULTS = {"conv_impl": 0, "fuse_l1": 0, "fuse_gather": 1, "tail_overlap": 1, "debug_stop": 0}
STATS = {"device_used_peak": 0}


@pytest.fixture(scope="module", autouse=True)
def _report_cost():
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    yield
    print(f"\n{Path(__file__).name}: {time.time() - t0:.0f} s; peak torch allocation "
          f"{torch.cuda.max_memory_allocated() / 2**30:.2f} GiB; peak device memory in use {STATS['device_used_peak'] / 2**30:.2f} GiB")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(golden_dir / "reference_tokens_golden.npz")


@pytest.fixture(scope="module")
def shipped(weights_npz):
    return M.load_npz_weights(weights_npz)


@pytest.fixture(scope="module")
def syn(shipped):
    return M.synthetic_igloo_weights(shipped)


def _cuda_tokens(tok):
    return torch.from_numpy(np.ascontiguousarray(tok, dtype=np.uint16).view(np.int16)).cuda().view(torch.uint16)


def _take(c, name, n, idx):
    """Buffer `name` of the last step (n windows) on the GPU, only the rows idx copied to the host."""
    x = c.debug_fetch(name, n)
    free, total = torch.cuda.mem_get_info()
    STATS["device_used_peak"] = max(STATS["device_used_peak"], total - free)
    s = x[idx].cpu()
    del x
    return s


def _run(c, x, opts, idx, stops=(2, 3, 0), ascii=False, last=None):
    """predict (tokens, or ASCII windows) at each debug stop with the options; the fetched rows idx of the last step's buffers
    (last = that step's window count), fp32 on the host, and the full probabilities of the final (stop 0) call."""
    for k, v in {**DEFAULTS, **opts}.items():
        c.set_option(k, v)
    m = last or len(x)
    ix = torch.as_tensor(idx, device="cuda")
    got, probs = {}, None
    try:
        for stop in stops:
            c.set_option("debug_stop", stop)
            p = (c.predict_ascii if ascii else c.predict_tokens)(x)
            c.check_status()                                    # no activation-range flag, no device-side failure

            def f(name):
                return _take(c, name, m, ix)
            if stop == 2:
                got.update(y1=f("buf0"), y2=f("buf1"), q0=f("q0"), mpi0=f("mpi0"))
            elif stop == 3:
                got.update(y2_3=f("buf1"), y3=f("buf0"))
            else:
                probs = p.cpu()
                got.update(y3_0=f("buf0"), q0=f("q0"), mpi0=f("mpi0"), q1=f("q1"), mpi1=f("mpi1"),
                           logits=f("logits")[:, :R.N_POOL], h0=f("h0"), h1=f("h1"), h2=f("h2"),
                           probs=probs[len(x) - m:][idx])
                if "y2_3" not in got:                           # a full step leaves y2 in buf1 and y3 in buf0
                    got.update(y2_3=f("buf1"), y3=got["y3_0"])
    finally:
        c.set_option("debug_stop", 0)
    return got, probs


def _f64(got):
    return {k: v.double() for k, v in got.items()}


def _regions(n, windows):
    """R.position_regions over the sample, plus the windows whose activation rows cross byte offset 2^31 / 2^32 and the first
    window wholly past it."""
    reg, preg = R.position_regions(n, windows=windows), R.position_regions(n, pooled=True, windows=windows)
    for e in (31, 32):
        first = 2 ** e // ROW_BYTES
        rows = [r for r, i in enumerate(windows) if i in (first, first + 1)]
        if rows:
            for d in (reg, preg):
                d[f"win {first}-{first + 1} (2^{e} B)"] = (rows, slice(None))
    return reg, preg


def _assert_bitwise(a, b, label, keys=None):
    for k in keys or a:
        if k in a and k in b:
            assert torch.equal(a[k], b[k]), f"{label}: {k} differs"


def _assert_paths_bitwise(runs):
    """The activations and q of the three paths are bitwise equal (the three w_v implementations issue the same passes in the
    same order).  mpi is not: the fused IGLOO kernel's gather sums in another order than patch_stream_kernel, which both
    fuse_l1 = 1 and fuse_gather = 0 use, so those two agree in everything and the default path only up to mpi's bar."""
    base, sep = runs["tc fused (default)"], runs["tc fuse_gather=0"]
    _assert_bitwise(base, runs["tc fuse_l1"], "tc fuse_l1", SAME_ALL_PATHS)
    _assert_bitwise(base, sep, "tc fuse_gather=0", SAME_ALL_PATHS)
    _assert_bitwise(sep, runs["tc fuse_l1"], "tc fuse_l1 vs tc fuse_gather=0")


# ------------------------------------------------------------------------------------------ arbitrary tokens, n <= 16
@pytest.mark.parametrize("which", ["in_range", "out_of_range"])
def test_arbitrary_tokens_every_stage(golden, shipped, syn, which):
    """The golden token windows (all tokens <= 256, or carrying 257 .. 65535) through the default path, fuse_l1 = 1 and
    fuse_gather = 0: every stage meets its bar against fp64 on its own input, the activations and q are bitwise equal across the paths,
    and the probabilities are within 1e-4 of the reference graph's, same argmax (shipped and synthetic IGLOO weights)."""
    from genomad_b200 import engine
    sel = golden["in_range"] if which == "in_range" else ~golden["in_range"]
    tok = golden["tokens"][sel]
    n = len(tok)
    x = _cuda_tokens(tok)
    runs = {}
    c = engine.Classifier(syn, device=0, max_batch=16)
    try:
        for path, opts in PATHS.items():
            runs[path] = _run(c, x, opts, list(range(n)))[0]
    finally:
        c.close()
    print(HEADER)
    bad = []
    for path, got in runs.items():
        bad += _check(f"tokens {which}, n={n}, {path}", syn, tok, _f64(got), tokens=tok)
        p = got["probs"].numpy()
        dp = np.abs(p - golden["synthetic"][sel]).max()
        print(f"{path}: max |dp| vs the reference graph {dp:.2e}")
        if dp > 1e-4 or not np.array_equal(p.argmax(1), golden["synthetic_fp64"][sel].argmax(1)):
            bad.append((path, "probs vs reference graph", dp))
    assert not bad
    _assert_paths_bitwise(runs)
    c = engine.Classifier(shipped, device=0, max_batch=16)
    try:
        for path, opts in PATHS.items():
            for k, v in {**DEFAULTS, **opts}.items():
                c.set_option(k, v)
            p = c.predict_tokens(x).cpu().numpy()
            c.check_status()
            assert np.abs(p - golden["shipped"][sel]).max() <= 1e-4, path
            assert np.array_equal(p.argmax(1), golden["shipped_fp64"][sel].argmax(1)), path
    finally:
        c.close()


# ------------------------------------------------------------------------------------------ batch 1024
@pytest.fixture(scope="module")
def clf1024(syn):
    from genomad_b200 import engine
    c = engine.Classifier(syn, device=0, max_batch=N)
    yield c
    c.close()


@pytest.fixture(scope="module")
def batch(golden):
    """1024 ASCII windows of the precision-study families, their tokens, and the same tokens with every window w = 1 (mod 3)
    replaced by golden token window w mod 16 (random, inconsistent and out-of-range tokens)."""
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tools"))
    import precision_study
    a = precision_study.make_windows(N, seed=61)
    tok = T.tokenize_windows(a)
    arb = np.arange(N) % 3 == 1
    mixed = tok.copy()
    mixed[arb] = golden["tokens"][np.arange(N)[arb] % 16]
    return a, tok, mixed, arb


def test_batch1024_sampled_stages(clf1024, syn, batch):
    """A 1024-window step, three paths: the fetched activations and q of the sampled windows are bitwise equal across the paths
    (everything is between fuse_l1 = 1 and fuse_gather = 0), every stage meets its bar against fp64 on its own input (per region, including the windows at 2^31 and 2^32 bytes and at the 8-window
    group edges), and windows that are a tokenization give bitwise the probabilities of predict_ascii on their bytes."""
    a, tok, mixed, arb = batch
    x = _cuda_tokens(mixed)
    runs, probs = {}, {}
    for path, opts in PATHS.items():
        runs[path], probs[path] = _run(clf1024, x, opts, SAMPLE)
    _assert_paths_bitwise(runs)
    assert torch.equal(probs["tc fuse_gather=0"], probs["tc fuse_l1"])
    da = torch.from_numpy(a).cuda()
    for path, opts in PATHS.items():
        _, p_ascii = _run(clf1024, da, opts, SAMPLE[:1], stops=(0,), ascii=True)
        keep = torch.from_numpy(~arb)
        assert torch.equal(p_ascii[keep], probs[path][keep]), path
    print(HEADER)
    bad = []
    for path in ("tc fused (default)", "tc fuse_gather=0"):            # fuse_l1 = 1: bitwise the fuse_gather = 0 run
        bad += _check(f"batch 1024, sampled windows, {path}", syn, mixed[SAMPLE], _f64(runs[path]), tokens=mixed[SAMPLE],
                      regions=_regions(N, SAMPLE))
    assert not bad


@pytest.mark.parametrize("n", [2 * N, 2 * N + 8])
def test_multistep_call_leaves_the_last_steps_buffers(clf1024, syn, batch, n):
    """A multi-step call with the tails overlapped (two buffer sets, alternating by step parity): afterwards the fetched y2 / y3 /
    q / mpi / logits / h0-h2 are those of the last step (bitwise equal to a one-step call on its windows, not equal to another
    step's, and within their bars against references built from that step's inputs), and the probabilities of every step are
    bitwise those of a one-step call.  2048 windows end on parity 1; 2056 make a third, partial step on parity 0."""
    _, _, mixed, _ = batch
    tok = np.concatenate([mixed, np.roll(mixed, 301, axis=0), mixed[[1, 7, 8, 466, 467, 933, 1016, 1023]]])[:n]
    steps = [tok[o:o + N] for o in range(0, n, N)]
    m = len(steps[-1])
    idx = SAMPLE if m == N else list(range(m))
    got, p_multi = _run(clf1024, _cuda_tokens(tok), {}, idx, stops=(0,), last=m)
    one = []
    for i, s in enumerate(steps):
        g1, p1 = _run(clf1024, _cuda_tokens(s), {}, idx if i == len(steps) - 1 else SAMPLE[:m], stops=(0,))
        assert torch.equal(p_multi[i * N:i * N + len(s)], p1), f"step {i}"
        one.append(g1)
    _assert_bitwise(got, one[-1], "multi-step vs one-step call of the last step")
    other = one[-2]
    assert not torch.equal(got["q1"][:2], other["q1"][:2]) and not torch.equal(got["h2"][:2], other["h2"][:2])
    print(HEADER)
    assert not _check(f"{n} windows in {len(steps)} steps, last step ({m} windows)", syn, steps[-1][idx], _f64(got),
                      regions=_regions(m, idx))
