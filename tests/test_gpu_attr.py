"""
Attributions on the H100 (run with `-m gpu -s` for the measured precision): gnm_attribute_* against the fp64 autograd reference
(tests/attr_ref.py) following the GPU's own max-pool routing, the routing against the fp64 argmax and the forward's q, and the
bitwise identities: probabilities equal to predict_ascii / predict_windows, repeatability, chunking, contigs against rows.
"""
import time
from pathlib import Path

import numpy as np
import pytest
import torch

from genomad_b200 import engine, synth
from oracle import igloo_model as M
from oracle import tokenizer as T
import attr_ref as A

pytestmark = pytest.mark.gpu

MB = 16                     # attribution chunk of the small-batch tests


@pytest.fixture(scope="module", autouse=True)
def _report_cost():
    t0 = time.time()
    yield
    print(f"\n{Path(__file__).name}: {time.time() - t0:.0f} s; peak torch allocation {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


@pytest.fixture(scope="module")
def weights(weights_npz):
    w = M.load_npz_weights(weights_npz)
    return {"shipped": w, "synthetic": M.synthetic_igloo_weights(w)}


@pytest.fixture(scope="module")
def windows(golden_dir):
    """golden windows, random ACGT, N runs, an all-N window and a 2.5 kb padded tail"""
    g = np.load(golden_dir / "reference_graph_golden.npz")["windows"][:4]
    rng = np.random.default_rng(21)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    rand = acgt[rng.integers(0, 4, (2, 6000))]
    runs = acgt[rng.integers(0, 4, 6000)].copy()
    runs[700:1500] = ord("N"); runs[5000:5090] = ord("N")
    alln = np.full(6000, ord("N"), dtype=np.uint8)
    tail = acgt[rng.integers(0, 4, 6000)].copy()
    tail[2500:] = ord("N")
    return np.concatenate([g, rand, runs[None], alln[None], tail[None]])        # 9 windows


def _attr_error(got, ref):
    """per window max_t |got - ref| / max_t |ref|; ref follows the GPU forward's max-pool routing and LeakyReLU branches"""
    return np.abs(got.astype(np.float64) - ref).max(axis=1) / np.maximum(np.abs(ref).max(axis=1), 1e-300)


def _check_against_fp64(c, asc, w, target, rows=None):
    """attributions of `asc` (a [n, 6000] uint8 array) against fp64 along the GPU's routing, on `rows` (default all)"""
    a = torch.from_numpy(asc).cuda()
    probs, attr = c.attribute_ascii(a, target)
    c.check_status()
    n = len(asc)
    rows = np.arange(n) if rows is None else np.asarray(rows)
    last0 = (n - 1) // c.attr_max_batch * c.attr_max_batch                       # routing buffers hold the last chunk
    in_last = rows[rows >= last0]
    r0 = c.debug_fetch("route0", n - last0).cpu().numpy()
    r1 = c.debug_fetch("route1", n - last0).cpu().numpy()
    k = in_last - last0
    # the forward's LeakyReLU branches, y1, y2, y3: joined row > 0 is exactly the kernels' hi16 > 0
    # (tests/test_attr_cpu.py::test_joined_row_sign_is_the_hi16_sign)
    masks = [(c.debug_fetch(b, n - last0)[k] > 0).cpu().numpy() for b in ("attr_y1", "buf1", "buf0")]
    tok = T.tokenize_windows(asc[in_last])
    ref = A.attribution(tok, w, target, routes=[r0[k], r1[k]], masks=masks)
    err = _attr_error(attr.cpu().numpy()[in_last], ref)
    return probs, attr, err


@pytest.mark.parametrize("variant", ["shipped", "synthetic"])
def test_attributions_within_1e4_of_fp64(weights, windows, variant):
    w = weights[variant]
    c = engine.Classifier(w, device=0, max_batch=64)
    try:
        c._attr_ctx(MB)
        worst = 0.0
        for target in (0, 1, 2):
            probs, attr, err = _check_against_fp64(c, windows, w, target)
            worst = max(worst, err.max())
            print(f"\n{variant} target {target}: per-window max|d attr| / max|attr| vs fp64 (GPU routing): "
                  + " ".join(f"{e:.1e}" for e in err))
            assert err.max() <= 1e-4, err
            assert torch.equal(probs, c.predict_ascii(torch.from_numpy(windows).cuda()))
        for n in (1, 7, MB, MB + 3):                                  # call sizes; the last chunk is checked
            asc = np.concatenate([windows] * 3)[:n]
            _, _, err = _check_against_fp64(c, asc, w, 2)
            assert err.max() <= 1e-4, (n, err)
        print(f"\n{variant}: worst {worst:.2e}")
    finally:
        c.close()


@pytest.mark.parametrize("opts", [{"fuse_l1": 1}, {"fuse_gather": 0}, {"tail_overlap": 0}])
def test_forward_options(weights, windows, opts):
    """The attribution pass re-runs layer 1 with embed_conv1_kernel and routes with conv_t's w_v pass, whichever forward path
    the options pick: its maxima must still be that step's q bit for bit, and the attributions within the bar."""
    w = weights["synthetic"]
    c = engine.Classifier(w, device=0, max_batch=2 * MB)               # the context is smaller than the handle
    try:
        c._attr_ctx(MB)
        for k, v in opts.items():
            c.set_option(k, v)
        probs, _, err = _check_against_fp64(c, windows, w, 2)
        n = len(windows)
        for s in (0, 1):
            assert torch.equal(c.debug_fetch(f"routeq{s}", n), c.debug_fetch(f"q{s}", n)), (opts, s)
        assert torch.equal(probs, c.predict_ascii(torch.from_numpy(windows).cuda()))
        print(f"\n{opts}: worst {err.max():.2e}")
        assert err.max() <= 1e-4, err
        with pytest.raises(engine.GnmError, match="max_batch"):
            c.debug_fetch("route0", MB + 1)
    finally:
        c.close()


def test_routing_is_the_forward_maxpool(weights, windows):
    w = weights["synthetic"]
    c = engine.Classifier(w, device=0, max_batch=16)
    try:
        c._attr_ctx(16)
        a = torch.from_numpy(windows).cuda()
        c.attribute_ascii(a, 1)
        n = len(windows)
        tok = T.tokenize_windows(windows)
        ref = A.routing(tok, w)
        for s in (0, 1):
            r = c.debug_fetch(f"route{s}", n).cpu().numpy()
            rq = c.debug_fetch(f"routeq{s}", n)
            q = c.debug_fetch(f"q{s}", n)
            assert torch.equal(rq, q), "routing maxima must be the forward's q bit for bit"
            r64, gap, top = ref[s]
            clear = gap > 1e-5 * (top + 1)
            agree = (r == r64)[clear].mean()
            print(f"\nIGLOO#{s}: routing equals the fp64 argmax on {agree:.6%} of {clear.sum()} clear pools "
                  f"({(~clear).sum()} near-ties skipped)")
            assert agree == 1.0
    finally:
        c.close()


@pytest.fixture(scope="module")
def batch():
    idx = synth.subsample_indices(40, 1_000_000, seed=4)
    a = synth.windows_numpy(idx, seed=4)
    a[3, 2000:] = ord("N")
    return a


def test_bitwise_identities(weights, batch):
    c = engine.Classifier(weights["shipped"], device=0, max_batch=32)
    c2 = engine.Classifier(weights["shipped"], device=0, max_batch=32)
    try:
        c._attr_ctx(16)
        c2._attr_ctx(5)
        a = torch.from_numpy(batch).cuda()
        p1, x1 = c.attribute_ascii(a, "virus")
        p2, x2 = c.attribute_ascii(a, 2)
        p3, x3 = c2.attribute_ascii(a, 2)                           # chunks of 5 instead of 16
        assert torch.equal(x1, x2) and torch.equal(p1, p2), "two calls give the same bits"
        assert torch.equal(x1, x3) and torch.equal(p1, p3), "attributions do not depend on chunking"
        assert torch.equal(p1, c.predict_ascii(a)), "probabilities are predict_ascii's"
        c.check_status()
        # contigs: attribute_contigs against attribute_ascii on the same windows gathered beforehand
        rng = np.random.default_rng(9)
        seqs = [bytes(rng.choice(list(b"ACGTacgtN"), int(L))) for L in (2600, 6000, 13000, 30011, 800)]
        res = c.attribute_contigs(seqs, "plasmid")
        seq, offs = c.contig_buffers(seqs)
        start, length, woff = c.contig_windows(seq, offs)
        rows = c.gather_windows(seq, start, length)
        pa, xa = c.attribute_ascii(rows, 1)
        assert torch.equal(res.attr, xa) and torch.equal(res.probs, pa)
        assert torch.equal(res.probs, c.predict_windows(seq, start, length))
        assert torch.equal(res.offsets, woff) and res.attr.shape == (int(woff[-1]), 5997)
        # the validation path has no backward pass
        c.set_option("conv_impl", 1)
        with pytest.raises(engine.GnmError, match="conv_impl"):
            c.attribute_ascii(a[:2], 0)
        c.set_option("conv_impl", 0)
    finally:
        c.close()
        c2.close()


def test_batch1024_sampled(weights):
    """A 1024-window call in 4 chunks of 256: sampled rows against fp64, and the largest |g_z3| s_w seen."""
    w = weights["synthetic"]
    idx = synth.subsample_indices(1024, 1_000_000, seed=8)
    asc = synth.windows_numpy(idx, seed=8)
    asc[1000, 3500:] = ord("N")
    c = engine.Classifier(w, device=0, max_batch=256)
    try:
        c._attr_ctx(256)
        rows = [768, 769, 900, 1000, 1023]                              # rows of the last chunk (the routing buffers hold it)
        probs, attr, err = _check_against_fp64(c, asc, w, 2, rows=rows)
        print(f"\nbatch 1024 (synthetic), sampled rows {rows}: " + " ".join(f"{e:.1e}" for e in err))
        assert err.max() <= 1e-4
        assert torch.equal(probs, c.predict_ascii(torch.from_numpy(asc).cuda()))
    finally:
        c.close()


def test_module_write_attributions(tmp_path, golden_dir, monkeypatch):
    """nn_classification.main with write_attributions on the reference module's toy input: predictions bitwise those of a run
    without the option, and every window's row equal to attribute_windows on the module's own windows."""
    import shutil
    from genomad_b200 import _paths, nn_classification
    for k in ("GENOMAD_B200_ATTRIBUTIONS", "GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS"):
        monkeypatch.delenv(k, raising=False)
    inp = golden_dir / "reference_module" / "input"
    runs = {}
    for name, opt in (("off", None), ("on", "virus")):
        out = tmp_path / name
        shutil.copytree(inp / "toy_find_proviruses", out / "toy_find_proviruses")
        nn_classification.main(inp / "toy.fna", out, False, 128, False, 2, False, False, write_attributions=opt)
        runs[name] = _paths.NNOutputs("toy", out)
    for attr in ("nn_classification_npz_output", "provirus_nn_classification_npz_output"):
        a, b = np.load(getattr(runs["off"], attr)), np.load(getattr(runs["on"], attr))
        assert np.array_equal(a["predictions"], b["predictions"]), attr
    z = np.load(runs["on"].nn_classification_attributions_output)
    assert str(z["target"]) == "virus" and z["attributions"].shape == (len(z["window_start"]), 5997)
    # the same windows through the device path: bitwise the same rows
    from genomad_b200 import sequence
    seqs = {sequence.accession(h): s for h, s in sequence.iter_fasta(inp / "toy.fna", strip_n=False)}
    c = engine.Classifier(None, device=0, max_batch=64)
    try:
        names = list(z["contig_names"])
        rows = np.stack([np.frombuffer(seqs[names[ci]][s: s + ln].upper().ljust(6000, b"N"), np.uint8)
                         for ci, s, ln in zip(z["window_contig"], z["window_start"], z["window_length"])])
        _, x = c.attribute_ascii(torch.from_numpy(rows).cuda(), "virus")
        assert np.array_equal(x.cpu().numpy(), z["attributions"])
    finally:
        c.close()
