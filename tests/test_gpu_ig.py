"""
Integrated gradients on the H100 (run with `-m gpu -s` for the measured precision): gnm_attribute_ig_* against the fp64 IG
reference (tests/ig_ref.py) at the same midpoint nodes, each row following the GPU forward's max-pool routing, LeakyReLU
branches and logits (from its h2); completeness; the payoff on windows classified confidently as the target, where gradient x
input is ~0 or exactly 0; and the bitwise identities: probabilities equal to predict_ascii, log p_c by the documented formula,
independence of the chunking, window order, batch composition and forward options; the module with --attribution-steps
against a run without it and against integrated_gradients_contigs.

Bar, per window: max_t |IG_gpu - IG_ref| <= 1e-4 * mean_k max_t |row_k,ref[t]| -- the per-row bar of the gradient x input
tests (tests/test_gpu_attr.py) carried through the mean over k.
"""
import time
from pathlib import Path

import numpy as np
import pytest
import torch

from genomad_b200 import engine
from oracle import igloo_model as M
from oracle import tokenizer as T
import ig_ref as I

pytestmark = pytest.mark.gpu

BAR = 1e-4
MB = 64                      # handle and attribution context of the small-batch tests: every row of a call in one chunk


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


def logp_formula(p32, target):
    """log p_c from float32 probabilities as gnm.h states it: -log1p(sum of the others, fp32, ascending) when p_c is the
    largest, log p_c otherwise; in fp64, rounded to fp32"""
    p = np.asarray(p32, dtype=np.float32)
    o = [i for i in range(3) if i != target]
    other = (np.float32(0) + p[:, o[0]]) + p[:, o[1]]
    top = (p[:, target] >= p[:, o[0]]) & (p[:, target] >= p[:, o[1]])
    return np.where(top, -np.log1p(other.astype(np.float64)), np.log(p[:, target].astype(np.float64))).astype(np.float32)


def _gpu_ig(c, asc, target, steps, baseline):
    """IG of `asc` and, for its rows (all in one chunk), the forward's routing, LeakyReLU branches (layers 1-3 and the head's
    ReLUs, appended to the masks) and logits"""
    a = torch.from_numpy(asc).cuda()
    probs, logp, attr = c.integrated_gradients_ascii(a, target, steps, baseline)
    c.check_status()
    rows = len(asc) * steps
    assert rows <= c.attr_max_batch
    routes = [c.debug_fetch(f"route{s}", rows).cpu().numpy() for s in (0, 1)]
    masks = [(c.debug_fetch(b, rows) > 0).cpu().numpy() for b in ("attr_y1", "buf1", "buf0", "h1", "h2")]
    h2 = c.debug_fetch("h2", rows).cpu().numpy().astype(np.float64)
    return probs.cpu().numpy(), logp.cpu().numpy(), attr.cpu().numpy(), routes, masks, h2


def _reference(tok, w, steps, baseline, routes, masks):
    """per-row fp64 logit Jacobians along the GPU rows' routing and branches (shared by every target and head scale)"""
    B = len(tok)
    return I.logit_jacobian(np.repeat(tok, steps, axis=0), w, np.tile(I.alphas(steps), B), baseline, routes, masks[:3],
                            head_masks=masks[3:])


def _check(attr, J, logits_at, target, steps, scale=1.0):
    """per-window error / bar, and the reference's IG and rows"""
    B = attr.shape[0]
    rows = I.rows_from_jacobian(logits_at / scale, J, target, scale).reshape(B, steps, -1)
    ig = rows.mean(axis=1)
    bar = BAR * np.abs(rows).max(axis=2).mean(axis=1)
    err = np.abs(attr.astype(np.float64) - ig).max(axis=1)
    return err / np.maximum(bar, 1e-300), ig, bar


@pytest.mark.parametrize("variant", ["shipped", "synthetic"])
def test_ig_within_bar_of_fp64(weights, windows, variant):
    w = weights[variant]
    tok = T.tokenize_windows(windows)
    c = engine.Classifier(w, device=0, max_batch=MB)
    try:
        c._attr_ctx(MB)
        pred = c.predict_ascii(torch.from_numpy(windows).cuda()).cpu().numpy()
        base_logp = {}
        worst = 0.0
        cases = [(m, b, list(range(len(windows))), (0, 1, 2)) for m in (1, 4) for b in I.BASELINES]
        cases += [(16, b, [0, 6, 8], (2,)) for b in I.BASELINES]
        for m, baseline, sel, targets in cases:
            lx, lb = I.endpoint_logits(tok[sel], w, baseline)
            for target in targets:
                probs, logp, attr, routes, masks, h2 = _gpu_ig(c, windows[sel], target, m, baseline)
                assert np.array_equal(probs, pred[sel]), "probabilities are not predict_ascii's"
                assert np.array_equal(logp[:, 0], logp_formula(probs, target))
                assert np.all(logp[:, 1] == logp[0, 1])
                key = (baseline, target)
                base_logp.setdefault(key, logp[0, 1])
                assert logp[0, 1] == base_logp[key], "log p_c(x') differs between calls"
                if target == targets[0]:
                    lg, J = _reference(tok[sel], w, m, baseline, routes, masks)
                logits = h2 @ w["d2w"].astype(np.float64) + w["d2b"].astype(np.float64)
                err, ig, bar = _check(attr, J, logits, target, m)
                worst = max(worst, err.max())
                print(f"\n{variant} m={m} {baseline} target {target}: error / bar " + " ".join(f"{e:.2f}" for e in err))
                assert err.max() <= 1.0, err
                if baseline == "N":
                    assert np.all(attr[tok[sel] == 0] == 0), "N-baseline IG must be 0 at token-0 positions"
                # completeness: the GPU's gap within fp64's at the same nodes plus the bar over the window
                delta = I.log_p(lx, target) - I.log_p(lb[None], target)[0]
                gap_ref = np.abs(ig.sum(axis=1) - delta)
                gap_gpu = np.abs(attr.astype(np.float64).sum(axis=1) - delta)
                assert np.all(gap_gpu <= gap_ref + bar * attr.shape[1]), (gap_gpu, gap_ref)
        print(f"\n{variant}: worst error / bar {worst:.3f}")
    finally:
        c.close()


def test_ig_on_confident_windows(weights, golden_dir):
    """Head-sharpened weights (d2w, d2b times k: the logits times k, nothing before the head changes) put golden windows at
    log-odds margins mu >= 40, where gradient x input is ~0 (mu < 104) or exactly 0: IG is nonzero there, meets the bar and
    adds up to log p_c(x) - log p_c(x') ~ -log p_c(x')."""
    asc = np.load(golden_dir / "reference_graph_golden.npz")["windows"]
    w0 = weights["shipped"]
    cases = [(4, 21, 1), (16, 16, 2), (16, 21, 1)]                  # (k, golden row, target): mu 48, 146, 194
    rows = sorted({r for _, r, _ in cases})
    tok = T.tokenize_windows(asc[rows])
    m = 16
    J = {}
    for k, r, target in cases:
        w = dict(w0)
        w["d2w"] = w0["d2w"] * np.float32(k)
        w["d2b"] = w0["d2b"] * np.float32(k)
        c = engine.Classifier(w, device=0, max_batch=MB)
        try:
            c._attr_ctx(MB)
            a = torch.from_numpy(asc[rows]).cuda()
            _, gi = c.attribute_ascii(a, target)
            for baseline in I.BASELINES:
                probs, logp, attr, routes, masks, h2 = _gpu_ig(c, asc[rows], target, m, baseline)
                if baseline not in J:                             # the rows before the head do not depend on k
                    J[baseline] = _reference(tok, w0, m, baseline, routes, masks)[1]
                i = rows.index(r)
                lx, lb = I.endpoint_logits(tok, w0, baseline)
                mu = k * (lx[i, target] - np.delete(lx[i], target).max())
                assert mu >= 40, mu
                logits = h2 @ w["d2w"].astype(np.float64) + w["d2b"].astype(np.float64)
                err, ig, bar = _check(attr, J[baseline], logits, target, m, scale=k)
                delta = I.log_p(lx, target, k) - I.log_p(lb[None], target, k)[0]
                gap_ref = abs(ig[i].sum() - delta[i])
                gap = abs(float(attr[i].astype(np.float64).sum()) - delta[i])
                print(f"\nk={k} row {r} target {target} {baseline}: mu {mu:.0f}, max |grad x input| "
                      f"{np.abs(gi[i].cpu().numpy()).max():.1e}, max |IG| {np.abs(attr[i]).max():.2e}, error / bar "
                      f"{err[i]:.2f}, sum IG {attr[i].sum():.4f} vs -log p_c(x') {-logp[i, 1]:.4f} (fp64 delta {delta[i]:.4f})")
                assert np.abs(attr[i]).max() > 0 and np.all(np.isfinite(attr[i]))
                assert err[i] <= 1.0
                assert gap <= gap_ref + bar[i] * attr.shape[1]
                assert -1e-15 < logp[i, 0] <= 0                                     # log p_c(x) is ~0 at such a margin
            if k == 16:
                assert torch.all(gi[rows.index(r)] == 0), "gradient x input is exactly 0 from mu ~ 104"
        finally:
            c.close()


def test_ig_bitwise_identities(weights, windows):
    w = weights["shipped"]
    a = torch.from_numpy(windows).cuda()
    big = engine.Classifier(w, device=0, max_batch=256)
    small = engine.Classifier(w, device=0, max_batch=64)
    try:
        big._attr_ctx(256)
        small._attr_ctx(64)
        m = 16
        for baseline in I.BASELINES:
            p1, l1, x1 = big.integrated_gradients_ascii(a, 2, m, baseline)          # one chunk of 16 windows
            p2, l2, x2 = small.integrated_gradients_ascii(a, 2, m, baseline)        # chunks of 4 windows
            assert torch.equal(x1, x2) and torch.equal(p1, p2) and torch.equal(l1, l2), "chunking"
            perm = torch.tensor([5, 0, 8, 3, 1, 7, 2, 6, 4], device="cuda")
            _, _, x3 = small.integrated_gradients_ascii(a[perm], 2, m, baseline)
            assert torch.equal(x3, x1[perm]), "window order"
            _, _, x4 = small.integrated_gradients_ascii(a[[2, 7]], 2, m, baseline)
            assert torch.equal(x4, x1[[2, 7]]), "batch composition"
            for opt in ("fuse_l1", "tail_overlap"):
                small.set_option(opt, 1 - small.get_option(opt))
                _, _, x5 = small.integrated_gradients_ascii(a, 2, m, baseline)
                small.set_option(opt, 1 - small.get_option(opt))
                assert torch.equal(x5, x1), opt
            assert torch.equal(p1, small.predict_ascii(a))
            small.check_status()
            big.check_status()
        # contigs and planned windows: the ASCII rows gathered beforehand
        rng = np.random.default_rng(9)
        seqs = [bytes(rng.choice(list(b"ACGTacgtN"), int(L))) for L in (2600, 6000, 13000, 800)]
        res = small.integrated_gradients_contigs(seqs, "plasmid", steps=4, baseline="N")
        seq, offs = small.contig_buffers(seqs)
        start, length, woff = small.contig_windows(seq, offs)
        rows = small.gather_windows(seq, start, length)
        pa, la, xa = small.integrated_gradients_ascii(rows, 1, 4, "N")
        assert torch.equal(res.attr, xa) and torch.equal(res.probs, pa) and torch.equal(res.logp, la)
        assert torch.equal(res.offsets, woff)
        # argument checks
        with pytest.raises(engine.GnmError, match="steps"):
            small.integrated_gradients_ascii(a[:1], 0, 65, "zero")
        with pytest.raises(ValueError):
            small.integrated_gradients_ascii(a[:1], 0, 4, "shuffled")
        small.set_option("conv_impl", 1)
        with pytest.raises(engine.GnmError, match="conv_impl"):
            small.integrated_gradients_ascii(a[:1], 0, 4, "zero")
        small.set_option("conv_impl", 0)
    finally:
        big.close()
        small.close()


def test_ig_fuse_gather_off_within_bar(weights, windows):
    w = weights["synthetic"]
    sel = [0, 6, 8]
    tok = T.tokenize_windows(windows[sel])
    c = engine.Classifier(w, device=0, max_batch=MB)
    try:
        c._attr_ctx(MB)
        c.set_option("fuse_gather", 0)
        m = 4
        probs, logp, attr, routes, masks, h2 = _gpu_ig(c, windows[sel], 2, m, "zero")
        _, J = _reference(tok, w, m, "zero", routes, masks)
        logits = h2 @ w["d2w"].astype(np.float64) + w["d2b"].astype(np.float64)
        err, _, _ = _check(attr, J, logits, 2, m)
        print(f"\nfuse_gather 0: error / bar " + " ".join(f"{e:.2f}" for e in err))
        assert err.max() <= 1.0
        assert np.array_equal(probs, c.predict_ascii(torch.from_numpy(windows[sel]).cuda()).cpu().numpy())
        c.check_status()
    finally:
        c.close()


def test_module_write_ig_attributions(tmp_path, golden_dir, monkeypatch):
    """nn_classification.main with --write-attributions virus --attribution-steps 8 on the reference module's toy input:
    predictions bitwise those of a run without the option, and the attributions NPZ (windows, IG rows, log_p_target) bitwise
    Classifier.integrated_gradients_contigs on the same contigs."""
    import shutil
    from genomad_b200 import _paths, nn_classification, sequence
    for k in ("GENOMAD_B200_ATTRIBUTIONS", "GENOMAD_B200_ATTRIBUTION_STEPS", "GENOMAD_B200_ATTRIBUTION_BASELINE",
              "GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS"):
        monkeypatch.delenv(k, raising=False)
    inp = golden_dir / "reference_module" / "input"
    runs = {}
    try:
        for name, kw in (("off", {}), ("on", {"write_attributions": "virus", "attribution_steps": 8})):
            out = tmp_path / name
            shutil.copytree(inp / "toy_find_proviruses", out / "toy_find_proviruses")
            nn_classification.main(inp / "toy.fna", out, False, 128, False, 2, False, False, **kw)
            runs[name] = _paths.NNOutputs("toy", out)
    finally:
        nn_classification.release_classifiers()
    for attr in ("nn_classification_npz_output", "provirus_nn_classification_npz_output"):
        a, b = np.load(getattr(runs["off"], attr)), np.load(getattr(runs["on"], attr))
        assert np.array_equal(a["predictions"], b["predictions"]), attr
    z = np.load(runs["on"].nn_classification_attributions_output)
    assert (str(z["method"]), int(z["steps"]), str(z["baseline"]), str(z["target"])) == ("integrated_gradients", 8, "zero", "virus")
    seqs = {sequence.accession(h): s for h, s in sequence.iter_fasta(inp / "toy.fna", strip_n=False)}
    c = engine.Classifier(None, device=0, max_batch=64)
    try:
        res = c.integrated_gradients_contigs([seqs[n] for n in z["contig_names"]], "virus", steps=8, baseline="zero")
        c.check_status()
        assert np.array_equal(res.contig.cpu().numpy(), z["window_contig"])
        assert np.array_equal(res.start.cpu().numpy(), z["window_start"])
        assert np.array_equal(res.length.cpu().numpy(), z["window_length"])
        assert np.array_equal(res.attr.cpu().numpy(), z["attributions"])
        assert np.array_equal(res.logp.cpu().numpy(), z["log_p_target"])
        assert len(z["attributions"]) > 0
    finally:
        c.close()
