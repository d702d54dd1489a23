"""
Classifier heads on an H100: inference (gnm_head_forward, gnm_head_segment_*) bitwise against the shipped classifier and
against fp64 for random heads, and one training step (gnm_head_train_step) against the fp64 statement in head_ref.py.
"""
import numpy as np
import pytest

import head_ref as R

pytestmark = pytest.mark.gpu

MB = 256


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch


@pytest.fixture(scope="module")
def w():
    from genomad_b200 import weights as W
    return W.load_weights()


def _windows(n, seed):
    rng = np.random.default_rng(seed)
    a = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, (n, 6000))].copy()
    gc = rng.uniform(0.3, 0.7, n)                      # vary composition so the embeddings spread
    hi = rng.random((n, 6000)) < gc[:, None]
    a[hi] = np.frombuffer(b"GC", np.uint8)[rng.integers(0, 2, int(hi.sum()))]
    a[n // 2, 3000:] = ord("N")
    return a


@pytest.fixture(scope="module")
def runs(torch, w):
    """Per conv_impl: (classifier, probabilities [3000, 3] of predict_ascii, embeddings [3000, 512] of embed_ascii)."""
    from genomad_b200 import engine
    a = torch.from_numpy(_windows(3000, 1)).cuda()
    out = {}
    for impl in (0, 1):
        clf = engine.Classifier(w, device=0, max_batch=MB)
        clf.set_option("conv_impl", impl)
        probs = clf.predict_ascii(a)
        _, emb = clf.embed_ascii(a)
        torch.cuda.synchronize()
        out[impl] = (clf, probs, emb)
    return out


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("n", [1, 127, 128, 129, MB, MB + 1, 3000])
def test_shipped_head_is_bitwise_the_classifier(runs, w, impl, n):
    from genomad_b200 import engine, weights as W
    clf, probs, emb = runs[impl]
    head = engine.Head(clf, W.shipped_head(w))
    hp = head.predict(emb[:n])
    assert hp.shape == (n, 3)
    assert np.array_equal(hp.cpu().numpy().view(np.uint32), probs[:n].cpu().numpy().view(np.uint32))


@pytest.mark.parametrize("impl", [0, 1])
def test_shipped_head_segment_reductions_are_bitwise(torch, runs, w, impl):
    from genomad_b200 import engine, weights as W
    clf, probs, emb = runs[impl]
    head = engine.Head(clf, W.shipped_head(w))
    rng = np.random.default_rng(3)
    cuts = np.sort(rng.choice(np.arange(1, 3000), 40, replace=False))
    off = torch.tensor(np.r_[0, cuts, cuts[-1], 3000].astype(np.int32), device="cuda")     # one empty contig
    hp = head.predict(emb)
    assert np.array_equal(head.segment_mean(hp, off).cpu().numpy(), clf.segment_mean(probs, off).cpu().numpy())
    assert np.array_equal(head.segment_sum(hp, off).cpu().numpy(), clf.segment_sum(probs, off).cpu().numpy())


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("C", [2, 7, 32])
def test_random_head_against_fp64(torch, runs, impl, C):
    from genomad_b200 import engine, weights as W
    clf, _, emb = runs[impl]
    a = R.random_head(C, 10 + C)
    head = engine.Head(clf, W.HeadFile(a, tuple(f"c{i}" for i in range(C)), ""))
    got = head.predict(emb).cpu().numpy().astype(np.float64)
    ref = R.infer(a, emb.cpu().numpy())
    err = np.abs(got - ref)
    print(f"C={C} impl={impl}: max {err.max():.3e}, p99.9 {np.quantile(err, 0.999):.3e}, median {np.median(err):.3e}")
    assert err.max() <= 1e-5
    off = np.array([0, 5, 5, 900, 3000], np.int32)
    mean = head.segment_mean(torch.from_numpy(got.astype(np.float32)).cuda(), torch.from_numpy(off).cuda()).cpu().numpy()
    for c in range(4):
        s = np.zeros(C, np.float32)
        for i in range(off[c], off[c + 1]):
            s = (s + got[i].astype(np.float32)).astype(np.float32)
        want = s / np.float32(max(off[c + 1] - off[c], 1))
        assert np.array_equal(mean[c], want)


TRAIN_MB = 1024


@pytest.mark.parametrize("C", [2, 3, 32])
@pytest.mark.parametrize("B", [1, 2, 255, 256, 257, TRAIN_MB])
def test_training_step_against_fp64(torch, runs, C, B):
    from genomad_b200 import engine
    X = runs[0][2]
    rng = np.random.default_rng(100 * C + B)
    init = R.random_head(C, C)
    init["bn1m"], init["bn1v"] = np.zeros(512, np.float32), np.ones(512, np.float32)
    labels = rng.integers(0, C - 1, X.shape[0]).astype(np.int32)        # class C - 1 never occurs
    cw = rng.uniform(0.5, 2.0, C).astype(np.float32)
    idx = rng.choice(X.shape[0], B, replace=False).astype(np.int64)
    lr, seed = 1e-3, 7
    tr = engine.HeadTrainer(init, device=0, max_batch=TRAIN_MB, seed=seed, learning_rate=lr)
    loss = tr.step(X, torch.from_numpy(idx).cuda(), torch.from_numpy(labels).cuda(), torch.from_numpy(cw).cuda())
    loss = float(loss.item())
    mask = tr.fetch("mask").astype(bool)
    assert np.array_equal(mask, R.keep_mask(seed, 0, B)), "dropout mask differs from the hash"
    g = tr.fetch("grad")
    after = tr.weights()
    p0 = {k: init[k] for k in ("d1w", "d1b", "bn1g", "bn1b", "d2w", "d2b")}
    ref_loss, cache = R.forward(p0, X.cpu().numpy()[idx], labels[idx], cw, mask)
    assert abs(loss - ref_loss) <= 1e-5 * abs(ref_loss), (loss, ref_loss)
    ref_g = R.backward(cache)
    for k, gr in ref_g.items():
        scale = np.abs(gr).max()
        if k == "d1b":
            # db1 = sum_r dz1 is zero in exact arithmetic (batch normalisation removes the bias: sum_r xh = 0); what is left is
            # the rounding of the fp32 terms it sums, so its scale is that of those terms
            scale = np.abs(cache["f"]["bn1g"] * cache["inv"] * (cache["mask"] / R.KEEP * (cache["y"] > 0))).max() * \
                np.abs(ref_g["bn1b"]).max()
        err = np.abs(g[k] - gr).max()
        print(f"C={C} B={B} {k}: max|g| {scale:.3e}, err {err:.3e}")
        assert err <= 1e-4 * scale or scale == 0 and err <= 1e-12, (k, err, scale)
    # Adam from the GPU's own gradients.  A parameter is stored in fp32, so the bar adds half an ulp of the result
    for k in p0:
        want, _, _ = R.adam(p0[k], g[k], 0, 0, 1, lr)
        ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
        assert (np.abs(after[k] - want) <= 1e-6 * lr + 0.5 * ulp).all(), k
    mm, mv = R.moving(np.zeros(512), np.ones(512), cache["mu"], cache["var"])
    assert np.abs(after["bn1m"] - mm).max() <= 1e-6 * max(np.abs(mm).max(), 1e-30) + 1e-12
    assert np.abs(after["bn1v"] - mv).max() <= 1e-6 * np.abs(mv).max()


def test_training_is_bitwise_reproducible(torch, runs):
    from genomad_b200 import engine
    X = runs[0][2]
    C = 5
    rng = np.random.default_rng(0)
    labels = torch.from_numpy(rng.integers(0, C, X.shape[0]).astype(np.int32)).cuda()
    cw = torch.from_numpy(rng.uniform(0.5, 2.0, C).astype(np.float32)).cuda()
    batches = [torch.from_numpy(rng.choice(X.shape[0], 200, replace=False).astype(np.int64)).cuda() for _ in range(50)]
    from genomad_b200 import weights as W

    def run(seed):
        tr = engine.HeadTrainer(W.initial_head(C, 3), device=0, max_batch=256, seed=seed)
        for b in batches:
            tr.step(X, b, labels, cw)
        return tr.weights()
    a, b, c = run(11), run(11), run(12)
    assert all(np.array_equal(a[k], b[k]) for k in a)
    assert not np.array_equal(a["d1w"], c["d1w"])


@pytest.mark.parametrize("bad", ["label", "index"])
def test_out_of_range_inputs_are_reported(torch, runs, bad):
    """A label outside [0, C) or a batch index outside [0, N) is not read; the trainer reports it at its next call."""
    from genomad_b200 import engine, weights as W
    X = runs[0][2]
    labels = np.zeros(X.shape[0], np.int32)
    idx = np.arange(8, dtype=np.int64)
    if bad == "label":
        labels[3] = 4
    else:
        idx[5] = X.shape[0]
    tr = engine.HeadTrainer(W.initial_head(4, 0), device=0, max_batch=8)
    tr.step(X, torch.from_numpy(idx).cuda(), torch.from_numpy(labels).cuda(), torch.ones(4, device="cuda"))
    with pytest.raises(engine.GnmError, match="label outside" if bad == "label" else "batch index outside"):
        tr.weights()
