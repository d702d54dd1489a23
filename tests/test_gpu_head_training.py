"""
Head training on an H100 (gnm_head_train_*) against the fp64 statement in head_ref.py, step by step over whole runs and on
confidently classified batches.  Run with `-m gpu -s` for the per-step and per-bin errors.

Whole runs: a free-running fp64 trajectory would drift from the GPU's chaotically (Adam's nearly sign-like updates, e.g. on
d1b, whose gradient is rounding noise), so every step t is checked against fp64 from the GPU's own state before it: its
parameters and moving statistics (weights()) and Adam moments (fetch after step t - 1).  The schedule covers later steps of
Adam and of the dropout key, moving statistics away from 0 and 1, the partial last batch of an epoch, the batch sizes where
the GEMMs' 32-row and 64-row tiles end, repeated indices, a zero class weight, a class weight of 25, three learning rates,
and B = max_batch.

Confident batches: a head sharpened by 2^k (d2w, d2b times 2^k multiply every training-mode logit by 2^k exactly, in fp32 as
in fp64) gives batches across the range of the labelled class's log-odds margin mu = l_y - max_{c != y} l_c.  Past mu ~ 9,
p_y - 1 and log(sum e^(l - max)) cancel in fp32; the kernel's loss and dZ2 must keep their precision there.
"""
import numpy as np
import pytest

import head_ref as R

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                       # fp32 unit roundoff
PARAMS = ("d1w", "d1b", "bn1g", "bn1b", "d2w", "d2b")
N_WIN = 3000
N_TRAIN = 1000                       # three batches of 256 and a last one of 232 per epoch
MB = 256
B1, B2 = 0.9, 0.999


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch


def _windows(n, seed):
    rng = np.random.default_rng(seed)
    a = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, (n, 6000))].copy()
    gc = rng.uniform(0.3, 0.7, n)                      # vary composition so the embeddings spread
    hi = rng.random((n, 6000)) < gc[:, None]
    a[hi] = np.frombuffer(b"GC", np.uint8)[rng.integers(0, 2, int(hi.sum()))]
    return a


@pytest.fixture(scope="module")
def emb(torch):
    """(classifier, embeddings float32 cuda [N_WIN, 512], the same on the host)"""
    from genomad_b200 import engine, weights as W
    clf = engine.Classifier(W.load_weights(), device=0, max_batch=MB)
    _, X = clf.embed_ascii(torch.from_numpy(_windows(N_WIN, 21)).cuda())
    torch.cuda.synchronize()
    yield clf, X, X.cpu().numpy()
    clf.close()


def _ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)


def _grad_errors(g, ref_g, cache):
    """{name: (max error, scale)} with the scale of test_gpu_head.py's bar: max |g|, and for d1b the size of the terms its
    sum cancels"""
    out = {}
    for k, gr in ref_g.items():
        scale = np.abs(gr).max()
        if k == "d1b":
            # db1 = sum_r dz1 is zero in exact arithmetic (batch normalisation removes the bias: sum_r xh = 0); what is left is
            # the rounding of the fp32 terms it sums, so its scale is that of those terms
            scale = np.abs(cache["f"]["bn1g"] * cache["inv"] * (cache["mask"] / R.KEEP * (cache["y"] > 0))).max() * \
                np.abs(ref_g["bn1b"]).max()
        out[k] = (float(np.abs(g[k].astype(np.float64) - gr).max()), float(scale))
    return out


def _grad_ok(e):
    err, scale = e
    return err <= 1e-4 * scale or scale == 0 and err <= 1e-12


def check_step(tr, loss, X, idx, labels, cw, seed, t, lr, pre, prev_m, prev_v, tag):
    """Step t of trainer tr (just taken on rows idx, with batch loss `loss`) against fp64 from the GPU's state before it:
    pre = weights() before the step, prev_m / prev_v = the Adam moments after step t - 1.  Returns (loss, moments after the
    step)."""
    B = len(idx)
    mask = tr.fetch("mask").astype(bool)
    assert np.array_equal(mask, R.keep_mask(seed, t, B)), f"{tag}: dropout mask differs from the hash at step {t}"
    g, m, v = tr.fetch("grad"), tr.fetch("adam_m"), tr.fetch("adam_v")
    stats = tr.fetch("batch_stats").astype(np.float64)
    after = tr.weights()
    assert tr.steps == t + 1, (tag, tr.steps, t)
    Xb = X[idx]
    p0 = {k: pre[k] for k in PARAMS}
    ref_loss, cache = R.forward(p0, Xb, labels[idx], cw, mask)

    # batch statistics.  z1 is 512 fp32 FMAs per value: its error is below 4 sqrt(512) u sum_k |x_k w_k| (partial sums no
    # larger than that, roundings of independent sign), bounded per column by ez from the largest |x_k| of the batch
    W1 = p0["d1w"].astype(np.float64)
    ez = 4 * np.sqrt(512) * U * (np.abs(Xb).max(0).astype(np.float64) @ np.abs(W1) + np.abs(p0["d1b"]))
    mu, var = cache["mu"], cache["var"]
    e_mu = ez + U * np.abs(mu)                                       # the mean of values off by ez, rounded to fp32
    dev = np.abs(cache["z"] - mu).mean(0)
    d = 2 * ez + U * np.abs(mu)                                      # error of z - mu as the GPU forms it
    e_var = 2 * dev * d + d * d + U * var                            # mean of its square, rounded to fp32
    e_inv = 0.5 * cache["inv"] ** 3 * e_var + U * cache["inv"]
    for name, got, want, bar in (("mu", stats[0], mu, e_mu), ("inv", stats[1], cache["inv"], e_inv),
                                 ("var", stats[2], var, e_var)):
        assert (np.abs(got - want) <= 1.01 * bar).all(), (tag, t, name, float((np.abs(got - want) / bar).max()))

    # loss and gradients, test_gpu_head.py's bars
    if ref_loss == 0:
        assert loss == 0, (tag, t, loss)
    assert abs(loss - ref_loss) <= 1e-5 * abs(ref_loss), (tag, t, loss, ref_loss)
    errs = _grad_errors(g, R.backward(cache), cache)
    bad = {k: e for k, e in errs.items() if not _grad_ok(e)}
    assert not bad, (tag, t, bad)

    # Adam moments: the fp64 recurrence from the GPU's m_{t-1}, v_{t-1} and g_t.  m_t = m + (g - m) c1 rounds g - m, the
    # constant c1 = fl(1 - b1), the product and the sum: at most u (3 c1 |g - m| + |m_t|).  v_t rounds g^2, g^2 - v, c2,
    # the product and the sum: at most u (c2 (g^2 + 3 |g^2 - v|) + |v_t|).  1 % covers the second-order terms.
    for k in PARAMS:
        gk, mk, vk = (x.astype(np.float64) for x in (g[k], prev_m[k], prev_v[k]))
        m64 = mk + (gk - mk) * (1 - B1)
        v64 = vk + (gk * gk - vk) * (1 - B2)
        assert (np.abs(m[k] - m64) <= 1.01 * U * (3 * (1 - B1) * np.abs(gk - mk) + np.abs(m64))).all(), (tag, t, k, "m")
        assert (np.abs(v[k] - v64) <= 1.01 * U * ((1 - B2) * (gk * gk + 3 * np.abs(gk * gk - vk)) + v64)).all(), \
            (tag, t, k, "v")
        # the parameters: Adam from the GPU's own p_{t-1}, g_t, m_{t-1}, v_{t-1} at t + 1, within 1e-6 lr + half an ulp
        want, _, _ = R.adam(pre[k], g[k], prev_m[k], prev_v[k], t + 1, lr)
        assert (np.abs(after[k] - want) <= 1e-6 * lr + 0.5 * _ulp(want)).all(), (tag, t, k, "adam")

    # moving statistics: R.moving of the previous fp32 values and the fp64 batch statistics.  The GPU's 0.99 prev + 0.01 mu
    # rounds both constants, both products and the sum, and carries the statistic's own error
    mm, mv = R.moving(pre["bn1m"], pre["bn1v"], mu, var)
    for name, got, want, prev, stat, e_stat in (("bn1m", after["bn1m"], mm, pre["bn1m"], mu, e_mu),
                                                ("bn1v", after["bn1v"], mv, pre["bn1v"], var, e_var)):
        bar = 0.01 * e_stat + 2 * U * (0.99 * np.abs(prev) + 0.01 * np.abs(stat)) + U * np.abs(want)
        assert (np.abs(got - want) <= 1.01 * bar).all(), (tag, t, name, float((np.abs(got - want) / bar).max()))

    worst = max(errs, key=lambda k: errs[k][0] / max(errs[k][1], 1e-300))
    print(f"{tag} t={t} B={B}: loss {abs(loss - ref_loss) / max(abs(ref_loss), 1e-300):.1e}, worst gradient {worst} "
          f"{errs[worst][0] / max(errs[worst][1], 1e-300):.1e} of its scale")
    return loss, m, v


class _Trainer:
    """engine.HeadTrainer that keeps the device tensors of each step alive and the last loss at hand"""

    def __init__(self, torch, init, seed, lr, max_batch=MB):
        from genomad_b200 import engine
        self.torch, self.seed, self.lr = torch, seed, lr
        self.tr = engine.HeadTrainer(init, device=0, max_batch=max_batch, seed=seed, learning_rate=lr)
        self.keep = []

    def step(self, Xd, idx, labels_d, cw):
        t = self.torch
        i, c = t.from_numpy(np.ascontiguousarray(idx, np.int64)).cuda(), t.from_numpy(np.asarray(cw, np.float32)).cuda()
        self.keep.append((i, c))
        self.loss = self.tr.step(Xd, i, labels_d, c)


def _schedule(C, rng):
    """labels [N_WIN], class weights, and the run: [(idx, class weights)]"""
    p = np.r_[np.full(C - 1, 0.98 / (C - 1)), 0.02]                 # class C - 1 is rare and weighs 25
    labels = rng.choice(C, N_WIN, p=p).astype(np.int32)
    cw = rng.uniform(0.5, 2.0, C).astype(np.float32)
    cw[C - 1] = 25.0
    epochs = [[perm[s: s + MB] for s in range(0, N_TRAIN, MB)] for perm in (rng.permutation(N_TRAIN) for _ in range(2))]
    odd = [rng.choice(N_TRAIN, b, replace=False) for b in (1, 31, 32, 33, 63, 64, 65)]
    main = [b for pair in zip(epochs[0] + epochs[1], odd + [None]) for b in pair if b is not None]
    assert [len(b) for b in main] == [256, 1, 256, 31, 256, 32, 232, 33, 256, 63, 256, 64, 256, 65, 232]
    run = [(b, cw) for b in main]
    rep = rng.choice(N_TRAIN, 60, replace=True)
    run.append((rng.permutation(np.r_[rep, rep[:20], rep[:5]]), cw))                       # repeated indices
    zero = 0
    cw0 = cw.copy()
    cw0[zero] = 0.0
    run.append((rng.choice(np.nonzero(labels[:N_TRAIN] == zero)[0], 16, replace=False), cw0))   # its only label weighs 0
    return labels, cw, run


def _run_checked(torch, emb, init, C, seed, lr, labels, run, tag):
    _, Xd, X = emb
    labels_d = torch.from_numpy(labels).cuda()
    tr = _Trainer(torch, init, seed, lr)
    pre = {k: v.copy() for k, v in init.items()}
    zeros = {k: np.zeros_like(init[k]) for k in PARAMS}
    pm, pv = zeros, zeros
    for t, (idx, cw) in enumerate(run):
        tr.step(Xd, idx, labels_d, cw)
        loss, pm, pv = check_step(tr.tr, float(tr.loss.item()), X, idx, labels, cw, seed, t, lr, pre, pm, pv, tag)
        if not np.any(cw[labels[idx]]):
            assert loss == 0
            g = tr.tr.fetch("grad")
            assert all(not np.any(g[k]) for k in PARAMS), f"{tag} t={t}: a batch whose labels weigh 0 has a gradient"
        pre = tr.tr.weights()
    return pre


@pytest.mark.parametrize("C", [2, 5, 32])
def test_whole_runs_step_by_step_against_fp64(torch, emb, C):
    from genomad_b200 import engine, weights as W
    clf, Xd, X = emb
    rng = np.random.default_rng(500 + C)
    labels, cw, run = _schedule(C, rng)
    init = R.random_head(C, 60 + C)                                  # non-zero moving statistics
    seed = 1000 + C
    final = _run_checked(torch, emb, init, C, seed, 1e-3, labels, run, f"C={C} lr=1e-3")
    assert not np.allclose(final["bn1m"], init["bn1m"]) and not np.allclose(final["bn1v"], init["bn1v"])
    for lr in (1e-4, 1e-2):
        short = [(rng.choice(N_TRAIN, b, replace=False), cw) for b in (256, 64, 33, 256)]
        _run_checked(torch, emb, init, C, seed + 1, lr, labels, short, f"C={C} lr={lr:g}")

    # the same run without a read between steps (reads synchronise the stream): bitwise the same result
    labels_d = torch.from_numpy(labels).cuda()
    free = _Trainer(torch, init, seed, 1e-3)
    for idx, c in run:
        free.step(Xd, idx, labels_d, c)
    again = free.tr.weights()
    assert free.tr.steps == len(run)
    assert all(np.array_equal(again[k].view(np.uint32), final[k].view(np.uint32)) for k in final), \
        "a run without intermediate reads ended elsewhere"

    # the trained head, moving statistics included, is scored as head_ref.infer states it on both conv_impl routes
    ref = R.infer(final, X)
    for impl in (0, 1):
        clf.set_option("conv_impl", impl)
        head = engine.Head(clf, W.HeadFile(final, tuple(f"c{i}" for i in range(C)), ""))
        err = np.abs(head.predict(Xd).cpu().numpy().astype(np.float64) - ref).max()
        head.close()
        print(f"C={C} trained head, conv_impl {impl}: max |p - fp64| {err:.2e}")
        assert err <= 1e-5, (impl, err)
    clf.set_option("conv_impl", 0)


def test_step_at_max_batch_against_fp64(torch, emb):
    from genomad_b200 import engine
    _, Xd, X = emb
    C, seed, lr, B = 7, 77, 1e-3, 65536
    rng = np.random.default_rng(7)
    labels = rng.integers(0, C, N_WIN).astype(np.int32)
    cw = rng.uniform(0.5, 2.0, C).astype(np.float32)
    init = R.random_head(C, 8)
    tr = _Trainer(torch, init, seed, lr, max_batch=B)
    idx = rng.integers(0, N_WIN, B)                                  # with repeats
    tr.step(Xd, idx, torch.from_numpy(labels).cuda(), cw)
    zeros = {k: np.zeros_like(init[k]) for k in PARAMS}
    check_step(tr.tr, float(tr.loss.item()), X, idx, labels, cw, seed, 0, lr, init, zeros, zeros, f"C={C} B=max_batch")
    with pytest.raises(engine.GnmError, match="B must be in"):
        tr.step(Xd, np.zeros(B + 1, np.int64), torch.from_numpy(labels).cuda(), cw)


# ------------------------------------------------------------------------------------------------------- confident batches
BINS = (("mu < 0", -np.inf, 0.0), ("0 <= mu < 9", 0.0, 9.0), ("9 <= mu < 17", 9.0, 17.0),
        ("17.5 <= mu < 40", 17.5, 40.0), ("mu >= 110", 110.0, np.inf))


def _bin(mu):
    for name, lo, hi in BINS:
        if lo <= mu < hi:
            return name
    return "-"                       # 17..17.5 and 40..110: checked with the batch, not a bin of its own


def _sharpen(a, k):
    out = dict(a)
    out["d2w"], out["d2b"] = a["d2w"] * np.float32(2.0 ** k), a["d2b"] * np.float32(2.0 ** k)
    return out


@pytest.mark.parametrize("C", [2, 5, 32])
def test_confident_batches_against_fp64(torch, emb, C):
    """Two heads, each sharpened by 2^k for k = 0..7, one step of a fresh trainer on a batch of 256 labelled by the fp64
    argmax of its training-mode logits (with the GPU's dropout mask):
      spread    head_ref.random_head, 8 rows given a wrong label: every batch mixes margins;
      dominant  W2 / 128 and b2 = 0.98 on one class: every row's margin is 0.98 2^k within a few %, so the batch sits in one
                bin (k = 4: 9..17, k = 5: 17.5..40, k = 7: >= 110); k <= 3 with 8 wrong rows, k >= 4 all confident."""
    _, Xd, X = emb
    seed, B = 300 + C, 256
    rng = np.random.default_rng(900 + C)
    cw = rng.uniform(0.5, 2.0, C).astype(np.float32)
    spread = R.random_head(C, 70 + C)
    dominant = R.random_head(C, 80 + C)
    dominant["d2w"] = dominant["d2w"] * np.float32(2.0 ** -7)
    dominant["d2b"] = np.where(np.arange(C) == C // 2, np.float32(0.98), np.float32(0)).astype(np.float32)
    mask = R.keep_mask(seed, 0, B)
    cases, failures = [], []
    for kind, head in (("spread", spread), ("dominant", dominant)):
        for k in range(8):
            a = _sharpen(head, k)
            idx = rng.choice(N_WIN, B, replace=False)
            p0 = {n: a[n] for n in PARAMS}
            _, c0 = R.forward(p0, X[idx], np.zeros(B, int), cw, mask)
            lg = c0["logits"]
            y = lg.argmax(1)
            if kind == "spread" or k <= 3:
                wrong = rng.choice(B, 8, replace=False)
                y[wrong] = (y[wrong] + 1 + rng.integers(0, C - 1, 8)) % C
            labels = np.zeros(N_WIN, np.int32)
            labels[idx] = y
            r = np.arange(B)
            mu = lg[r, y] - np.where(np.arange(C)[None, :] == y[:, None], -np.inf, lg).max(1)
            bins = [_bin(m) for m in mu]
            tr = _Trainer(torch, a, seed, 1e-3)
            tr.step(Xd, idx, torch.from_numpy(labels).cuda(), cw)
            assert np.array_equal(tr.tr.fetch("mask").astype(bool), mask)
            g = tr.tr.fetch("grad")
            loss = float(tr.loss.item())
            ref_loss, cache = R.forward(p0, X[idx], y, cw, mask)
            errs = _grad_errors(g, R.backward(cache), cache)
            e_loss = abs(loss - ref_loss) / ref_loss if ref_loss else abs(loss)
            finite = np.isfinite(loss) and all(np.all(np.isfinite(g[n])) for n in PARAMS)
            pure = bins[0] if len(set(bins)) == 1 else None
            name = f"C={C} {kind} x2^{k}"
            if not finite:
                failures.append(f"{name}: loss or gradient not finite")
            if pure == "mu >= 110":
                # every other e is 0.0f: the loss and dZ2, so every gradient, are exactly 0 (fp64 keeps ~e^-mu); the
                # recorded "errors" are |loss| and max |g|
                errs = {n: (float(np.abs(g[n]).max()), 0.0) for n in PARAMS}
                cases.append((name, bins, pure, abs(loss), errs))
                print(f"\n{name}: mu {mu.min():.1f} .. {mu.max():.1f} ({pure}), loss {loss!r}, max |g| "
                      f"{max(e[0] for e in errs.values()):.1e}", end="")
                if loss != 0 or any(e[0] for e in errs.values()):
                    failures.append(f"{name}: loss {loss!r}, max |g| {max(e[0] for e in errs.values()):.1e} in bin >= 110")
                continue
            cases.append((name, bins, pure, e_loss, errs))
            rel = {n: e[0] / e[1] if e[1] else e[0] for n, e in errs.items()}
            worst = max(rel, key=rel.get)
            print(f"\n{name}: mu {mu.min():.1f} .. {mu.max():.1f} ({pure or 'mixed'}), loss {loss!r}: error {e_loss:.1e}, "
                  f"worst gradient {worst} {rel[worst]:.1e}", end="")
            if not e_loss <= 1e-5:
                failures.append(f"{name}: loss {loss!r} against {ref_loss!r} ({e_loss:.1e})")
            for n, e in errs.items():
                if not _grad_ok(e):
                    failures.append(f"{name}: {n} {e[0]:.2e} against max |g| {e[1]:.2e} ({e[0] / e[1]:.1e})")
    print()
    for b, _, _ in BINS:
        rows = sum(bins.count(b) for _, bins, _, _, _ in cases)
        pure = [c for c in cases if c[2] == b]
        mixed = [c for c in cases if c[2] is None and b in c[1]]
        line = f"C={C} bin {b}: {rows} rows"
        for what, cs in (("pure batches", pure), ("mixed batches", mixed)):
            if cs:
                el = max(c[3] for c in cs)
                eg = max(e[0] / e[1] if e[1] else e[0] for c in cs for e in c[4].values())
                line += f"; {len(cs)} {what}: loss {el:.1e}, gradients {eg:.1e} of max |g|"
        print(line)
        assert rows, f"C={C}: no row in bin {b}"
    for b in ("9 <= mu < 17", "17.5 <= mu < 40", "mu >= 110"):
        assert any(c[2] == b for c in cases), f"C={C}: no batch lies wholly in bin {b}"
    assert not failures, "\n".join(failures)
