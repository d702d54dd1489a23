"""
Novelty attributions on an H100 (run with `-m gpu -s` for the measured ratios, completeness gaps and the motif share):
gnm_attribute_novelty_* and gnm_attribute_novelty_ig_* through engine.Head.

- Heads fitted on the encoder's own embeddings of composition contigs (C = 2, 3, 7, 32), scored on typical windows of the same
  generators (D ~ 1) and on novel ones (the golden windows, GC-skewed random windows: D >> 1), every target drawn at random.
- Bitwise: the probabilities are predict_ascii's, the distances Head.novelty(embed_ascii(...)), IG's dist_target[:, 0] each
  window's distance to its target, and the h1 the seed reads is embed_ascii's.
- Stages (tests/novelty_attr_ref.py): the seed g_h1 within its derived bound of fp64 on the GPU's own h1; each attribution row
  within 1e-4 of max |row| of the fp64 vector-Jacobian product sum_j g_h1[j] h1(x)[j] along the GPU forward's routing,
  LeakyReLU branches and h1 > 0 mask (the bar of test_gpu_head_attr.py for the same backward pass), for gradient x input and
  for IG rows at the same nodes.
- Invariance: the same bits under another batch composition, order and chunking (chunks across max_batch), and refusals.
- Reported, not asserted: the IG completeness gap at m = 8, 32 and 64, and the share of positive attribution mass on the
  planted motif's 4-mers for motif contigs scored against a head that never saw them.
"""
import numpy as np
import pytest

import novelty_attr_ref as NA

pytestmark = pytest.mark.gpu

BAR = 1e-4


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch


@pytest.fixture(scope="module")
def w(weights_npz):
    from oracle import igloo_model as M
    return M.load_npz_weights(weights_npz)


@pytest.fixture(scope="module")
def clf(torch, w):
    from genomad_b200 import engine
    c = engine.Classifier(w, device=0, max_batch=256)
    c._attr_ctx(128)
    yield c
    c.close()


def _composition(clf, seed, per_class, classes=("gc35", "gc65", "motif")):
    """(embeddings [W, 512], composition class [W], ASCII windows [W, 6000]) of the windows of seeded composition contigs"""
    import test_gpu_head_module as HM
    rng = np.random.default_rng(seed)
    seqs, cls = [], []
    for _ in range(per_class):
        for c, kind in enumerate(classes):
            seqs.append(HM._contig(rng, kind))
            cls.append(c)
    seq, offs = clf.contig_buffers(seqs)
    start, length, woff = clf.contig_windows(seq, offs)
    X = clf.embed_windows(seq, start, length)[1].cpu().numpy()
    asc = clf.gather_windows(seq, start, length).cpu().numpy()
    return X, np.repeat(np.array(cls, np.int32), np.diff(woff.cpu().numpy())), asc


@pytest.fixture(scope="module")
def comp(clf):
    return _composition(clf, 7, 16)


def _fit_head(torch, clf, X, y, C, seed=0):
    from genomad_b200 import engine, weights as W
    fit = engine.novelty_fit(clf, torch.from_numpy(X).cuda(), torch.arange(len(X), dtype=torch.int64, device="cuda"),
                             torch.from_numpy(y).cuda(), C)
    h = engine.Head(clf, W.HeadFile(W.initial_head(C, seed), tuple(f"c{i}" for i in range(C)), ""))
    h.set_novelty(fit.center, fit.whitening, fit.means)
    return h, fit


def _labels(y, C, seed):
    """composition classes split into C labels, every label used"""
    rng = np.random.default_rng(seed)
    lab = (y * C // 3 + rng.integers(0, max(1, C // 3), len(y))) % C if C > 3 else np.minimum(y, C - 1)
    lab[:C] = np.arange(C)
    return lab.astype(np.int32)


def _novel_windows(golden_dir, n, seed):
    z = np.load(golden_dir / "reference_graph_golden.npz")["windows"][:n // 2]
    rng = np.random.default_rng(seed)
    r = np.frombuffer(b"ACGT", np.uint8)[rng.choice(4, (n - len(z), 6000), p=[0.45, 0.05, 0.05, 0.45])].copy()
    r[0, 2500:] = ord("N")
    return np.concatenate([z, r])


def _eq(x, y):
    return np.array_equal(x.cpu().numpy() if hasattr(x, "cpu") else x, y.cpu().numpy() if hasattr(y, "cpu") else y)


def _forward_state(clf, rows):
    routes = [clf.debug_fetch(f"route{s}", rows).cpu().numpy() for s in (0, 1)]
    masks = [(clf.debug_fetch(b, rows) > 0).cpu().numpy() for b in ("attr_y1", "buf1", "buf0")]
    return routes, masks, clf.debug_fetch("h1", rows).cpu().numpy(), clf.debug_fetch("attr_g_h1", rows).cpu().numpy()


@pytest.mark.parametrize("C", [2, 3, 7, 32])
def test_attributions_bitwise_and_stages(torch, clf, w, comp, golden_dir, C):
    from oracle import tokenizer as T
    X, y, asc_c = comp
    head, fit = _fit_head(torch, clf, X, _labels(y, C, C), C)
    rng = np.random.default_rng(C)
    asc = np.concatenate([asc_c[rng.choice(len(asc_c), 10, replace=False)], _novel_windows(golden_dir, 10, C)])
    n = len(asc)
    a = torch.from_numpy(asc).cuda()
    tg = rng.integers(0, C, n).astype(np.int32)
    try:
        probs, dist, attr = head.attribute_novelty_ascii(a, tg)
        clf.check_status()
        routes, masks, h1, g_h1 = _forward_state(clf, n)
        emb = clf.embed_ascii(a)[1]
        assert _eq(probs, clf.predict_ascii(a)) and _eq(dist, head.novelty(emb)) and _eq(h1, emb)
        D = dist.cpu().numpy()
        dmin = D.min(1)
        assert dmin[:10].max() < 5 and (dmin[10:] > 50).sum() >= 4, (dmin[:10], dmin[10:])
        g, bound = NA.grad_bound(h1, fit.center, fit.whitening, fit.means, tg)
        seed_ratio = NA.grad_ratio(g_h1, g, bound)
        ref = NA.encoder_vjp(T.tokenize_windows(asc), w, g_h1, routes=routes, masks=masks, h1_mask=h1 > 0)
        at = attr.cpu().numpy().astype(np.float64)
        err = np.abs(at - ref).max(1) / np.abs(ref).max(1)
        print(f"\nC={C}: D typical {np.median(dmin[:10]):.2f}, novel up to {dmin[10:].max():.0f}; seed / bound {seed_ratio:.3f}; "
              f"backward within {err.max():.2e} of max |attr|", end="")
        assert seed_ratio <= 1.0
        assert np.all(err <= BAR), err
        assert np.all(np.isfinite(at))
    finally:
        head.close()


def test_integrated_gradients_at_the_same_nodes(torch, clf, w, comp, golden_dir):
    from oracle import tokenizer as T
    X, y, asc_c = comp
    head, fit = _fit_head(torch, clf, X, _labels(y, 3, 3), 3)
    asc = np.concatenate([asc_c[:1], _novel_windows(golden_dir, 2, 1)[:1]])
    tok = T.tokenize_windows(asc)
    a = torch.from_numpy(asc).cuda()
    tg = np.array([int(y[0]), 2], np.int32)
    gaps = {}
    try:
        _, dist0, _ = head.attribute_novelty_ascii(a, tg)
        probs0 = clf.predict_ascii(a)                          # before the loop: a forward rewrites the debug buffers
        # D_c(x') is one baseline row's distance to each window's own target
        _, _, dt, _ = head.integrated_gradients_novelty_ascii(a, tg, 4, "N")
        _, _, dts, _ = head.integrated_gradients_novelty_ascii(a, np.full(2, tg[1], np.int32), 4, "N")
        assert np.all(dts.cpu().numpy()[:, 1] == dt.cpu().numpy()[1, 1])
        for m in (8, 32, 64):
            for baseline in ("zero", "N"):
                probs, dist, dt, ig = head.integrated_gradients_novelty_ascii(a, tg, m, baseline)
                clf.check_status()
                assert _eq(dist, dist0) and _eq(probs, probs0)
                assert _eq(dt[:, 0], dist.cpu().numpy()[np.arange(2), tg])
                ig, dt = ig.cpu().numpy().astype(np.float64), dt.cpu().numpy().astype(np.float64)
                gaps[(m, baseline)] = ig.sum(1) - (dt[:, 0] - dt[:, 1])
                if m != 8:
                    continue
                rows = 2 * m
                routes, masks, h1, g_h1 = _forward_state(clf, rows)
                rt = np.repeat(tg, m)
                g, bound = NA.grad_bound(h1, fit.center, fit.whitening, fit.means, rt)
                assert NA.grad_ratio(g_h1, g, bound) <= 1.0
                al = np.tile((np.arange(m) + 0.5) / m, 2)
                ref = NA.encoder_vjp(np.repeat(tok, m, axis=0), w, g_h1, alpha=al, baseline=baseline, routes=routes,
                                     masks=masks, h1_mask=h1 > 0).reshape(2, m, -1).mean(1)
                err = np.abs(ig - ref).max(1) / np.abs(ref).max(1)
                assert np.all(err <= BAR), (baseline, err)
    finally:
        head.close()
    print("\ncompleteness gap sum IG - (D_c(x) - D_c(x')) [typical, novel]: " +
          "; ".join(f"m={m} {b}: {np.array2string(v, precision=3)}" for (m, b), v in gaps.items()), end="")


def test_invariance_and_refusals(torch, w, comp, golden_dir):
    from genomad_b200 import engine
    X, y, asc_c = comp
    asc = np.concatenate([asc_c[:20], _novel_windows(golden_dir, 20, 5)])
    perm = np.random.default_rng(2).permutation(len(asc))
    one = engine.Classifier(w, device=0, max_batch=256)
    one._attr_ctx(256)
    other = engine.Classifier(w, device=0, max_batch=64)
    other._attr_ctx(16)                                        # 40 windows in chunks of 16; IG m = 4 in chunks of 4
    try:
        h1, _ = _fit_head(torch, one, X, _labels(y, 7, 7), 7)
        h2, _ = _fit_head(torch, other, X, _labels(y, 7, 7), 7)
        tg = np.random.default_rng(3).integers(0, 7, len(asc)).astype(np.int32)
        a, ap = torch.from_numpy(asc).cuda(), torch.from_numpy(asc[perm]).cuda()
        p, d, at = h1.attribute_novelty_ascii(a, tg)
        p2, d2, at2 = h2.attribute_novelty_ascii(ap, tg[perm])
        assert _eq(p2, p.cpu().numpy()[perm]) and _eq(d2, d.cpu().numpy()[perm]) and _eq(at2, at.cpu().numpy()[perm])
        sub = slice(5, 11)
        _, _, at3 = h1.attribute_novelty_ascii(a[sub], tg[sub])
        assert _eq(at3, at.cpu().numpy()[sub])
        _, _, dt, ig = h1.integrated_gradients_novelty_ascii(a, tg, 4, "N")
        _, _, dt2, ig2 = h2.integrated_gradients_novelty_ascii(ap, tg[perm], 4, "N")
        assert _eq(dt2, dt.cpu().numpy()[perm]) and _eq(ig2, ig.cpu().numpy()[perm])
        # a class name, and planned windows of contigs: the same values as the ASCII rows of those windows
        _, _, atc = h1.attribute_novelty_ascii(a, "c3")
        _, _, atc2 = h1.attribute_novelty_ascii(a, np.full(len(asc), 3))
        assert _eq(atc, atc2)
        import test_gpu_head_module as HM
        rng = np.random.default_rng(4)
        seqs = [HM._contig(rng, k) for k in ("gc35", "motif", "gc65")]
        rec = h1.attribute_novelty_contigs(seqs)
        dist, counts = h1.novelty_contigs(seqs)
        _, nearest, _ = engine.novelty_scores(dist.cpu().numpy(), counts.cpu().numpy(), np.zeros(0, np.float32))
        assert _eq(rec.target, np.repeat(nearest, counts.cpu().numpy()))
        seq, offs = one.contig_buffers(seqs)
        start, length, _ = one.contig_windows(seq, offs)
        wa = one.gather_windows(seq, start, length)
        _, dw, atw = h1.attribute_novelty_ascii(wa, rec.target.cpu().numpy())
        assert _eq(rec.attr, atw) and _eq(rec.head_probs, dw)
        irec = h1.integrated_gradients_novelty_contigs(seqs, 4, "zero")
        _, _, dtw, igw = h1.integrated_gradients_novelty_ascii(wa, rec.target.cpu().numpy(), 4, "zero")
        assert _eq(irec.attr, igw) and _eq(irec.logp, dtw)
        # refusals: a target outside [0, C), in Python and by the C call (naming the index); a head without a model;
        # conv_impl = 1
        bad = tg.copy()
        bad[5] = 7
        with pytest.raises(ValueError, match=r"target\[5\] = 7"):
            h1.attribute_novelty_ascii(a, bad)
        lib, out = one.lib, torch.empty((len(asc), 5997), device="cuda")
        for v in (7, -1):
            bad[5] = v
            rc = lib.gnm_attribute_novelty_ascii(one._h, one._attr_ctx(), h1._hd, a.data_ptr(), len(asc), engine._ptr(bad),
                                                 None, None, out.data_ptr(), one._stream())
            assert rc != 0 and f"target[5] = {v} is not a class of the head, in [0, 7)".encode() in lib.gnm_last_error()
            rc = lib.gnm_attribute_novelty_ig_ascii(one._h, one._attr_ctx(), h1._hd, a.data_ptr(), len(asc), engine._ptr(bad),
                                                    4, 0, None, None, None, out.data_ptr(), one._stream())
            assert rc != 0 and b"target[5]" in lib.gnm_last_error()
        from genomad_b200 import weights as W
        plain = engine.Head(one, W.HeadFile(W.initial_head(7, 0), tuple(f"c{i}" for i in range(7)), ""))
        with pytest.raises(engine.GnmError, match="no novelty model"):
            plain.attribute_novelty_ascii(a, 0)
        with pytest.raises(engine.GnmError, match="no novelty model"):
            plain.integrated_gradients_novelty_ascii(a, 0, 4)
        plain.close()
        one.set_option("conv_impl", 1)
        with pytest.raises(engine.GnmError, match="conv_impl = 0"):
            h1.attribute_novelty_ascii(a, tg)
        one.set_option("conv_impl", 0)
        assert _eq(h1.attribute_novelty_ascii(a, tg)[2], at)
        one.check_status()
        other.check_status()
        h1.close()
        h2.close()
    finally:
        one.close()
        other.close()


def test_planted_motif_share(torch, clf):
    """Report only: a head fitted on gc35 and gc65; motif contigs are novel, and their windows' attributions to the distance to
    the nearest class should sit on the planted motif (24 % of the bases)."""
    import test_gpu_head_module as HM
    X, y, _ = _composition(clf, 9, 12, classes=("gc35", "gc65"))
    head, _ = _fit_head(torch, clf, X, y, 2)
    rng = np.random.default_rng(10)
    seqs = [HM._contig(rng, "motif") for _ in range(4)]
    try:
        rec = head.attribute_novelty_contigs(seqs)
        irec = head.integrated_gradients_novelty_contigs(seqs, 32, "zero")
    finally:
        head.close()
    start = rec.start.cpu().numpy()
    out = []
    for name, r in (("gradient x input", rec), ("IG m=32", irec)):
        at = r.attr.cpu().numpy()
        on_tot, pos_tot, frac = 0.0, 0.0, []
        for i in range(len(at)):
            t = start[i] + np.arange(at.shape[1])
            L = len(seqs[int(r.contig[i])])
            on = ((t % 50) <= 12 - 4) & (t - t % 50 + 12 < L)     # 4-mer inside a motif copy (TTAGGGTTAGGG every 50 nt)
            p = np.maximum(at[i], 0)
            on_tot += p[on].sum()
            pos_tot += p.sum()
            frac.append(on.mean())
        out.append(f"{name}: {on_tot / max(pos_tot, 1e-30):.1%} of positive mass on motif 4-mers ({np.mean(frac):.1%} of tokens)")
    print("\n" + "; ".join(out) + f"; median D {np.median(rec.head_probs.cpu().numpy().min(1)):.0f}", end="")


def test_module_runs_on_the_composition_set(torch, clf, tmp_path):
    """nn-classification --head with a novelty head fitted on composition-contig embeddings, on held-out contigs of the same
    generators: the per-sequence segment mean of the attribution file's distance is bitwise the novelty file's novelty; at
    stride 6000 the window novelty rows' per-sequence means are bitwise its distances; at stride 1000 the rows are bitwise
    Head.novelty of embed_windows."""
    import test_gpu_head_module as HM
    from genomad_b200 import _paths, engine, nn_classification as nnc, weights as W
    X, y, _ = _composition(clf, 12, 8)
    _, fit = _fit_head(torch, clf, X, y, 3)
    hp = tmp_path / "h.npz"
    W.save_head(hp, W.initial_head(3, 0), HM.CLASSES, W.load_weights(),
                novelty={"novelty_center": fit.center, "novelty_whitening": fit.whitening, "novelty_means": fit.means,
                         "novelty_calibration": np.sort(np.random.default_rng(0).uniform(0.5, 3, 19)).astype(np.float32)})
    fa = tmp_path / "in.fna"
    HM.write_set(fa, 13, 3)
    nnc.main(fa, tmp_path / "a", False, 128, False, 2, False, False, head=hp, write_novelty_attributions=True,
             write_window_novelty=True)
    nnc.main(fa, tmp_path / "b", False, 128, False, 2, False, False, head=hp, write_window_novelty=True, window_stride=1000)
    oa, ob = _paths.NNOutputs("in", tmp_path / "a"), _paths.NNOutputs("in", tmp_path / "b")
    za = np.load(oa.nn_classification_head_novelty_attributions_output)
    nv = np.load(oa.nn_classification_head_novelty_npz_output)
    zw = np.load(oa.nn_classification_head_novelty_windows_npz_output)
    counts = np.bincount(za["window_contig"], minlength=len(nv["contig_names"]))
    offs = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)).cuda()
    head = engine.Head(clf, W.load_head(hp, W.load_weights()))
    try:
        m = head.segment_mean(torch.from_numpy(za["distance"][:, None].copy()).cuda(), offs).cpu().numpy()[:, 0]
        assert np.array_equal(m, nv["novelty"]) and np.array_equal(za["target_class"], np.repeat(nv["nearest_class"], counts))
        assert np.isfinite(za["attributions"]).all()
        md = head.segment_mean(torch.from_numpy(zw["distances"]).cuda(), offs).cpu().numpy()
        assert np.array_equal(md, nv["distances"])
        z1 = np.load(ob.nn_classification_head_novelty_windows_npz_output)
        seqs = [s for _, s in _read_fasta(fa)]
        seq, o2 = clf.contig_buffers(seqs)
        start, length, _ = clf.contig_windows(seq, o2, stride=1000)
        ref = head.novelty(clf.embed_windows(seq, start, length)[1]).cpu().numpy()
        assert z1["distances"].shape == ref.shape and np.array_equal(z1["distances"], ref)
        assert np.array_equal(z1["novelty"], ref.min(1)) and np.array_equal(z1["nearest_class"], ref.argmin(1))
    finally:
        head.close()
    print(f"\nmodule: {len(za['distance'])} attributed windows, {len(z1['distances'])} stride-1000 windows; median novelty "
          f"{np.median(nv['novelty']):.2f}", end="")


def _read_fasta(path):
    name, out = None, []
    for line in open(path):
        line = line.strip()
        if line.startswith(">"):
            name = line[1:].split()[0]
            out.append([name, ""])
        elif line:
            out[-1][1] += line
    return [(n, s) for n, s in out]
