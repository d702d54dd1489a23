"""
Head attributions on an H100 (run with `-m gpu -s` for the measured precision): gnm_attribute_head_* and
gnm_attribute_head_ig_* through engine.Head.

- The shipped tail as a C = 3 head (weights.shipped_head) gives bitwise the Classifier's attributions, integrated gradients
  and logp, for every target, both baselines, chunked and unchunked, and head probabilities bitwise the shipped ones.
- The head probabilities are bitwise Head.predict of the windows' embeddings; attributions and IG do not depend on the chunk
  size, the window order, fuse_l1 or tail_overlap; a target outside [0, C) is refused.
- Seeded heads at C = 2, 7 and 32 (head_ref.random_head), sharpened by powers of two (W2, b2 times k multiply every logit by
  k exactly), on the golden windows, every target, shipped and synthetic IGLOO weights, against the fp64 autograd reference
  (tests/head_attr_ref.py) along the GPU forward's routing, LeakyReLU branches and head ReLU branches, at the GPU forward's
  head logits: within 1e-4 of max |attr| per window up to a log-odds margin mu < 40, finite beyond, exactly 0 once every
  off-target p is 0.0f.  The bins are those of test_gpu_attr_confidence.py.
- IG at m = 64 against fp64 at the same nodes, with the completeness gap sum IG - (log p_c(x) - log p_c(x')) printed and
  checked against fp64's, log p_c in the form ig_logp_kernel states (gnm.h).
"""
from types import SimpleNamespace

import numpy as np
import pytest

import head_attr_ref as R
import head_ref as HR
import ig_ref as I

pytestmark = pytest.mark.gpu

BAR = 1e-4
SHARPEN = (1, 8, 64, 1024)          # powers of two: every logit times k, exactly


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch


@pytest.fixture(scope="module")
def weights(weights_npz):
    from oracle import igloo_model as M
    w = M.load_npz_weights(weights_npz)
    return {"shipped": w, "synthetic": M.synthetic_igloo_weights(w)}


@pytest.fixture(scope="module")
def golden(golden_dir):
    from oracle import tokenizer as T
    asc = np.load(golden_dir / "reference_graph_golden.npz")["windows"]
    return asc, T.tokenize_windows(asc)


def _windows(n, seed):
    rng = np.random.default_rng(seed)
    a = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, (n, 6000))].copy()
    gc = rng.uniform(0.3, 0.7, n)
    hi = rng.random((n, 6000)) < gc[:, None]
    a[hi] = np.frombuffer(b"GC", np.uint8)[rng.integers(0, 2, int(hi.sum()))]
    a[n // 2, 3000:] = ord("N")
    return a


def _head(arrays, C_, k=1):
    a = {key: np.asarray(v, dtype=np.float32) for key, v in arrays.items()}
    if k != 1:
        a["d2w"] = a["d2w"] * np.float32(k)
        a["d2b"] = a["d2b"] * np.float32(k)
    return SimpleNamespace(arrays=a, class_names=tuple(f"k{i}" for i in range(C_)))


def _eq(x, y):
    return np.array_equal(x.cpu().numpy(), y.cpu().numpy())


@pytest.mark.parametrize("variant", ["shipped", "synthetic"])
def test_shipped_head_is_bitwise_the_classifier(torch, weights, golden, variant):
    from genomad_b200 import engine, weights as W
    w = weights[variant]
    a = torch.from_numpy(np.concatenate([golden[0], _windows(13, 3)])).cuda()
    big = engine.Classifier(w, device=0, max_batch=512)       # one chunk: 37 windows, and 37 x 8 IG rows
    big._attr_ctx(512)
    small = engine.Classifier(w, device=0, max_batch=64)      # chunks of 8 windows, IG one window per chunk
    small._attr_ctx(8)
    try:
        heads = [engine.Head(c, W.shipped_head(w)) for c in (big, small)]
        for target in range(3):
            p0, a0 = big.attribute_ascii(a, target)
            for h, t in zip(heads, (target, W.SHIPPED_CLASSES[target])):
                p, hp, at = h.attribute_ascii(a, t)
                assert _eq(p, p0) and _eq(hp, p0) and _eq(at, a0), (variant, target)
            for baseline in ("zero", "N"):
                p0, l0, a0 = big.integrated_gradients_ascii(a, target, 8, baseline)
                for h in heads:
                    p, hp, lp, at = h.integrated_gradients_ascii(a, target, 8, baseline)
                    assert _eq(p, p0) and _eq(hp, p0) and _eq(lp, l0) and _eq(at, a0), (variant, target, baseline)
        big.check_status()
        small.check_status()
    finally:
        big.close()
        small.close()


def test_head_probs_and_independence(torch, weights):
    from genomad_b200 import engine
    w = weights["shipped"]
    arrays = HR.random_head(7, 17)
    asc = _windows(40, 5)
    a = torch.from_numpy(asc).cuda()
    perm = np.random.default_rng(2).permutation(len(asc))
    ap = torch.from_numpy(asc[perm]).cuda()
    one = engine.Classifier(w, device=0, max_batch=512)
    one._attr_ctx(512)
    other = engine.Classifier(w, device=0, max_batch=64)
    other._attr_ctx(16)
    other.set_option("fuse_l1", 1 - one.get_option("fuse_l1"))
    other.set_option("tail_overlap", 1 - one.get_option("tail_overlap"))
    try:
        h1, h2 = engine.Head(one, _head(arrays, 7)), engine.Head(other, _head(arrays, 7))
        pred = h1.predict(one.embed_ascii(a)[1])
        for target in (0, 3, 6):
            p, hp, at = h1.attribute_ascii(a, target)
            assert _eq(hp, pred) and _eq(p, one.predict_ascii(a))
            p2, hp2, at2 = h2.attribute_ascii(a, target)
            assert _eq(hp2, hp) and _eq(at2, at)
            _, hp3, at3 = h2.attribute_ascii(ap, f"k{target}")
            assert np.array_equal(hp3.cpu().numpy(), hp.cpu().numpy()[perm])
            assert np.array_equal(at3.cpu().numpy(), at.cpu().numpy()[perm])
            _, ihp, lp, ig = h1.integrated_gradients_ascii(a, target, 8, "N")
            assert _eq(ihp, pred)
            _, ihp2, lp2, ig2 = h2.integrated_gradients_ascii(ap, target, 8, "N")
            assert np.array_equal(ihp2.cpu().numpy(), pred.cpu().numpy()[perm])
            assert np.array_equal(lp2.cpu().numpy(), lp.cpu().numpy()[perm])
            assert np.array_equal(ig2.cpu().numpy(), ig.cpu().numpy()[perm])
        # planned windows of contigs: the same values as the ASCII rows of those windows
        rng = np.random.default_rng(4)
        seqs = [np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)].tobytes() for n in (13000, 6000, 2500)]
        rec = h1.attribute_contigs(seqs, 2)
        seq, offs = one.contig_buffers(seqs)
        start, length, _ = one.contig_windows(seq, offs)
        wa = one.gather_windows(seq, start, length)
        _, hpw, atw = h1.attribute_ascii(wa, 2)
        assert _eq(rec.attr, atw) and _eq(rec.head_probs, hpw) and _eq(rec.head_probs, h1.predict(one.embed_windows(seq, start, length)[1]))
        irec = h1.integrated_gradients_contigs(seqs, 2, 4, "zero")
        _, _, lpw, igw = h1.integrated_gradients_ascii(wa, 2, 4, "zero")
        assert _eq(irec.attr, igw) and _eq(irec.logp, lpw)
        # refusals: in Python, and by the C call itself
        for bad in (7, -1, "virus"):
            with pytest.raises(ValueError):
                h1.attribute_ascii(a, bad)
        lib = one.lib
        for bad in (7, -1):
            rc = lib.gnm_attribute_head_ascii(one._h, one._attr_ctx(), h1._hd, a.data_ptr(), 1, bad, None, None,
                                              torch.empty((1, 5997), device="cuda").data_ptr(), one._stream())
            assert rc != 0 and b"target must be a class of the head, in [0, 7)" in lib.gnm_last_error()
            rc = lib.gnm_attribute_head_ig_ascii(one._h, one._attr_ctx(), h1._hd, a.data_ptr(), 1, bad, 4, 0, None, None,
                                                 None, torch.empty((1, 5997), device="cuda").data_ptr(), one._stream())
            assert rc != 0 and b"target must be a class of the head" in lib.gnm_last_error()
        one.check_status()
        other.check_status()
    finally:
        one.close()
        other.close()


def _bin(mu):
    if mu < 0:
        return "A"
    if mu < 9:
        return "B"
    if mu < 17:
        return "C"
    if mu < 17.5:
        return "C/D"
    if mu < 40:
        return "D"
    return "-" if mu < 110 else "E"


@pytest.mark.parametrize("variant", ["shipped", "synthetic"])
def test_head_attributions_against_fp64(torch, weights, golden, variant):
    from genomad_b200 import engine
    w = weights[variant]
    asc, tok = golden
    n = len(asc)
    a = torch.from_numpy(asc).cuda()
    clf = engine.Classifier(w, device=0, max_batch=32)
    clf._attr_ctx(32)                                           # one chunk: the debug buffers hold every window
    bins, failures = {}, []
    try:
        for C_, seed in ((2, 21), (7, 22), (32, 23)):
            arrays = HR.random_head(C_, seed)
            head = engine.Head(clf, _head(arrays, C_))
            head.attribute_ascii(a, 0)
            clf.check_status()
            routes = [clf.debug_fetch(f"route{s}", n).cpu().numpy() for s in (0, 1)]
            masks = [(clf.debug_fetch(b, n) > 0).cpu().numpy() for b in ("attr_y1", "buf1", "buf0")]
            h1 = clf.debug_fetch("h1", n).cpu().numpy()
            hh = clf.debug_fetch("h2", n).cpu().numpy()               # the head's hidden rows
            head.close()
            logits = hh.astype(np.float64) @ arrays["d2w"].astype(np.float64) + arrays["d2b"].astype(np.float64)
            _, J = R.logit_jacobian(tok, R.with_head(w, arrays), routes=routes, masks=masks, head_masks=[h1 > 0, hh > 0])
            for k in SHARPEN:
                head = engine.Head(clf, _head(arrays, C_, k))
                for target in range(C_):
                    _, hp, at = head.attribute_ascii(a, target)
                    clf.check_status()
                    hp, at = hp.cpu().numpy(), at.cpu().numpy()
                    assert np.all(np.isfinite(at)), (variant, C_, k, target)
                    lg = k * logits
                    mu = lg[:, target] - np.delete(lg, target, axis=1).max(axis=1)
                    ref = R.rows_from_jacobian(logits, J, target, scale=k)
                    err = np.abs(at.astype(np.float64) - ref).max(axis=1) / np.maximum(np.abs(ref).max(axis=1), 1e-300)
                    for r in range(n):
                        b = _bin(mu[r])
                        off_zero = bool(np.all(np.delete(hp[r], target) == 0))
                        if b == "E" or off_zero:
                            bins.setdefault("E" if off_zero else b, []).append(0.0)
                            if off_zero and not np.all(at[r] == 0):
                                failures.append(f"C={C_} x{k} row {r} target {target}: off-target p all 0, attr not 0")
                        elif b == "-":
                            bins.setdefault(b, []).append(0.0)
                        else:
                            bins.setdefault(b, []).append(err[r])
                            if not err[r] <= BAR:
                                failures.append(f"C={C_} x{k} row {r} target {target} (bin {b}, mu {mu[r]:.1f}): {err[r]:.2e}")
                head.close()
    finally:
        clf.close()
    print(f"\n{variant}: " + "; ".join(f"bin {b}: {len(v)} cases, worst {max(v):.2e}" for b, v in sorted(bins.items())))
    for b in ("A", "B", "E"):
        assert b in bins, f"bin {b} is empty"
    assert any(b in bins for b in ("C", "C/D", "D")), "no confident case below mu 40"
    assert not failures, "\n".join(failures[:40])


def _logp_kernel_form(logits, c):
    """log p_c as ig_logp_kernel states it: -log1p(sum_{i != c} p_i) when p_c is the largest, log p_c otherwise"""
    lg = np.asarray(logits, dtype=np.float64)
    e = np.exp(lg - lg.max(axis=1, keepdims=True))
    p = e / e.sum(axis=1, keepdims=True)
    other = np.delete(p, c, axis=1)
    top = np.all(p[:, c:c + 1] >= other, axis=1)
    return np.where(top, -np.log1p(other.sum(axis=1)), np.log(p[:, c]))


def test_head_ig_against_fp64_at_the_same_nodes(torch, weights, golden):
    from genomad_b200 import engine
    w = weights["shipped"]
    asc, tok = golden[0][[3, 16]], golden[1][[3, 16]]
    m = 64
    arrays = HR.random_head(2, 31)
    hw = R.with_head(w, arrays)
    a = torch.from_numpy(asc).cuda()
    clf = engine.Classifier(w, device=0, max_batch=2 * m)
    clf._attr_ctx(2 * m)                                        # both windows' rows in one chunk
    try:
        head = engine.Head(clf, _head(arrays, 2))
        for baseline, target in (("zero", 0), ("N", 1)):
            _, _, lp, ig = head.integrated_gradients_ascii(a, target, m, baseline)
            clf.check_status()
            rows = 2 * m
            routes = [clf.debug_fetch(f"route{s}", rows).cpu().numpy() for s in (0, 1)]
            masks = [(clf.debug_fetch(b, rows) > 0).cpu().numpy() for b in ("attr_y1", "buf1", "buf0")]
            h1 = clf.debug_fetch("h1", rows).cpu().numpy()
            hh = clf.debug_fetch("h2", rows).cpu().numpy()
            logits = hh.astype(np.float64) @ arrays["d2w"].astype(np.float64) + arrays["d2b"].astype(np.float64)
            rt = np.repeat(tok, m, axis=0)
            al = np.tile((np.arange(m) + 0.5) / m, 2)
            _, J = R.logit_jacobian(rt, hw, alpha=al, baseline=baseline, routes=routes, masks=masks,
                                    head_masks=[h1 > 0, hh > 0])
            ref = R.rows_from_jacobian(logits, J, target).reshape(2, m, -1).mean(axis=1)
            ig, lp = ig.cpu().numpy().astype(np.float64), lp.cpu().numpy().astype(np.float64)
            err = np.abs(ig - ref).max(axis=1) / np.abs(ref).max(axis=1)
            # fp64 endpoints: log p_c at the windows and at the baseline
            lx, _ = R.logit_jacobian(tok, hw, baseline=baseline, batch=8)
            with torch.no_grad():
                lb = I.logits_onehot(I.interp_onehot(tok[:1], np.zeros(1), baseline), hw).numpy()
            # the endpoints in the form ig_logp_kernel states (gnm.h), evaluated on fp64 probabilities
            dp64 = _logp_kernel_form(lx, target) - _logp_kernel_form(lb, target)[0]
            gap, gap64 = ig.sum(axis=1) - (lp[:, 0] - lp[:, 1]), ref.sum(axis=1) - dp64
            print(f"\nC=2 target {target} baseline {baseline} m={m}: IG within {err.max():.2e} of max |IG|; completeness "
                  f"gap {np.array2string(gap, precision=4)} (fp64 at the same nodes {np.array2string(gap64, precision=4)}); "
                  f"log p_c(x), log p_c(x') {np.array2string(lp, precision=3)}", end="")
            assert np.all(err <= BAR), err
            # log p_c comes from the fp32 probabilities (gnm.h): exact to fp32 rounding while p_c is a normal number; a
            # p_c below FLT_MIN (log p_c < -87.3) keeps only the bits of a subnormal
            normal = np.all(lp > np.log(np.finfo(np.float32).tiny), axis=1)
            assert np.all(normal <= (np.abs(gap - gap64) <= 1e-3 * np.maximum(1.0, np.abs(ig).sum(axis=1)))), (gap, gap64)
            assert np.all(normal | (np.minimum(lp[:, 0], lp[:, 1]) < -80)), lp
        head.close()
    finally:
        clf.close()
