"""
Stage-by-stage precision of the attribution backward pass on the GPU (run with `-m gpu -s` for the tables).

Every backward stage's output, fetched with gnm_debug_fetch ("attr_*"), is compared with its fp64 reference on the kernel's OWN
input (tests/attr_stage_ref.py), with the region maxima of stage_ref.position_regions: positions 0-5 and 5991-5996 are where the
time reversal and the TMA zero fill meet.  Bars: stage_ref.BARS, derived by tests/test_attr_stage_recipes_cpu.py.

    head      probabilities, h1, h2               -> attr_g_out                   attr_head
    IGLOO#1   g_out, logits1, q1, route1, y3 > 0  -> attr_gz3 / s_w (+ the pack)  attr_gz3_rows (the rows' storage format)
    conv3 bwd attr_gz3, W3, y2 > 0, s2            -> attr_gz2                     conv_bwd_tc
    IGLOO#0   g_out, logits0, q0, route0          -> attr_gy1                     attr_igloo
    conv2 bwd attr_gz2 / s2, W2, y1 > 0, s_w g_y1 -> attr_gz1                     conv_bwd_tc
    layer 1   attr_gz1, tokens, s_w               -> attributions                 attr_layer1

The matrix: shipped and synthetic weights, targets 0/1/2, golden windows, N runs, the all-N window and a short tail, chunk sizes
1, 7 and chunk + 3; the forward's conv3 weight-scale sweep; and the compensated family W3, b3 x 2^k with IGLOO#1's w_v and
w_mult x 2^-k, the same model by LeakyReLU homogeneity, whose s2 s_w g_z2 rows are the same bits at every k.
"""
import numpy as np
import pytest
import torch

import attr_ref as A
import attr_stage_ref as S
import stage_ref as R
from oracle import igloo_model as M
from oracle import tokenizer as T

pytestmark = pytest.mark.gpu

MB = 8


@pytest.fixture(scope="module")
def shipped(weights_npz):
    return M.load_npz_weights(weights_npz)


@pytest.fixture(scope="module")
def windows(golden_dir):
    """golden windows, N runs, an all-N window and a short padded tail"""
    g = np.load(golden_dir / "reference_graph_golden.npz")["windows"][:4]
    rng = np.random.default_rng(23)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    runs = acgt[rng.integers(0, 4, 6000)].copy()
    runs[700:1500] = ord("N"); runs[5000:5090] = ord("N")
    alln = np.full(6000, ord("N"), dtype=np.uint8)
    tail = acgt[rng.integers(0, 4, 6000)].copy()
    tail[1200:] = ord("N")
    return np.concatenate([g, runs[None], alln[None], tail[None]])          # 7 windows


def _scaled(w, **factors):
    out = dict(w)
    for k, f in factors.items():
        out[k] = (np.asarray(w[k], np.float64) * f).astype(np.float32)
    return out


def _attribute(c, asc, target):
    """attribute_ascii, with the last chunk's forward and backward buffers as fp64 CPU tensors (IGLOO#1's logits from a
    predict_ascii of the same windows: the attribution call's forward is that step, bit for bit)"""
    n = len(asc)
    last0 = (n - 1) // c.attr_max_batch * c.attr_max_batch
    m = n - last0
    a = torch.from_numpy(asc).cuda()
    c.predict_ascii(a[last0:])
    c.check_status()
    logits1 = c.debug_fetch("logits", m)[:, :R.N_POOL].double().cpu()
    probs, attr = c.attribute_ascii(a, target)
    c.check_status()

    def f(name):
        return c.debug_fetch(name, m).double().cpu()
    got = {k: f(k) for k in ("h1", "h2", "q0", "q1", "mpi1", "h0", "attr_y1", "buf1", "buf0", "attr_g_out", "attr_s_w",
                             "attr_s2", "attr_gz3", "attr_gz2", "attr_gy1", "attr_gz1")}
    got.update(logits1=logits1, logits0=f("logits")[:, :R.N_POOL], probs=probs[last0:].double().cpu(),
               attr=attr[last0:].double().cpu(), route0=c.debug_fetch("route0", m).cpu().numpy(),
               route1=c.debug_fetch("route1", m).cpu().numpy(), last0=last0, probs_all=probs, attr_all=attr)
    return got


def _check(label, w, asc, target, got):
    """every backward stage against its bar; one table row per stage; returns the misses"""
    tok = T.tokenize_windows(asc[got["last0"]:])
    n = len(tok)
    reg = R.position_regions(n)
    reg["pos 5991-5996"] = (slice(None), slice(5991, 5997))
    s_w, s2 = got["attr_s_w"], got["attr_s2"]
    y1m, y2m, y3m = got["attr_y1"] > 0, got["buf1"] > 0, got["buf0"] > 0
    checks = [
        ("head", "attr_head", got["attr_g_out"], S.head_backward(got["probs"], got["h1"], got["h2"], w, target), {}),
        ("IGLOO#1 -> s_w g_z3 rows", "attr_gz3_rows", got["attr_gz3"],
         R.Ref(*(x * s_w.reshape(-1, 1, 1) for x in S.igloo_backward(got["attr_g_out"][:, 128:], got["logits1"], got["q1"],
                                                                     got["route1"], w, 1, y3m))), reg),
        ("conv3 bwd -> s2 s_w g_z2 rows", "conv_bwd_tc", got["attr_gz2"],
         S.conv_backward(got["attr_gz3"], w["c3w"], y2m, out_scale=s2), reg),
        ("IGLOO#0 -> g_y1", "attr_igloo", got["attr_gy1"],
         S.igloo_backward(got["attr_g_out"][:, :128], got["logits0"], got["q0"], got["route0"], w, 0), reg),
        ("conv2 bwd -> s_w g_z1", "conv_bwd_tc", got["attr_gz1"],
         S.conv_backward(got["attr_gz2"], w["c2w"], y1m, got["attr_gy1"], s_w, 1.0 / s2), reg),
        ("layer 1 -> attr", "attr_layer1", got["attr"], S.layer1(got["attr_gz1"], tok, w, s_w), {}),
    ]
    bad = []
    for stage, key, g, ref, regions in checks:
        m = R.metrics(g, ref, regions)
        rms_bar, max_bar = R.BARS[key]
        worst = max(v for k, v in m.items() if k.startswith("max"))
        ok = m["rms"] <= rms_bar and worst <= max_bar
        per_region = ", ".join(f"{k[4:]} {v:.1e}" for k, v in m.items() if k.startswith("max ")) or "-"
        print(f"| {label} | {stage} | {m['rms']:.2e} | {rms_bar:.0e} | {m['max']:.2e} | {max_bar:.1e} | {per_region} | "
              f"{'ok' if ok else 'MISS'} |")
        if not ok:
            bad.append((label, stage, m))
    # the two scales are the powers of two the kernels promise
    gz3max, gz2max = got["attr_gz3"].abs().amax(dim=(1, 2)), got["attr_gz2"].abs().amax(dim=(1, 2))
    live = gz3max > 0
    assert torch.all((gz3max[live] >= 0.25) & (gz3max[live] <= 0.5)), (label, gz3max)
    assert torch.all((gz2max[live] >= 1) & (gz2max[live] <= 2)), (label, gz2max)
    assert torch.equal(torch.frexp(s_w)[0], torch.full_like(s_w, 0.5)) and torch.equal(torch.frexp(s2)[0], torch.full_like(s2, 0.5))
    return bad


def _attr_vs_fp64(w, asc, target, got):
    """per-window max |attr - fp64| / max |fp64| along the GPU's routing and LeakyReLU branches"""
    tok = T.tokenize_windows(asc[got["last0"]:])
    masks = [(got[k] > 0).numpy() for k in ("attr_y1", "buf1", "buf0")]
    ref = A.attribution(tok, w, target, routes=[got["route0"], got["route1"]], masks=masks)
    return np.abs(got["attr"].numpy() - ref).max(axis=1) / np.maximum(np.abs(ref).max(axis=1), 1e-300)


HEADER = ("\n| configuration | stage | rms err / rms scale | bar | max err / sum abs terms | bar | max per region | |"
          "\n|---|---|---|---|---|---|---|---|")


@pytest.mark.parametrize("variant", ["shipped", "synthetic"])
def test_backward_stages(shipped, windows, variant):
    from genomad_b200 import engine
    w = shipped if variant == "shipped" else M.synthetic_igloo_weights(shipped)
    c = engine.Classifier(w, device=0, max_batch=MB)
    try:
        c._attr_ctx(MB)
        print(HEADER)
        bad = []
        for target in (0, 1, 2):
            bad += _check(f"{variant}, target {target}", w, windows, target, _attribute(c, windows, target))
        for n in (1, 7, MB + 3):                                            # chunk sizes; the last chunk is checked
            asc = np.concatenate([windows] * 2)[:n]
            bad += _check(f"{variant}, n = {n}, chunk {MB}", w, asc, 2, _attribute(c, asc, 2))
        assert not bad, bad
    finally:
        c.close()


@pytest.mark.parametrize("k", [-8, -6, -4, -2, 0, 1, 2])
def test_conv3_weight_scale_sweep(shipped, windows, k):
    """conv3's weights and bias x 2^k (the forward's own sweep): every backward stage within its bar, attributions within
    1e-4 of fp64.  With s_w g_z2 stored as it came, conv3 x 2^-4 already lost g_z2's lo8 correction."""
    from genomad_b200 import engine
    w = _scaled(M.synthetic_igloo_weights(shipped), c3w=2.0 ** k, c3b=2.0 ** k)
    c = engine.Classifier(w, device=0, max_batch=MB)
    try:
        c._attr_ctx(MB)
        got = _attribute(c, windows, 2)
        print(HEADER)
        bad = _check(f"conv3 x 2^{k}", w, windows, 2, got)
        err = _attr_vs_fp64(w, windows, 2, got)
        print(f"\nconv3 x 2^{k}: max |s_w g_z2| {float((got['attr_gz2'].abs().amax(dim=(1, 2)) / got['attr_s2']).max()):.2e}; "
              "attributions vs fp64: " + " ".join(f"{e:.1e}" for e in err))
        assert not bad, bad
        assert err.max() <= 1e-4, err
    finally:
        c.close()


FWD = ("q1", "mpi1", "logits1", "h0", "h1", "h2", "probs", "attr_y1", "buf1", "buf0")


def test_compensated_conv3_scale(shipped, windows):
    """W3, b3 x 2^k with IGLOO#1's w_v and w_mult x 2^-k: the same model.  From conv3 x 2^-8 (the forward sweep's floor) up to
    the largest k with 32 max |y3| 2^k < 65504: no range error, probabilities within 1e-4 of the oracle with the same class
    calls, every stage within its bar, attributions within 1e-4 of fp64, and where the forward's buffers are bitwise those of
    k = 0, the attributions and the g_z2 rows are bitwise too."""
    from genomad_b200 import engine
    asc = windows[:4]
    tok = T.tokenize_windows(asc)
    _, it = M.forward(tok, shipped, torch.float32, return_intermediates=True)
    k_top = int(np.floor(np.log2(65504 / (32 * float(it["y3"].abs().max())))))
    oracle = M.forward(tok, shipped, torch.float32)
    runs, bad = {}, []
    print(HEADER)
    for k in [0] + [k for k in range(-8, k_top + 1) if k != 0]:
        f, g = 2.0 ** k, 2.0 ** -k
        w = _scaled(shipped, c3w=f, c3b=f, ig1_w_v=g, ig1_w_mult=g)
        c = engine.Classifier(w, device=0, max_batch=MB)
        try:
            c._attr_ctx(MB)
            got = _attribute(c, asc, 2)
        finally:
            c.close()
        p = got["probs"].numpy()
        assert np.abs(p - oracle).max() <= 1e-4 and np.array_equal(p.argmax(1), oracle.argmax(1)), (k, p, oracle)
        bad += _check(f"compensated k = {k}", w, asc, 2, got)
        err = _attr_vs_fp64(w, asc, 2, got)
        assert err.max() <= 1e-4, (k, err)
        runs[k] = got
        same_fwd = all(torch.equal(got[b], runs[0][b] * (2.0 ** k if b == "buf0" else 1)) for b in FWD)
        same_attr = torch.equal(got["attr"], runs[0]["attr"])
        gz2 = float((got["attr_gz2"].abs().amax(dim=(1, 2)) / got["attr_s2"]).max())
        print(f"| compensated k = {k} | max |s_w g_z2| = {gz2:.3e} | forward bitwise k = 0: {same_fwd} | "
              f"attributions bitwise: {same_attr} | worst attr err {err.max():.1e} | | |")
        if same_fwd:
            assert same_attr and torch.equal(got["attr_gz2"], runs[0]["attr_gz2"]), k
    assert not bad, bad


def test_integrated_gradients_compensated(shipped, windows):
    """Integrated gradients (the same backward rows) on the compensated set at k = 2, which saturated the g_z2 rows' hi8 plane
    before they had a scale of their own: no range error, and the unscaled model's probabilities, log p and attributions
    within 1e-4 (the forward is not bitwise: y3 entries in fp16's subnormal range do not scale exactly)."""
    from genomad_b200 import engine
    a = torch.from_numpy(windows[:2]).cuda()
    out = []
    for k in (0, 2):
        f, g = 2.0 ** k, 2.0 ** -k
        w = _scaled(shipped, c3w=f, c3b=f, ig1_w_v=g, ig1_w_mult=g)
        c = engine.Classifier(w, device=0, max_batch=16)
        try:
            c._attr_ctx(16)
            out.append(c.integrated_gradients_ascii(a, 2, steps=8))
            c.check_status()
        finally:
            c.close()
    (p0, l0, a0), (p2, l2, a2) = out
    assert float((p0 - p2).abs().max()) <= 1e-4 and float((l0 - l2).abs().max()) <= 1e-4
    err = ((a2 - a0).abs().amax(dim=1) / a0.abs().amax(dim=1)).cpu().numpy()
    print(f"\nintegrated gradients, compensated k = 2 against k = 0: " + " ".join(f"{e:.1e}" for e in err))
    assert err.max() <= 1e-4, err
