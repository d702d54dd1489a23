"""
CPU self-test of the attribution backward pass's stage references and bars (no GPU; run with -s for the table).

* tests/attr_stage_ref.py, composed stage by stage, is attr_ref.decomposed (the kernels' decomposition) to fp64 rounding.
* The operand rows of conv3's backward output and conv2's backward accumulation over them are emulated from the packing code
  (test_stage_recipes.act_planes / conv_weight_planes and the recipe's passes), on golden windows with synthetic IGLOO weights
  and conv3's weights and bias times 2^k.  The old rule stored s_w g_z2 as it came: its lo8 correction (and, for small
  weights, its hi8 plane) fell into e4m3's subnormal range, and conv2's backward pass missed the conv_tc bar (at k = 0 the
  max bar; from k = -4 on both, by MARGIN).  The current rule stores s2 s_w g_z2, max in [1, 2), and must hold the
  conv_bwd_tc bars with MARGIN at every k, and conv_tc's RMS bar too.
* The fp32 CUDA-core stages (head, IGLOO, layer 1) are emulated in float32 on fp32 inputs; each must hold its bar in
  stage_ref.BARS with MARGIN and a mutant of each (a reduced-precision operand, a dropped path) must miss it by MARGIN, so the
  bars the GPU stage tests use (tests/test_gpu_attr_stages.py) are derived, not guessed.
"""
import numpy as np
import pytest
import torch

import attr_ref as A
import attr_stage_ref as S
import stage_ref as R
import test_stage_recipes as SR
from oracle import igloo_model as M
from oracle import tokenizer as T

D = torch.float64
F32 = torch.float32
MARGIN = SR.MARGIN
TARGET = 2


def _scaled(w, f):
    out = dict(w)
    for k in ("c3w", "c3b"):
        out[k] = (np.asarray(w[k], np.float64) * f).astype(np.float32)
    return out


@pytest.fixture(scope="module")
def base(weights_npz, golden_dir):
    w = M.load_npz_weights(weights_npz)
    tok = T.tokenize_windows(np.load(golden_dir / "reference_graph_golden.npz")["windows"][:4])
    return w, M.synthetic_igloo_weights(w), tok


def _forward(tok, w):
    """fp64 forward intermediates and the backward pass up to conv3's backward output, through attr_stage_ref"""
    with torch.no_grad():
        _, it = M.forward(tok, w, D, return_intermediates=True)
    routes = [r for r, _, _ in A.routing(tok, w)]
    h1 = R.dense_bn_relu(it["h0"], w, 0).value
    h2 = R.dense_bn_relu(h1, w, 1).value
    probs = R.head_softmax(h2, w).value
    g_out = S.head_backward(probs, h1, h2, w, TARGET).value
    lg = [it[f"ig{s}"]["mpi"] @ torch.as_tensor(w[f"ig{s}_w_qk"], dtype=D) for s in (0, 1)]
    q = [R.wv_pool(it[y], w[f"ig{s}_w_v"]).value for s, y in ((0, "y1"), (1, "y3"))]
    g_z3 = S.igloo_backward(g_out[:, 128:], lg[1], q[1], routes[1], w, 1, it["y3"] > 0).value
    s_w = torch.as_tensor(S.pow2_scale(g_z3.abs().amax(dim=(1, 2)).numpy(), -1))
    g_z2 = S.conv_backward(g_z3 * s_w.reshape(-1, 1, 1), w["c3w"], it["y2"] > 0).value          # s_w g_z2
    return dict(it=it, routes=routes, h1=h1, h2=h2, probs=probs, g_out=g_out, lg=lg, q=q, g_z3=g_z3, s_w=s_w, g_z2=g_z2)


def conv_bwd_emulate(g, W, scale):
    """conv_t_attr_kernel<kConvBwd> over the operand rows of scale * g (per window), as the kernel computes it: time-reversed
    rows, W[j]^T packed by the forward's weight split, e4m3 corrections first, then the fp16 main pass; fp32 out, / scale."""
    sc = torch.as_tensor(np.asarray(scale), dtype=D).reshape(-1, 1, 1)
    main_w, c1_w, c2_w, Sx = SR.conv_weight_planes(torch.as_tensor(W).transpose(1, 2), "fixed")
    hi, lo8, hi8 = SR.act_planes((g * sc).flip(1))
    acc = 0
    for c in range(0, 128, 16):
        sl = slice(c, c + 16)
        acc = acc + R._causal(lo8[..., sl].to(D), c1_w[:, sl].to(D)) + R._causal(hi8[..., sl].to(D), c2_w[:, sl].to(D))
    acc = acc + R._causal(hi.to(D), main_w.to(D))
    return (acc * 2.0 ** -Sx).float().to(D).flip(1) / sc


def test_composed_stages_are_the_decomposition(base):
    """attr_stage_ref's stages chained (with s2) reproduce attr_ref.decomposed to fp64 rounding."""
    w0, syn, tok = base
    for w, rows, target in ((w0, [0, 1], 2), (syn, [2, 3], 0)):
        ref = A.decomposed(tok[rows], w, target)
        got = S.compose(tok[rows], w, target)
        err = np.abs(got - ref).max(axis=1) / np.abs(ref).max(axis=1)
        assert err.max() < 1e-12, err


@pytest.fixture(scope="module")
def sweeps(base):
    _, syn, tok = base
    return {k: (_scaled(syn, 2.0 ** k), _forward(tok, _scaled(syn, 2.0 ** k))) for k in (0, -4, -8)}


def test_gz2_rows_old_rule_misses_and_s2_holds_the_conv_bar(sweeps):
    """conv2's backward pass over the stored g_z2 rows against fp64 over the exact s_w g_z2: storage plus accumulation."""
    rms_bar, max_bar = R.BARS["conv_bwd_tc"]
    rows, bad = [], []
    for k, (w, f) in sweeps.items():
        v = f["g_z2"]
        mask = f["it"]["y1"] > 0
        ref = S.conv_backward(v, w["c2w"], mask)
        s2 = S.pow2_scale(v.abs().amax(dim=(1, 2)).numpy(), 1)
        for rule, scale in (("old rule (s_w g_z2 as it comes)", np.ones(len(v))), ("s2 s_w g_z2, max in [1, 2)", s2)):
            d = S._lrelu_d(mask)
            m = R.metrics(conv_bwd_emulate(v, w["c2w"], scale) * d, ref, R.position_regions(len(v)))
            worst = max(x for key, x in m.items() if key.startswith("max"))
            if rule.startswith("old"):
                tc_rms, tc_max = R.BARS["conv_tc"]
                ok = m["rms"] > tc_rms or worst > tc_max
                if k <= -4:
                    ok = ok and (m["rms"] >= MARGIN * rms_bar or worst >= MARGIN * max_bar)
            else:
                ok = m["rms"] * MARGIN <= min(rms_bar, R.BARS["conv_tc"][0]) and worst * MARGIN <= max_bar
            rows.append((k, rule, float(v.abs().max()), m["rms"], worst, ok))
            if not ok:
                bad.append((k, rule, m))
    print(f"\n| conv3 x 2^k | g_z2 rows | max s_w g_z2 | rms err / rms scale (bar {rms_bar:.0e}) | max (bar {max_bar:.1e}) | ok |"
          "\n|---|---|---|---|---|---|")
    for k, rule, vmax, rms, mx, ok in rows:
        print(f"| {k} | {rule} | {vmax:.2e} | {rms:.2e} | {mx:.2e} | {'yes' if ok else 'NO'} |")
    assert not bad, bad


def _f32(x):
    return torch.as_tensor(np.asarray(x)).float().to(D)


def test_cuda_core_stage_bars(base, sweeps):
    """head, IGLOO#1 (with the g_z3 mask), IGLOO#0 and layer 1 in float32 against fp64 on the same fp32 inputs."""
    _, syn, tok = base
    w, f = sweeps[0]
    it = f["it"]
    probs, h1, h2, g_out = (_f32(f[k]) for k in ("probs", "h1", "h2", "g_out"))
    lg, q, y3m = [_f32(x) for x in f["lg"]], [_f32(x) for x in f["q"]], it["y3"] > 0
    g_z1 = _f32(S.conv_backward(f["g_z2"], w["c2w"], it["y1"] > 0).value)
    s_w = f["s_w"].numpy()
    gz3_32 = S.igloo_backward(g_out[:, 128:], lg[1], q[1], f["routes"][1], w, 1, y3m, F32).value.to(D)
    half_d1 = dict(w, d1w=np.asarray(w["d1w"]).astype(np.float16).astype(np.float32))
    cases = {
        "attr_head": (S.head_backward(probs, h1, h2, w, TARGET),
                      {"recipe": S.head_backward(probs, h1, h2, w, TARGET, F32).value,
                       "d1w in fp16": S.head_backward(probs, h1, h2, half_d1, TARGET, F32).value}),
        "attr_igloo": (S.igloo_backward(g_out[:, 128:], lg[1], q[1], f["routes"][1], w, 1, y3m),
                       {m or "recipe": S.igloo_backward(g_out[:, 128:], lg[1], q[1], f["routes"][1], w, 1, y3m, F32, m).value
                        for m in ("", "no patch path", "first routed channel")}),
        "attr_igloo ": (S.igloo_backward(g_out[:, :128], lg[0], q[0], f["routes"][0], w, 0),
                        {m or "recipe": S.igloo_backward(g_out[:, :128], lg[0], q[0], f["routes"][0], w, 0, dt=F32, mutant=m).value
                         for m in ("", "no patch path", "first routed channel")}),
        # IGLOO#1's output as conv3's backward pass reads it: s_w g_z3 in operand rows (hi16 + lo8 of 32 s_w g_z3, max in
        # [0.25, 0.5)); mutant: the rows without their lo8 plane
        "attr_gz3_rows": (R.Ref(*(x * f["s_w"].reshape(-1, 1, 1) for x in S.igloo_backward(g_out[:, 128:], lg[1], q[1],
                                                                                         f["routes"][1], w, 1, y3m))),
                          {"recipe": SR.store(_f32(gz3_32 * f["s_w"].reshape(-1, 1, 1)), True),
                           "hi16 only": SR.f16(32.0 * _f32(gz3_32 * f["s_w"].reshape(-1, 1, 1))).to(D) / 32.0}),
        "attr_layer1": (S.layer1(g_z1, tok, w, s_w),
                        {m or "recipe": S.layer1(g_z1, tok, w, s_w, F32, m).value for m in ("", "g_z1 in fp16")}),
    }
    print("\n| stage | case | rms | rms bar | max | max bar | ok |\n|---|---|---|---|---|---|---|")
    bad = []
    for key, (ref, got) in cases.items():
        rms_bar, max_bar = R.BARS[key.strip()]
        for case, g in got.items():
            m = R.metrics(g, ref, R.position_regions(len(tok)) if g.dim() == 3 else None)
            worst = max(x for k2, x in m.items() if k2.startswith("max"))
            if case == "recipe":
                ok = m["rms"] * MARGIN <= rms_bar and worst * MARGIN <= max_bar
            else:
                ok = m["rms"] >= MARGIN * rms_bar or worst >= MARGIN * max_bar
            print(f"| {key} | {case}{'' if case == 'recipe' else '  [mutant]'} | {m['rms']:.2e} | {rms_bar:.0e} | {worst:.2e} | "
                  f"{max_bar:.0e} | {'yes' if ok else 'NO'} |")
            if not ok:
                bad.append((key, case, m))
    assert not bad, bad
