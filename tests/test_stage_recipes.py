"""
CPU self-test of the stage bars (no GPU).  Each tensor-core recipe is emulated from the library's packing code (gnm_create in
csrc/api.cu, the activation planes of csrc/common.cuh): the operands are formed exactly as the kernels form them, with torch's
float16 / float8_e4m3fn / TF32 rounding, and the products are summed in fp64.  The same is done for mutants of each recipe -- a
dropped correction pass, a single pass, truncated TF32 operands, and the conv corrections added after the main pass into an
accumulator that keeps only 14 significant bits (the Hopper hazard: e4m3 products reach the accumulator with reduced precision) --
and for conv and w_v weights scaled down until the old operand scaling rules (conv: d <= 16, hi = fp16(W); w_v: no scaling at all)
left their lo planes subnormal.  Two CUDA-core references are emulated too: the fp32 validation conv (768 sequential fp32 FMAs per
output) and a model of the 3 x TF32 GEMMs whose accumulator truncates to fp32 after every K = 8 step of the tensor core.

The test asserts that every recipe meets its bar in tests/stage_ref.py with at least 2x margin and that every mutant misses it by at
least 2x, so the bars the GPU stage tests use are derived rather than guessed.  Run with -s for the table.
"""
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import stage_ref as R
from oracle import igloo_model as M
from oracle import tokenizer as T

D = torch.float64
MARGIN = 2.0


# ------------------------------------------------------------------------------------------ operand formats
def f16(x):
    return x.float().half().float()


def e4m3(x):
    return x.float().clamp(-448.0, 448.0).to(torch.float8_e4m3fn).float()      # SATFINITE, round to nearest even


def tf32_trunc(x):
    return (x.float().view(torch.int32) & ~0x1FFF).view(torch.float32)


def tf32_rn(x):
    b = x.float().view(torch.int32)
    return ((b + 0x0FFF + ((b >> 13) & 1)) & ~0x1FFF).view(torch.float32)


def trunc_sig(x, bits=14):
    """x rounded toward zero to `bits` significant bits (a model of an accumulator with reduced precision)."""
    m, e = torch.frexp(x.to(D))
    return torch.ldexp(torch.trunc(m * 2.0 ** bits) / 2.0 ** bits, e)


# ------------------------------------------------------------------------------------------ conv: fp16 main + 2 x e4m3 corrections
def conv_weight_planes(W, rule):
    """The three weight planes gnm_create packs for one conv layer and the common exponent S of the passes.
    rule "fixed": shift may go negative (d up to 40) and hi is split from the scaled weight; "old": shift >= 0 and hi = fp16(W)."""
    W = W.float()
    wmax = float(W.abs().max())
    shift = math.ceil(math.log2(np.float32(wmax) / np.float32(0.78)))
    if rule == "old":
        d = 16 - max(0, shift)
        S = 5 + d
        whi = f16(W)
        return f16(whi * 2.0 ** d), e4m3(whi * 2.0 ** (S - 12)), e4m3((W - whi) * 2.0 ** (S - 7)), S
    d = min(16 - shift, 40)
    S = 5 + d
    ws = W * 2.0 ** d
    hi = f16(ws)
    return hi, e4m3(hi * 2.0 ** -7), e4m3((ws - hi) * 2.0 ** -2), S


def act_planes(y):
    """hi16, lo8, hi8 of Y = 32 y (the conv's operand planes, common.cuh)."""
    Y = (32.0 * y).float()
    hi = f16(Y)
    return hi, e4m3((Y - hi) * 128.0), e4m3(hi * 4.0)


def store(y, out_fp8):
    """The value a consumer (and gnm_debug_fetch) sees: hi16 + lo8 (conv2) or hi16 + lo16 (everything else) of Y = 32 y."""
    Y = (32.0 * y).float()
    hi = f16(Y)
    lo = e4m3((Y - hi) * 128.0) / 128.0 if out_fp8 else f16(Y - hi)
    return (hi.to(D) + lo.to(D)) / 32.0


def conv_emulate(y, W, b, rule="fixed", variant="recipe", out_fp8=True):
    main_w, c1_w, c2_w, S = conv_weight_planes(torch.as_tensor(W), rule)
    hi, lo8, hi8 = act_planes(y)
    c = R._causal
    main = c(hi.to(D), main_w.to(D))
    if variant == "single pass":
        acc = main
    elif variant == "no Alo*Whi":
        acc = main + c(hi8.to(D), c2_w.to(D))
    elif variant == "no Ahi*Wlo":
        acc = main + c(lo8.to(D), c1_w.to(D))
    else:
        # the e4m3 passes as the tensor core issues them: K = 32 (16 channel pairs) per instruction, 8 per tap
        chunks = []
        for g in range(0, 128, 16):
            sl = slice(g, g + 16)
            chunks.append(c(lo8[..., sl].to(D), c1_w[:, sl].to(D)) + c(hi8[..., sl].to(D), c2_w[:, sl].to(D)))
        if variant == "recipe":              # corrections first (their small sums lose nothing), then the fp16 main pass
            acc = sum(chunks) + main
        elif variant == "corr after main, 14-bit acc":
            acc = trunc_sig(main.float())
            for ch in chunks:
                acc = trunc_sig(acc + ch)
        else:
            raise ValueError(variant)
    pre = (acc * 2.0 ** -S).float() + torch.as_tensor(b).float()
    return store(torch.where(pre > 0, pre, pre * np.float32(0.1)), out_fp8)


def conv_fp32_emulate(y, W, b, out_fp8=False):
    """conv_ref_kernel (conv_impl = 1): per output, fmaf over taps j = 0..5 and input channels 0..127 in that order, from the
    activations as fp32 (hi16 + lo16 / 32), then bias, LeakyReLU and the hi16 + lo16 split."""
    x = y.float()
    W = torch.as_tensor(W).float()
    B, L, _ = x.shape
    xp = torch.cat([torch.zeros(B, 5, 128), x], dim=1)
    acc = torch.zeros(B, L, 128, dtype=torch.float32)
    for j in range(6):
        for ci in range(128):                 # fp64 product of two fp32 values is exact: one rounding per FMA
            acc = (acc.to(D) + xp[:, j:j + L, ci:ci + 1].to(D) * W[j, ci].to(D)).float()
    pre = acc + torch.as_tensor(b).float()
    return store(torch.where(pre > 0, pre, pre * np.float32(0.1)), out_fp8)


# ------------------------------------------------------------------------------------------ w_v: fp16 x 3
def wv_emulate(y, Wv, variant="recipe", rule="fixed"):
    """rule "fixed": the fp16 split of w_v * 2^e with max |w_v| * 2^e in [2^13, 2^14) (gnm_create); "old": of w_v itself."""
    Wv = torch.as_tensor(Wv).reshape(128, 128).float()
    e = 0
    if rule == "fixed":
        e = max(-24, min(40, 14 - math.frexp(float(Wv.abs().max()))[1]))
    Wv = Wv * 2.0 ** e
    Y = (32.0 * y).float()
    yh = f16(Y); yl = f16(Y - yh)
    wh = f16(Wv); wl = f16(Wv - wh)
    yh, yl, wh, wl = (t.to(D) for t in (yh, yl, wh, wl))
    z = yh @ wh
    if variant in ("recipe", "no Ahi*Wlo"):
        z = z + yl @ wh
    if variant in ("recipe", "no Alo*Whi"):
        z = z + yh @ wl
    return R._pool(z * 2.0 ** -e / 32.0)


# ------------------------------------------------------------------------------------------ patch gather: fp16 hi/lo x hi/lo
def gather_emulate(y, w, s, variant="recipe"):
    P = torch.as_tensor(np.asarray(w[f"ig{s}_random_patches"]).reshape(-1, 4), dtype=torch.long)
    ent = (torch.as_tensor(w[f"ig{s}_w_mult"])[0].float() * torch.as_tensor(w[f"ig{s}_w_summer"]).float().reshape(1, 4, 128))
    ent = ent * np.float32(1 / 32)
    wmax = float(ent.abs().max())
    k2 = max(-24, min(40, 14 - math.frexp(wmax)[1]))
    x = ent * 2.0 ** k2
    wh = f16(x); wl = f16(x - wh)
    Y = (32.0 * y).float()
    yh = f16(Y); yl = f16(Y - yh)
    A = yh + (0 if variant in ("single pass", "no Alo") else yl)
    Bw = wh + (0 if variant in ("single pass", "no Wlo") else wl)
    out = []
    for i in range(A.shape[0]):
        out.append((A[i][P].to(D) * Bw.to(D)).sum(dim=(1, 2)))
    return torch.stack(out) * 2.0 ** -k2 + torch.as_tensor(w[f"ig{s}_w_bias"]).to(D).reshape(-1)


# ------------------------------------------------------------------------------------------ logits / dense: 3 x TF32
def tf32x3_emulate(a, B, variant="recipe", split=None):
    """split: K products per split-K partial (logits 352, dense0 32, dense1 64), only used by the accumulator model."""
    a, B = torch.as_tensor(a).float(), torch.as_tensor(B).float()
    if variant == "single pass RN":
        return tf32_rn(a).to(D) @ tf32_rn(B).to(D)
    ah = tf32_trunc(a); al = tf32_trunc(a - ah)
    bh = tf32_trunc(B); bl = tf32_trunc(B - bh)
    ah, al, bh, bl = (t.to(D) for t in (ah, al, bh, bl))
    if variant == "recipe, truncating accumulator":
        # a model, not a measurement of the hardware: each partial runs through an fp32 accumulator that rounds toward zero
        # after every K = 8 step of each pass; the partials are added in fp32 (splitk_reduce_kernel)
        out = torch.zeros(a.shape[0], B.shape[1], dtype=torch.float32)
        K = a.shape[1]
        for k0 in range(0, K, split):
            acc = torch.zeros(a.shape[0], B.shape[1], dtype=D)
            for k in range(k0, min(K, k0 + split), 8):
                sl = slice(k, min(K, k + 8))
                for x, y in ((ah, bh), (al, bh), (ah, bl)):
                    acc = trunc_sig(acc + x[:, sl] @ y[sl], 24)
            out = out + acc.float()
        return out.to(D)
    z = ah @ bh
    if variant in ("recipe", "no Ahi*Blo"):
        z = z + al @ bh
    if variant in ("recipe", "no Alo*Bhi"):
        z = z + ah @ bl
    return z


# ------------------------------------------------------------------------------------------ the test
@pytest.fixture(scope="module")
def data(weights_npz):
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tools"))
    import precision_study
    w = M.synthetic_igloo_weights(M.load_npz_weights(weights_npz))
    a = precision_study.make_windows(8, seed=0)[[2, 4, 6]]         # tandem repeat, Markov chain, N islands
    tok = T.tokenize_windows(a)
    _, it = M.forward(tok, w, torch.float32, return_intermediates=True)
    y1 = store(it["y1"], False)
    y2 = store(it["y2"], True)
    y3 = store(it["y3"], False)
    return w, y1, y2, y3, it


def _row(table, stage, case, bar, value, ok):
    table.append((stage, case, value, bar, value / bar, ok))


def test_recipes_pass_and_mutants_fail_their_bars(data):
    w, y1, y2, y3, it = data
    table, bad = [], []

    def check(stage, bar_key, ref, cases, recipe_names=("recipe",), report_only=()):
        bar = R.BARS[bar_key][0]
        for case, got in cases.items():
            v = R.metrics(got, ref)["rms"]
            good = case in recipe_names
            if case in report_only:
                _row(table, stage, case + "  [reported only]", bar, v, True)
                continue
            ok = v * MARGIN <= bar if good else v >= MARGIN * bar
            _row(table, stage, case + ("" if good else "  [mutant]"), bar, v, ok)
            if not ok:
                bad.append((stage, case, v, bar))

    # conv2 on y1 and conv3 on y2 (shipped conv weights), and conv2 with the weights scaled down
    for stage, yin, kw, kb, fp8 in (("conv2", y1, "c2w", "c2b", True), ("conv3", y2, "c3w", "c3b", False)):
        ref = R.conv(yin, w[kw], w[kb])
        variants = ("recipe", "no Alo*Whi", "no Ahi*Wlo", "single pass", "corr after main, 14-bit acc")
        check(stage, "conv_tc", ref, {v: conv_emulate(yin, w[kw], w[kb], "fixed", v, fp8) for v in variants})
    # conv3 with weights and bias scaled by 2^k (y3 scales with them; its hi16 + lo16 planes keep full precision down to tiny
    # values, so the output shows the contraction's error): the old rule (d <= 16, hi = fp16(W)) loses the Ahi * Wlo correction
    for k in (-2, -4, -6, -8):
        W, b = (w["c3w"] * 2.0 ** k).astype(np.float32), (w["c3b"] * 2.0 ** k).astype(np.float32)
        ref = R.conv(y2, W, b)
        cases = {"recipe": conv_emulate(y2, W, b, "fixed", out_fp8=False), "old scaling rule": conv_emulate(y2, W, b, "old", out_fp8=False)}
        # above 2^-8 the old rule's loss is still inside the bar: a point of comparison, not a mutant
        check(f"conv3 x 2^{k}", "conv_tc", ref, cases, report_only=("old scaling rule",) if k > -8 else ())
    # the fp32 validation conv (conv_impl = 1) on the first 1024 positions; mutant: it reads only the hi16 plane
    yc = y2[:, :1024]
    ref = R.conv(yc, w["c3w"], w["c3b"])
    check("conv3 fp32 validation", "conv_fp32", ref,
          {"recipe": conv_fp32_emulate(yc, w["c3w"], w["c3b"]),
           "input hi16 only": conv_fp32_emulate(f16(32.0 * yc).to(D) / 32.0, w["c3w"], w["c3b"]),
           "tensor-core recipe": conv_emulate(yc, w["c3w"], w["c3b"], out_fp8=False)},
          report_only=("tensor-core recipe",))
    # w_v (IGLOO#0 on y1, IGLOO#1 on y3), shipped and scaled by 2^k: the old packing (no scaling) loses the Ahi * Wlo correction
    for s, yin in ((0, y1), (1, y3)):
        for k in (0, -4, -6, -8):
            Wv = (w[f"ig{s}_w_v"] * 2.0 ** k).astype(np.float32)
            ref = R.wv_pool(yin, Wv)
            variants = ("recipe", "no Alo*Whi", "no Ahi*Wlo", "single pass") if k == 0 else ("recipe",)
            cases = {v: wv_emulate(yin, Wv, v) for v in variants}
            cases["old packing (scale 1)"] = wv_emulate(yin, Wv, "recipe", "old")
            # above 2^-6 the old packing's loss is still inside the bar: a point of comparison, not a mutant
            check(f"w_v#{s} x 2^{k}", "wv", ref, cases, report_only=("old packing (scale 1)",) if k > -6 else ())
    # patch gather
    for s, yin in ((0, y1), (1, y3)):
        ref = R.gather(yin, w, s)
        check(f"gather#{s}", "gather", ref, {v: gather_emulate(yin, w, s, v) for v in ("recipe", "no Alo", "no Wlo", "single pass")})
    # logits (mpi @ w_qk) and the two dense layers (pre-activation: the tensor-core part of the stage)
    mpi = it["ig1"]["mpi"]
    tf_variants = ("recipe", "no Alo*Bhi", "no Ahi*Blo", "single pass", "single pass RN")
    tf_recipes = ("recipe", "recipe, truncating accumulator")
    h0 = it["h0"]
    h1 = torch.relu(R.dense_bn_relu(h0, w, 0).value)
    for name, hin, Wd, split in (("logits", mpi, w["ig1_w_qk"], 352), ("dense0", h0, w["d0w"], 32), ("dense1", h1, w["d1w"], 64)):
        cases = {v: tf32x3_emulate(hin, Wd, v) for v in tf_variants}
        cases["recipe, truncating accumulator"] = tf32x3_emulate(hin, Wd, "recipe, truncating accumulator", split)
        check(name, "tf32x3", R.matmul(hin, Wd), cases, recipe_names=tf_recipes)

    print("\n| stage | case | rms err / rms scale | bar | err / bar | ok |\n|---|---|---|---|---|---|")
    for stage, case, v, bar, r, ok in table:
        print(f"| {stage} | {case} | {v:.2e} | {bar:.0e} | {r:.2f} | {'yes' if ok else 'NO'} |")
    assert not bad, bad


def test_max_bars_hold_for_the_recipes(data):
    """The per-output bars (|err| / sum |terms|) hold with 2x margin for each recipe, in every region the GPU tests look at."""
    w, y1, y2, y3, it = data
    regions = R.position_regions(y1.shape[0])
    cases = [("conv_tc", conv_emulate(y1, w["c2w"], w["c2b"]), R.conv(y1, w["c2w"], w["c2b"])),
             ("conv_tc", conv_emulate(y2, w["c3w"], w["c3b"], out_fp8=False), R.conv(y2, w["c3w"], w["c3b"])),
             ("conv_tc", conv_emulate(y2, w["c3w"] / 256, w["c3b"] / 256, out_fp8=False), R.conv(y2, w["c3w"] / 256, w["c3b"] / 256)),
             ("wv", wv_emulate(y1, w["ig0_w_v"]), R.wv_pool(y1, w["ig0_w_v"])),
             ("wv", wv_emulate(y3, w["ig1_w_v"]), R.wv_pool(y3, w["ig1_w_v"])),
             ("gather", gather_emulate(y3, w, 1), R.gather(y3, w, 1)),
             ("tf32x3", tf32x3_emulate(it["ig1"]["mpi"], w["ig1_w_qk"]), R.matmul(it["ig1"]["mpi"], w["ig1_w_qk"]))]
    for key, got, ref in cases:
        m = R.metrics(got, ref, regions if got.dim() == 3 and got.shape[1] == R.L_TOK else None)
        worst = max(v for k, v in m.items() if k.startswith("max"))
        print(f"{key}: max {worst:.2e} (bar {R.BARS[key][1]:.0e})")
        assert worst * MARGIN <= R.BARS[key][1], (key, m)
