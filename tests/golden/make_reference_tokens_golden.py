#!/usr/bin/env python
"""
Golden vectors for the from-tokens entry point (gnm_forward_tokens, Classifier.predict_tokens) on token windows that are NOT a
tokenization: the reference's own model definition, genomad/neural_network/{model,igloo}.py, imported by path and executed on
tests/golden/keras_shim.py exactly as make_reference_graph_golden.py does.  Its first op, tf.one_hot(x, depth=257), accepts any
integer and gives an all-zero row to a value outside [0, 257); the stand-in's one_hot does the same.

    python tests/golden/make_reference_tokens_golden.py     # needs the reference checkout; seconds -> reference_tokens_golden.npz

The 16 windows (`kinds` names them):
  uniform random tokens in [0, 256] (and in [1, 256]); tokenizations with every odd position replaced by a random token (the
  outer tokens of each layer-1 half stay a consistent pair, the middle one does not); all 0; all 256; tokenizations that are
  inconsistent only at positions 0-5, 250-262 (the 256-position segment seam of embed_conv1_kernel) and 5990-5996; sparse
  random substitutions; an untouched tokenization; and windows carrying out-of-range values 257, 4096, 32767, 32768, 65535
  (sprinkled, at the seams, all 65535, alternating 256 / 257).
Stored: tokens (uint16), in_range (all tokens <= 256), the reference graph's probabilities in fp32 and fp64 with the shipped
weights and with synthetic O(1) IGLOO weights, and the reference graph's layer-1 activations (after the first LeakyReLU, fp64,
shipped weights) at the positions `l1_pos`, every 4th channel.
"""
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ROOT = HERE.parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
sys.path.insert(0, str(HERE))
import keras_shim  # noqa: E402
from make_reference_graph_golden import REF, igloo_layers, load_reference_model_module, set_synthetic  # noqa: E402

OUT_OF_RANGE = np.array([257, 4096, 32767, 32768, 65535])
SEAMS = np.r_[0:6, 250:263, 5990:5997]
L1_POS = np.unique(np.r_[0:8, 248:266, 5986:5997, 0:5997:97])


def token_windows():
    """[16, 5997] int64 token windows and their names."""
    from oracle import tokenizer as T
    import precision_study
    rng = np.random.default_rng(2026)
    base = T.tokenize_windows(precision_study.make_windows(16, seed=77)).astype(np.int64)   # base[1] is all N: all 0
    L = base.shape[1]
    odd = np.arange(1, L, 2)
    wins, kinds = [], []

    def add(kind, t):
        wins.append(np.asarray(t, np.int64)); kinds.append(kind)

    add("uniform [0, 256]", rng.integers(0, 257, L))
    add("uniform [0, 256]", rng.integers(0, 257, L))
    for b in (2, 4):
        t = base[b].copy(); t[odd] = rng.integers(0, 257, odd.size); add("tokenization, odd positions random", t)
    add("all 0", np.zeros(L))
    add("all 256", np.full(L, 256))
    for b in (0, 7):
        t = base[b].copy(); t[SEAMS] = rng.integers(1, 257, SEAMS.size); add("tokenization, seams random", t)
    t = base[5].copy()
    pos = rng.choice(L, 300, replace=False); t[pos] = OUT_OF_RANGE[np.arange(300) % 5]; t[[0, 255, 256, 5996]] = [65535, 257, 32768, 4096]
    add("tokenization, sprinkled > 256", t)
    t = rng.integers(0, 257, L)
    pos = rng.choice(L, 600, replace=False); t[pos] = OUT_OF_RANGE[np.arange(600) % 5]
    add("uniform, sprinkled > 256", t)
    add("all 65535", np.full(L, 65535))
    t = base[6].copy(); t[SEAMS] = OUT_OF_RANGE[np.arange(SEAMS.size) % 5]; add("tokenization, seams > 256", t)
    add("alternating 256 / 257", np.where(np.arange(L) % 2 == 0, 256, 257))
    add("uniform [1, 256]", rng.integers(1, 257, L))
    t = base[8].copy(); pos = rng.choice(L, 180, replace=False); t[pos] = rng.integers(1, 257, 180)
    add("tokenization, 3% random", t)
    add("tokenization (N islands)", base[6])
    return np.stack(wins), np.array(kinds)


def main():
    import torch
    from oracle import igloo_model as M
    tok, kinds = token_windows()
    assert tok.shape == (16, 5997) and tok.min() >= 0 and tok.max() <= 65535
    np.random.seed(0)
    model_mod, igloo_mod = load_reference_model_module()
    clf = model_mod.create_classifier()
    clf.load_weights(REF / "data" / "nn_classifier.h5")
    out = {}
    for dt, suffix in ((np.float32, ""), (np.float64, "_fp64")):
        keras_shim.set_float(dt)
        out["shipped" + suffix] = clf.predict(tok, batch_size=8)
    # layer 1 of the reference graph (one-hot -> conv -> LeakyReLU), fp64, shipped weights
    enc, _ = igloo_layers(clf, igloo_mod)
    x = tok
    for lay in enc.layers[1:]:
        x = lay._run(x)
        if isinstance(lay, keras_shim.LeakyReLU):
            break
    out["l1_shipped_fp64"] = np.asarray(x)[:, L1_POS, ::4]
    w = M.load_npz_weights(ROOT / "genomad_b200" / "data" / "nn_classifier.npz")
    wsyn = M.synthetic_igloo_weights(w)
    set_synthetic(clf, igloo_mod, wsyn)
    for dt, suffix in ((np.float32, ""), (np.float64, "_fp64")):
        keras_shim.set_float(dt)
        out["synthetic" + suffix] = clf.predict(tok, batch_size=8)
    keras_shim.set_float(np.float32)
    path = HERE / "reference_tokens_golden.npz"
    np.savez_compressed(path, tokens=tok.astype(np.uint16), kinds=kinds, in_range=(tok <= 256).all(1), l1_pos=L1_POS, **out)
    for key, ww in (("shipped", w), ("synthetic", wsyn)):
        o64 = np.concatenate([M.forward(tok[i:i + 8], ww, torch.float64) for i in range(0, 16, 8)])
        print(f"reference graph vs oracle, fp64, {key}: max |dp| {np.abs(o64 - out[key + '_fp64']).max():.3e}")
    print("wrote", path)


if __name__ == "__main__":
    main()
