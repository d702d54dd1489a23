#!/usr/bin/env python
"""
Golden vectors of the reference's ENCODER sub-model: create_classifier() -> load_weights(nn_classifier.h5) on tests/golden/keras_shim.py
(helpers of make_reference_graph_golden.py), then the classifier's `model` layer -- create_encoder(), IGLOO block + Dense(512) +
BatchNorm + ReLU (genomad/neural_network/model.py:14-31) -- is asked for `predict` directly.

    python tests/golden/make_reference_encoder_golden.py     # needs /root/reference; a few minutes -> reference_encoder_golden.npz

Inputs: the 24 token windows of reference_graph_golden.npz ("graph_*") and the 16 of reference_tokens_golden.npz ("tokens_*").
Stored per input set: encoder outputs [n, 512] in fp32 and fp64 arithmetic, with the shipped weights and with synthetic O(1) IGLOO
weights (oracle.igloo_model.synthetic_igloo_weights assigned to the reference layers' variables).  The run ends with the
distance of tests/encoder_ref.py, the CPU restatement the tests use, to the stored fp64 outputs.
"""
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
import make_reference_graph_golden as G  # noqa: E402


def main():
    import torch
    import encoder_ref as E
    from oracle import igloo_model as M
    np.random.seed(0)                                          # the reference draws random patches at build time (then overwritten)
    model_mod, igloo_mod = G.load_reference_model_module()
    clf = model_mod.create_classifier()
    clf.load_weights(G.REF / "data" / "nn_classifier.h5")
    enc, _ = G.igloo_layers(clf, igloo_mod)
    assert enc.name == "model", enc.name
    inputs = {"graph": np.load(HERE / "reference_graph_golden.npz")["tokens"],
              "tokens": np.load(HERE / "reference_tokens_golden.npz")["tokens"]}
    w = M.load_npz_weights(G.ROOT / "genomad_b200" / "data" / "nn_classifier.npz")
    wsyn = M.synthetic_igloo_weights(w)
    out = {}

    def run(variant):
        for name, tok in inputs.items():
            t64 = tok.astype(np.int64)
            G.keras_shim.set_float(np.float32)
            out[f"{name}_{variant}"] = enc.predict(t64, batch_size=8).astype(np.float32)
            G.keras_shim.set_float(np.float64)
            out[f"{name}_{variant}_fp64"] = enc.predict(t64, batch_size=8).astype(np.float64)
            G.keras_shim.set_float(np.float32)

    run("shipped")
    G.set_synthetic(clf, igloo_mod, wsyn)
    run("synthetic")
    dst = HERE / "reference_encoder_golden.npz"
    np.savez_compressed(dst, graph_tokens=inputs["graph"], tokens_tokens=inputs["tokens"], **out)
    for name, tok in inputs.items():
        for variant, ww in (("shipped", w), ("synthetic", wsyn)):
            o64 = E.encoder(tok, ww, torch.float64)
            o32 = E.encoder(tok, ww, torch.float32)
            ref = out[f"{name}_{variant}_fp64"]
            print("%s/%s: encoder_ref fp64 vs reference fp64 %.3e, encoder_ref fp32 vs reference fp64 %.3e, max |e| %.3f" %
                  (name, variant, np.abs(o64 - ref).max(), np.abs(o32 - ref).max(), np.abs(ref).max()))
    print("wrote", dst)


if __name__ == "__main__":
    main()
