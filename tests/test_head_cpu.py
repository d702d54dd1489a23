"""
CPU checks of the classifier-head path: the fp64 statement in head_ref.py (backward against finite differences, inference of
the shipped head against the oracle), the dropout hash, the head file format, LABELS.tsv parsing, the split and the class
weights of train-head.
"""
import numpy as np
import pytest

import head_ref as R
from genomad_b200 import train_head as T, weights as W


@pytest.fixture(scope="module")
def w():
    return W.load_weights()


@pytest.mark.parametrize("C", [2, 3, 32])
@pytest.mark.parametrize("B", [1, 2, 257])
def test_backward_matches_finite_differences(C, B):
    rng = np.random.default_rng(C * 1000 + B)
    p = {k: v.astype(np.float64) for k, v in R.random_head(C, C).items() if k not in ("bn1m", "bn1v")}
    X = np.maximum(rng.normal(0, 1, (B, 512)), 0)
    labels = rng.integers(0, C, B)
    cw = rng.uniform(0.3, 3.0, C)
    mask = R.keep_mask(5, 3, B)
    _, cache = R.forward(p, X, labels, cw, mask)
    g = R.backward(cache)
    for k in p:
        flat = p[k].reshape(-1)
        for i in rng.choice(flat.size, min(flat.size, 6), replace=False):
            h = 1e-6
            old = flat[i]
            flat[i] = old + h
            lp, _ = R.forward(p, X, labels, cw, mask)
            flat[i] = old - h
            lm, _ = R.forward(p, X, labels, cw, mask)
            flat[i] = old
            fd = (lp - lm) / (2 * h)
            assert abs(fd - g[k].reshape(-1)[i]) <= 1e-6 * max(1.0, abs(fd)), (k, i, fd, g[k].reshape(-1)[i])


def test_shipped_head_inference_matches_the_oracle(w):
    """At C = 3 with shipped_head, head_ref.infer on the encoder output h1 is the oracle's head (which starts at dense_0)."""
    import torch
    from oracle import igloo_model as M
    rng = np.random.default_rng(0)
    h0 = torch.from_numpy(rng.normal(0, 1, (16, 256)))
    wt = M.load_npz_weights(W.DEFAULT_NPZ)
    ref = M.head(h0, wt, torch.float64).numpy()
    f = {k: np.asarray(wt[k], np.float64) for k in ("d0w", "d0b", "bn0g", "bn0b", "bn0m", "bn0v")}
    z = h0.numpy() @ f["d0w"] + f["d0b"]
    h1 = np.maximum(f["bn0g"] * (z - f["bn0m"]) / np.sqrt(f["bn0v"] + R.EPS_BN) + f["bn0b"], 0)
    assert np.abs(R.infer(W.shipped_head(w).arrays, h1) - ref).max() <= 1e-12


def test_mask_rate_and_determinism():
    m = R.keep_mask(0, 0, 2000)[:, :500]            # 10^6 draws
    assert abs(m.mean() - 0.8) <= 0.002
    assert np.array_equal(R.keep_mask(0, 0, 10), R.keep_mask(0, 0, 10))
    assert not np.array_equal(R.keep_mask(0, 1, 10), R.keep_mask(0, 0, 10))
    assert not np.array_equal(R.keep_mask(1, 0, 10), R.keep_mask(0, 0, 10))


def _save(tmp_path, w, arrays, names, **override):
    import zipfile
    p = tmp_path / "h.npz"
    W.save_head(p, arrays, names, w)
    if override:
        with np.load(p) as z:
            d = {k: z[k] for k in z.files}
        d.update(override)
        np.savez(p, **d)
    return p


def test_head_file_round_trip_and_bytes(tmp_path, w):
    h = W.shipped_head(w)
    p = _save(tmp_path, w, h.arrays, h.class_names)
    b = p.read_bytes()
    back = W.load_head(p, w)
    assert back.class_names == W.SHIPPED_CLASSES and back.encoder_sha256 == W.encoder_sha256(w)
    assert all(np.array_equal(back.arrays[k], h.arrays[k]) for k in W.HEAD_KEYS)
    W.save_head(p, h.arrays, h.class_names, w)
    assert p.read_bytes() == b


@pytest.mark.parametrize("case", ["shape", "dtype", "C1", "C33", "dup", "badname", "sha"])
def test_load_head_rejects(tmp_path, w, case):
    h = W.shipped_head(w)
    k2w, k2b = W.KEYS["d2w"][0], W.KEYS["d2b"][0]
    over = {"shape": {W.KEYS["d1w"][0]: np.zeros((512, 511), np.float32)},
            "dtype": {W.KEYS["d1b"][0]: np.zeros(512, np.float64)},
            "C1": {k2w: np.zeros((512, 1), np.float32), k2b: np.zeros(1, np.float32), "class_names": np.array(["a"])},
            "C33": {k2w: np.zeros((512, 33), np.float32), k2b: np.zeros(33, np.float32),
                    "class_names": np.array([f"c{i}" for i in range(33)])},
            "dup": {"class_names": np.array(["a", "b", "a"])},
            "badname": {"class_names": np.array(["a", "b c", "d"])},
            "sha": {"encoder_sha256": np.array("0" * 64)}}[case]
    p = _save(tmp_path, w, h.arrays, h.class_names, **over)
    key = {"shape": "dense_1", "dtype": "dense_1", "C1": "class_names", "C33": "class_names", "dup": "class_names",
           "badname": "class_names", "sha": "encoder_sha256"}[case]
    with pytest.raises(ValueError, match=key):
        W.load_head(p, w)


def test_encoder_hash_ignores_the_head(w):
    w2 = dict(w)
    w2["d2w"] = w["d2w"] * 2
    assert W.encoder_sha256(w2) == W.encoder_sha256(w)
    w2["c1b"] = w["c1b"] + 1
    assert W.encoder_sha256(w2) != W.encoder_sha256(w)


def test_initial_head_is_glorot_and_seeded():
    a, b = W.initial_head(7, 3), W.initial_head(7, 3)
    assert all(np.array_equal(a[k], b[k]) for k in a)
    assert np.abs(a["d1w"]).max() <= np.sqrt(6 / 1024) and np.abs(a["d2w"]).max() <= np.sqrt(6 / 519)
    assert abs(a["d1w"].std() - np.sqrt(6 / 1024) / np.sqrt(3)) < 1e-3
    assert not a["d1b"].any() and (a["bn1g"] == 1).all() and (a["bn1v"] == 1).all()


@pytest.mark.parametrize("text, msg", [
    ("name\tclass\nx\ta\n", "header"),
    ("seq_name\tclass\nx\n", "line 2"),
    ("seq_name\tclass\nx\ta\tb\n", "line 2"),
    ("seq_name\tclass\nx\t\n", "line 2"),
])
def test_labels_parse_errors(tmp_path, text, msg):
    p = tmp_path / "l.tsv"
    p.write_text(text)
    with pytest.raises(ValueError, match=msg):
        T.read_labels(p)


def test_labels_match_errors():
    names = np.array([f"s{i}" for i in range(20)])
    with pytest.raises(ValueError, match="more than once: s1"):
        T.label_records(names, ["s1", "s2", "s1"], ["a", "b", "a"], ("a", "b"))
    unknown = [f"u{i}" for i in range(12)]
    with pytest.raises(ValueError, match="12 labelled name.*u9 and 2 more"):
        T.label_records(names, unknown, ["a"] * 12, ("a",))
    lab = T.label_records(names, ["s3", "s0"], ["b", "a"], ("a", "b"))
    assert lab[0] == 0 and lab[3] == 1 and (np.delete(lab, [0, 3]) == -1).all()
    with pytest.raises(ValueError, match="1 classes"):
        T.class_names_of(["a", "a"])
    with pytest.raises(ValueError, match="does not match"):
        T.class_names_of(["a", "b/c"])


def test_split_and_balanced_weights_worked_example():
    # class 0: 10 sequences, class 1: 3, class 2: 1; fraction 0.2 -> hold out 2, 1 (at least one), 0 (keeps its only one)
    seq_class = np.array([0] * 10 + [1] * 3 + [2])
    val = T.split_sequences(seq_class, 3, 0.2, seed=0)
    assert [int(val[seq_class == c].sum()) for c in range(3)] == [2, 1, 0]
    assert np.array_equal(val, T.split_sequences(seq_class, 3, 0.2, seed=0))
    assert not T.split_sequences(seq_class, 3, 0.0, seed=0).any()
    # 6 training windows: 3 of class 0, 2 of class 1, 1 of class 2 -> N / (C N_c) = 6/9, 6/6, 6/3
    cw = T.class_weights(np.array([0, 0, 0, 1, 1, 2]), 3, "balanced")
    assert np.allclose(cw, [6 / 9, 1.0, 2.0])
    assert (T.class_weights(np.array([0, 1]), 2, "none") == 1).all()
