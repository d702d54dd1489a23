"""
End to end on an H100: nn-classification --head and train-head.
  * the shipped head through --head gives bitwise the main predictions;
  * a head trained on three synthetic composition classes classifies held-out sequences of the same generators;
  * two train-head runs write byte-identical head files.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CLASSES = ("gc35", "gc65", "motif")


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch


def _contig(rng, kind):
    n = int(rng.integers(20_000, 60_001))
    gc = {"gc35": 0.35, "gc65": 0.65, "motif": 0.5}[kind]
    p = np.array([(1 - gc) / 2, gc / 2, gc / 2, (1 - gc) / 2])
    s = np.frombuffer(b"ACGT", np.uint8)[rng.choice(4, n, p=p)].copy()
    if kind == "motif":                               # a planted periodic motif every 50 bases
        motif = np.frombuffer(b"TTAGGGTTAGGG", np.uint8)
        for a in range(0, n - len(motif), 50):
            s[a: a + len(motif)] = motif
    return s.tobytes().decode()


def write_set(path, seed, per_class):
    """FASTA of per_class contigs of each class (interleaved) and its labels TSV; returns the labels {name: class}."""
    rng = np.random.default_rng(seed)
    labels = {}
    with open(path, "w") as f:
        for i in range(per_class):
            for kind in CLASSES:
                name = f"s{seed}_{kind}_{i}"
                labels[name] = kind
                f.write(f">{name}\n{_contig(rng, kind)}\n")
    with open(str(path) + ".labels.tsv", "w") as f:
        f.write("seq_name\tclass\n")
        f.writelines(f"{k}\t{v}\n" for k, v in labels.items())
    return labels


def test_shipped_head_through_nn_classification_is_bitwise(torch, tmp_path):
    from genomad_b200 import nn_classification as nnc, weights as W
    w = W.load_weights()
    h = W.shipped_head(w)
    hp = tmp_path / "shipped_head.npz"
    W.save_head(hp, h.arrays, h.class_names, w)
    fa = tmp_path / "in.fna"
    write_set(fa, 5, 4)
    nnc.main(fa, tmp_path / "out", False, 128, False, 2, False, False, head=hp)
    d = tmp_path / "out" / "in_nn_classification"
    main = np.load(d / "in_nn_classification.npz")["predictions"]
    z = np.load(d / "in_nn_classification_head.npz")
    assert list(z["class_names"]) == ["chromosome", "plasmid", "virus"]
    assert np.array_equal(z["predictions"].view(np.uint32), main.view(np.uint32))


def _print_margins(head_arrays, X, labels):
    """How confidently the written head classifies its training windows: the log-odds margin of the labelled class,
    mu = l_y - max_{c != y} l_c, from fp64 inference-mode logits.  Past mu ~ 9 a float32 p_y - 1 keeps only a few bits."""
    f = {k: np.asarray(v, np.float64) for k, v in head_arrays.items()}
    z = X.astype(np.float64) @ f["d1w"] + f["d1b"]
    h = np.maximum((z - f["bn1m"]) / np.sqrt(f["bn1v"] + 1e-3) * f["bn1g"] + f["bn1b"], 0)
    lg = h @ f["d2w"] + f["d2b"]
    r = np.arange(len(lg))
    mu = lg[r, labels] - np.where(np.arange(lg.shape[1])[None, :] == labels[:, None], -np.inf, lg).max(1)
    edges = [-np.inf, 0, 9, 12, 17, 40, np.inf]
    counts = np.histogram(mu, edges)[0]
    print(f"training-window margins under the written head ({len(mu)} windows): median {np.median(mu):.1f}, "
          f"p10 {np.quantile(mu, 0.1):.1f}, p90 {np.quantile(mu, 0.9):.1f}, max {mu.max():.1f}; "
          + ", ".join(f"[{lo:g}, {hi:g}): {n}" for lo, hi, n in zip(edges[:-1], edges[1:], counts)))


def test_train_head_learns_composition_classes(torch, tmp_path, monkeypatch):
    from genomad_b200 import nn_classification as nnc, train_head, weights as W
    train_fa, test_fa = tmp_path / "train.fna", tmp_path / "test.fna"
    write_set(train_fa, 1, 60)
    truth = write_set(test_fa, 2, 20)
    seen = {}
    make = train_head._make_trainer

    def spy(*args, **kwargs):            # records the training matrix, labels and batch rows of the first run
        tr = make(*args, **kwargs)
        step = tr.step

        def recorded(X, idx, labels, cw, loss=None):
            seen.setdefault("X", X)
            seen.setdefault("labels", labels)
            seen.setdefault("idx", []).append(idx.clone())
            return step(X, idx, labels, cw, loss=loss)
        tr.step = recorded
        return tr
    runs = []
    for k in range(2):
        out = tmp_path / f"head{k}"
        with monkeypatch.context() as m:
            if k == 0:
                m.setattr(train_head, "_make_trainer", spy)
            train_head.main(train_fa, str(train_fa) + ".labels.tsv", out, epochs=10, batch_size=256, seed=3, verbose=False)
        runs.append((out / "train_head.npz").read_bytes())
    assert runs[0] == runs[1], "two train-head runs wrote different head files"
    tsv = (tmp_path / "head0" / "train_head_training.tsv").read_text().splitlines()
    print("\n".join(tsv))
    rows = torch.unique(torch.cat(seen["idx"])).cpu().numpy()
    best = W.load_head(tmp_path / "head0" / "train_head.npz", W.load_weights())
    _print_margins(best.arrays, seen["X"].cpu().numpy()[rows], seen["labels"].cpu().numpy()[rows])
    nnc.main(test_fa, tmp_path / "scored", False, 128, False, 2, False, False, head=tmp_path / "head0" / "train_head.npz")
    z = np.load(tmp_path / "scored" / "test_nn_classification" / "test_nn_classification_head.npz")
    names, preds, cls = z["contig_names"], z["predictions"], list(z["class_names"])
    acc = float(np.mean([cls[int(np.argmax(p))] == truth[str(n)] for n, p in zip(names, preds)]))
    print(f"held-out sequence accuracy: {acc:.4f} over {len(names)} sequences")
    assert acc >= 0.95
