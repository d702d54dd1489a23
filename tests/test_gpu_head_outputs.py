"""
End to end on an H100: the head's strand and window files, the Head API for contigs in memory, and train-head --both-strands.
  * the shipped head (the classifier's own tail) gives bitwise the strand file's and the window file's scores, and the same
    TSV bytes, at stride 6000, at stride 1000 and with --single-window;
  * with a seeded C = 7 head, Head.window_scores is Head.predict of the windows' embeddings, Head.classify_contigs on the
    reverse strand is the forward call on the reverse-complemented contigs, and the module's files are these API results;
  * train-head --both-strands is reproducible, embeds the reverse windows as Classifier.embed_windows(..., reverse=True) does,
    and trains a head that classifies held-out sequences and their reverse complements.
"""
import numpy as np
import pytest

from genomad_b200 import _paths, engine, nn_classification as nnc, sequence, train_head, weights as W
from test_gpu_head_module import write_set
from test_gpu_strands import _module_input, _rc_file

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _shipped_head_file(path):
    w = W.load_weights()
    h = W.shipped_head(w)
    W.save_head(path, h.arrays, h.class_names, w)
    return path


# ------------------------------------------------------------------------------------------ the shipped head as the oracle
@pytest.mark.parametrize("stride,single_window", [(6000, False), (1000, False), (6000, True)])
def test_shipped_head_files_are_the_shipped_files(torch, tmp_path, stride, single_window):
    hp = _shipped_head_file(tmp_path / "shipped_head.npz")
    fa = _module_input(tmp_path / "sample.fna")
    nnc.main(fa, tmp_path / "out", single_window, 128, False, 4, False, False, head=hp, both_strands=True,
             write_window_scores=True, window_stride=stride)
    o = _paths.NNOutputs("sample", tmp_path / "out")
    zs, zh = np.load(o.nn_classification_strands_npz_output), np.load(o.nn_classification_head_strands_npz_output)
    for k in nnc.STRANDS:
        assert np.array_equal(_bits(zh[k]), _bits(zs[k])), k
    assert o.nn_classification_head_strands_output.read_bytes() == o.nn_classification_strands_output.read_bytes()
    zw, zhw = np.load(o.nn_classification_windows_npz_output), np.load(o.nn_classification_head_windows_npz_output)
    assert int(zhw["window_stride"]) == stride and len(zw["predictions"]) > 0
    assert np.array_equal(_bits(zhw["predictions"]), _bits(zw["predictions"]))
    assert o.nn_classification_head_windows_output.read_bytes() == o.nn_classification_windows_output.read_bytes()


# ------------------------------------------------------------------------------------------ a seeded C = 7 head
@pytest.fixture(scope="module")
def head7(torch, tmp_path_factory):
    d = tmp_path_factory.mktemp("head7")
    w = W.load_weights()
    hp = d / "h7.npz"
    W.save_head(hp, W.initial_head(7, 11), tuple(f"k{i}" for i in range(7)), w)
    clf = nnc._make_classifier(128, 0)
    h = engine.Head(clf, W.load_head(hp, w))
    yield clf, h, hp
    h.close()


def _raw_records(fa):
    return [s for _, s in sequence.iter_fasta(fa, strip_n=False)]


@pytest.mark.parametrize("stride", [6000, 1000, 2501])
def test_window_scores_are_predict_of_the_embeddings(torch, tmp_path, head7, stride):
    clf, h, _ = head7
    seqs = _raw_records(_module_input(tmp_path / "s.fna"))
    ws = h.window_scores(seqs, stride)
    ref = clf.window_scores(seqs, stride)
    assert ws.probs.shape == (ref.probs.shape[0], 7) and ref.probs.shape[0] > 0
    for a, b in zip(ws[1:], ref[1:]):
        assert torch.equal(a, b)
    seq, offs = clf.contig_buffers(seqs)
    start, length, _ = clf.contig_windows(seq, offs, stride=stride)
    assert torch.equal(ws.probs, h.predict(clf.embed_windows(seq, start, length)[1]))


def test_classify_contigs_reverse_is_forward_of_rc(torch, tmp_path, head7):
    clf, h, _ = head7
    seqs = _raw_records(_module_input(tmp_path / "s.fna"))
    rc = [sequence.reverse_complement(s) for s in seqs]
    for single in (False, True):
        m_r, c_r = h.classify_contigs(seqs, single, strand="reverse")
        m_f, c_f = h.classify_contigs(rc, single)
        assert m_r.shape == (len(seqs), 7) and torch.equal(m_r, m_f) and torch.equal(c_r, c_f)
        m_a, c_a = h.classify_contigs(seqs, single)
        assert torch.equal(c_a, clf.classify_contigs(seqs, single)[1])
        assert torch.equal(engine.both_strands(m_a, m_r), engine.both_strands(m_f, h.classify_contigs(rc, single,
                                                                                                      strand="reverse")[0]))
    with pytest.raises(ValueError):
        h.classify_contigs(seqs[:2], strand="both")
    empty = h.classify_contigs([b"NNNN", b""])
    assert empty[0].shape == (2, 7) and not empty[0].any() and not empty[1].any()


@pytest.mark.parametrize("stride", [6000, 1000])
def test_module_files_are_the_api(torch, tmp_path, head7, stride):
    clf, h, hp = head7
    fa = _module_input(tmp_path / "sample.fna")
    seqs = _raw_records(fa)
    nnc.main(fa, tmp_path / "out", False, 128, False, 4, False, False, head=hp, both_strands=True,
             write_window_scores=True, window_stride=stride)
    o = _paths.NNOutputs("sample", tmp_path / "out")
    z = np.load(o.nn_classification_head_strands_npz_output)
    fwd, rev = h.classify_contigs(seqs)[0].cpu().numpy(), h.classify_contigs(seqs, strand="reverse")[0].cpu().numpy()
    assert len(z["contig_names"]) == len(seqs)
    assert np.array_equal(_bits(z["forward"]), _bits(fwd)) and np.array_equal(_bits(z["reverse"]), _bits(rev))
    assert np.array_equal(_bits(z["both_strands"]), _bits(engine.both_strands(fwd, rev)))
    zw = np.load(o.nn_classification_head_windows_npz_output)
    ws = h.window_scores(seqs, stride)
    assert np.array_equal(_bits(zw["predictions"]), _bits(ws.probs.cpu().numpy()))
    assert np.array_equal(zw["window_start"], ws.start.cpu().numpy())
    assert np.array_equal(zw["window_length"], ws.length.cpu().numpy())


# ------------------------------------------------------------------------------------------ train-head --both-strands
def _accuracy(tmp_path, head_path, fa, truth, tag):
    nnc.main(fa, tmp_path / tag, False, 128, False, 4, False, False, head=head_path, both_strands=True)
    o = _paths.NNOutputs(fa.name.rsplit(".", 1)[0], tmp_path / tag)
    z = np.load(o.nn_classification_head_strands_npz_output)
    cls = list(z["class_names"])
    return {k: float(np.mean([cls[int(np.argmax(p))] == truth[str(n)] for n, p in zip(z["contig_names"], z[k])]))
            for k in nnc.STRANDS}


def test_train_head_both_strands(torch, tmp_path, monkeypatch):
    train_fa, test_fa = tmp_path / "train.fna", tmp_path / "test.fna"
    write_set(train_fa, 1, 60)
    truth = write_set(test_fa, 2, 20)
    (tmp_path / "rc").mkdir()
    test_rc = _rc_file(test_fa, tmp_path / "rc" / "test.fna")
    seen = {}
    make = train_head._make_trainer

    def spy(*args, **kwargs):
        tr = make(*args, **kwargs)
        step = tr.step

        def recorded(X, idx, labels, cw, loss=None):
            seen.setdefault("X", X)
            return step(X, idx, labels, cw, loss=loss)
        tr.step = recorded
        return tr
    runs = []
    for k in range(2):
        with monkeypatch.context() as m:
            if k == 0:
                m.setattr(train_head, "_make_trainer", spy)
            train_head.main(train_fa, str(train_fa) + ".labels.tsv", tmp_path / f"both{k}", epochs=10, batch_size=256,
                            seed=3, verbose=False, both_strands=True)
        runs.append((tmp_path / f"both{k}" / "train_head.npz").read_bytes())
    assert runs[0] == runs[1], "two train-head --both-strands runs wrote different head files"
    print("\n".join((tmp_path / "both0" / "train_head_training.tsv").read_text().splitlines()))
    # rows [N_f, N_f + N_r) of X: Classifier.embed_windows(..., reverse=True) of the records' reverse windows, in file order
    clf = nnc._make_classifier(128, 0)
    seq, offs = clf.contig_buffers(_raw_records(train_fa))
    fs, fl, _ = clf.contig_windows(seq, offs)
    rs, rl, _ = clf.contig_windows(seq, offs, reverse=True)
    X = seen["X"]
    Nf, Nr = fs.numel(), rs.numel()
    assert X.shape == (Nf + Nr, 512)
    assert torch.equal(X[:Nf], clf.embed_windows(seq, fs, fl)[1])
    assert torch.equal(X[Nf:], clf.embed_windows(seq, rs, rl, reverse=True)[1])
    hb = tmp_path / "both0" / "train_head.npz"
    acc_f, acc_r = _accuracy(tmp_path, hb, test_fa, truth, "scored_f"), _accuracy(tmp_path, hb, test_rc, truth, "scored_r")
    print(f"--both-strands head, both_strands scores: held-out {acc_f['both_strands']:.4f}, "
          f"reverse-complemented {acc_r['both_strands']:.4f} (forward-strand scores {acc_f['forward']:.4f} / "
          f"{acc_r['forward']:.4f})")
    train_head.main(train_fa, str(train_fa) + ".labels.tsv", tmp_path / "fwd", epochs=10, batch_size=256, seed=3,
                    verbose=False)
    acc_o = _accuracy(tmp_path, tmp_path / "fwd" / "train_head.npz", test_rc, truth, "scored_o")
    print(f"forward-only head on the reverse-complemented set: forward scores {acc_o['forward']:.4f}, both_strands "
          f"{acc_o['both_strands']:.4f}")
    assert acc_f["both_strands"] >= 0.95 and acc_r["both_strands"] >= 0.95
