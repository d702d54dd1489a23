"""
CPU tests of `nn-classification --head` and `train-head` with stub classifiers (tests/window_stub.py, tests/head_stub.py) behind the
real module code: the head files' format and values, the main outputs bitwise those of a run without --head, the restart rule
(head files missing, another head, the same head), the refusal of a head trained on another encoder, and for train-head which
windows are embedded and get which label, the split by sequence, the output files and the refusals.
"""
import hashlib

import numpy as np
import pytest
import torch
from click.testing import CliRunner

import head_stub as HS
import window_stub as WS
from genomad_b200 import _paths, cli, nn_classification, sequence, train_head, weights as W
from test_strands_cpu import EmbedStub, stub_emb
from test_window_scores_cpu import _contig_outputs, _module_fasta, _run


@pytest.fixture
def stub(monkeypatch):
    clf = EmbedStub()
    WS.install(monkeypatch.setattr, nn_classification, clf)
    monkeypatch.setattr(nn_classification, "_make_head", HS.StubHead)
    for k in ("GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS", "GENOMAD_B200_ATTRIBUTIONS",
              "GENOMAD_B200_BOTH_STRANDS", "RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    return clf


def _expected_head(fa, C):
    """Per contig: the fp32 running mean of the stub head's probabilities of its windows' stub embeddings."""
    pf = sequence.ParsedFasta(fa)
    try:
        idx = pf.index()
        win = pf.export_windows(0, pf.n_windows, np.empty((pf.n_windows, 6000), np.uint8))
    finally:
        pf.close()
    return idx.names, WS.running_mean(HS.stub_head_probs(stub_emb(win), C), idx.offsets)


def test_head_files_format_and_values(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    hp = HS.write_head(tmp_path / "h.npz", 4, 1, names=("alpha", "beta", "gamma.1", "d-4"))
    o = _run(fa, tmp_path / "out", head=hp)
    names, want = _expected_head(fa, 4)
    z = np.load(o.nn_classification_head_npz_output)
    assert set(z.files) == {"contig_names", "predictions", "class_names", "head_sha256"}
    assert list(z["contig_names"]) == list(names) and list(z["class_names"]) == ["alpha", "beta", "gamma.1", "d-4"]
    assert z["predictions"].dtype == np.float32 and np.array_equal(z["predictions"], want)
    assert str(z["head_sha256"]) == hashlib.sha256(hp.read_bytes()).hexdigest()
    lines = o.nn_classification_head_output.read_text().split("\n")
    assert lines[0] == "seq_name\talpha_score\tbeta_score\tgamma.1_score\td-4_score" and lines[-1] == ""
    for line, n, p in zip(lines[1:-1], names, want):
        assert line == n + "".join(f"\t{float(x):.4f}" for x in p)


def test_main_outputs_unchanged_by_head(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    hp = HS.write_head(tmp_path / "h.npz", 3, 2)
    plain = _contig_outputs(_run(fa, tmp_path / "plain"))
    with_head = _contig_outputs(_run(fa, tmp_path / "head", head=hp))
    assert plain == with_head


def test_restart_rule(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    ha, hb = HS.write_head(tmp_path / "a.npz", 3, 1), HS.write_head(tmp_path / "b.npz", 5, 2)
    out = tmp_path / "out"
    o = _run(fa, out, head=ha)
    n0 = len(stub.windows_seen())
    assert n0 > 0
    _run(fa, out, head=ha)                                         # same head: nothing is classified again
    assert len(stub.windows_seen()) == n0
    o.nn_classification_head_output.unlink()                       # a head file missing: classified again
    _run(fa, out, head=ha)
    assert len(stub.windows_seen()) == 2 * n0 and o.nn_classification_head_output.exists()
    _run(fa, out, head=hb)                                         # another head: classified again, its files replace A's
    assert len(stub.windows_seen()) == 3 * n0
    z = np.load(o.nn_classification_head_npz_output)
    assert str(z["head_sha256"]) == hashlib.sha256(hb.read_bytes()).hexdigest() and z["predictions"].shape[1] == 5


def test_head_for_another_encoder_is_refused_before_any_work(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    other = dict(W.load_weights())
    other["c1b"] = other["c1b"] + np.float32(1)
    hp = HS.write_head(tmp_path / "h.npz", 3, 1, weights=other)
    with pytest.raises(SystemExit) as e:
        _run(fa, tmp_path / "out", head=hp)
    assert e.value.code == 1
    assert len(stub.windows_seen()) == 0
    assert not _paths.NNOutputs("sample", tmp_path / "out").nn_classification_npz_output.exists()


# ------------------------------------------------------------------------------------------------ train-head
def _train_set(path):
    """12 records: 3 classes x 3 labelled (windows 1..5), one labelled record without a window, two unlabelled ones."""
    rng = np.random.default_rng(3)
    recs, labels = [], {}
    for i in range(9):
        name = f"r{i}"
        recs.append((name, np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 6000 * (1 + i % 5))].tobytes()))
        labels[name] = ("red", "green", "blue")[i % 3]
        if i == 4:
            recs.append(("unlabelled_a", np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 13000)].tobytes()))
    recs.append(("all_n", b"N" * 500))                                 # stripped of n/N: no window
    labels["all_n"] = "red"
    recs.append(("unlabelled_b", np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 7000)].tobytes()))
    with open(path, "wb") as f:
        for n, s in recs:
            f.write(f">{n}\n".encode() + s + b"\n")
    lab = path.with_suffix(".tsv")
    lab.write_text("seq_name\tclass\n" + "".join(f"{k}\t{v}\n" for k, v in labels.items()))
    return path, lab, labels


@pytest.fixture
def trainer_stubs(monkeypatch, stub):
    made = []

    def make_trainer(*a):
        made.append(HS.StubTrainer(*a))
        return made[-1]
    monkeypatch.setattr(train_head, "_make_classifier", lambda device: stub)
    monkeypatch.setattr(train_head, "_free_bytes", lambda clf: 1 << 40)
    monkeypatch.setattr(train_head, "_make_trainer", make_trainer)
    monkeypatch.setattr(train_head, "_make_head", HS.StubHead)
    return made


def test_train_head_windows_labels_and_split(tmp_path, stub, trainer_stubs):
    fa, lab, labels = _train_set(tmp_path / "train.fna")
    train_head.main(fa, lab, tmp_path / "out", epochs=3, batch_size=4, validation_fraction=0.34, seed=5, verbose=False)
    tr = trainer_stubs[0]
    pf = sequence.ParsedFasta(fa)
    try:
        idx = pf.index()
        names = list(idx.names)
        used = [i for i, n in enumerate(names) if n in labels and idx.offsets[i + 1] > idx.offsets[i]]
        win = np.concatenate([pf.export_windows(int(idx.offsets[i]), int(idx.offsets[i + 1] - idx.offsets[i]),
                                                np.empty((int(idx.offsets[i + 1] - idx.offsets[i]), 6000), np.uint8))
                              for i in used])
    finally:
        pf.close()
    # only the labelled records' windows were embedded, in file order; X holds their embeddings
    assert np.array_equal(stub.windows_seen(), win)
    assert np.array_equal(tr.X.numpy(), stub_emb(win))
    classes = ("blue", "green", "red")
    row_seq = np.repeat(np.arange(len(used)), [int(idx.offsets[i + 1] - idx.offsets[i]) for i in used])
    row_class = np.array([classes.index(labels[names[used[s]]]) for s in row_seq])
    steps = tr.steps
    n_train = None
    for e in range(3):
        ep = steps[e * len(steps) // 3: (e + 1) * len(steps) // 3]
        rows = np.concatenate([s[0] for s in ep])
        n_train = n_train or len(rows)
        assert len(rows) == n_train and len(set(rows.tolist())) == n_train            # every training window once per epoch
        assert all(len(s[0]) == 4 for s in ep[:-1]) and 1 <= len(ep[-1][0]) <= 4        # the last partial batch is kept
        for r, l in ep:
            assert np.array_equal(l, row_class[r])                                      # each window has its sequence's label
    train_rows = set(np.concatenate([s[0] for s in steps]).tolist())
    train_seqs = set(row_seq[list(train_rows)].tolist())
    assert set(np.nonzero(np.isin(row_seq, list(train_seqs)))[0].tolist()) == train_rows   # whole sequences only
    held = set(range(len(used))) - train_seqs
    assert len(held) == 3 and {row_class[row_seq == s][0] for s in held} == {0, 1, 2}       # one per class (0.34 x 3)
    n = np.bincount(row_class[sorted(train_rows)], minlength=3)
    assert np.allclose(tr.cw.numpy(), n.sum() / (3 * n))
    # outputs
    head = W.load_head(tmp_path / "out" / "train_head.npz", W.load_weights())
    assert head.class_names == classes
    assert all(np.array_equal(head.arrays[k], tr.init[k]) for k in W.HEAD_KEYS)
    tsv = (tmp_path / "out" / "train_head_training.tsv").read_text().split("\n")
    assert tsv[0] == "epoch\ttrain_loss\tvalidation_loss\tvalidation_window_accuracy\tvalidation_sequence_accuracy"
    assert [x.split("\t")[0] for x in tsv[1:-1]] == ["1", "2", "3"] and tsv[1].split("\t")[1] == "0.500000"
    log = (tmp_path / "out" / "train_head_training.log").read_text()
    assert "2 FASTA record(s) without a label skipped; 1 labelled record(s) without a window skipped" in log


def test_train_head_refusals(tmp_path, stub, trainer_stubs, monkeypatch):
    fa, lab, labels = _train_set(tmp_path / "train.fna")
    bad = tmp_path / "bad.tsv"
    bad.write_text("seq_name\tclass\n" + "".join(f"missing{i}\tred\n" for i in range(12)) + "r0\tblue\n")
    with pytest.raises(SystemExit):
        train_head.main(fa, bad, tmp_path / "o1", verbose=False)
    assert "12 labelled name(s) not found in the FASTA: missing0" in (tmp_path / "o1" / "train_head_training.log").read_text()
    res = CliRunner().invoke(cli.cli, ["train-head", str(fa), str(lab), str(tmp_path / "o2"), "--seed", "-1"])
    assert res.exit_code == 2 and "seed" in res.output.lower()
    assert len(stub.windows_seen()) == 0
