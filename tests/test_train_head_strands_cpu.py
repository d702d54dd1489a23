"""
CPU tests of `train-head --both-strands` with the stub classifier, head and trainer (tests/window_stub.py, tests/head_stub.py)
behind the real module code: X holds the forward rows and then the reverse rows of the used records, the reverse rows are the
stub's embeddings of the reverse list's windows, labels repeat per strand, the split holds out the same sequences as without
the option and keeps both strands of a sequence on one side, the class weights count both strands, and the validation sequence
accuracy uses the strand-averaged scores.
"""
import numpy as np
import pytest

import head_stub as HS
from genomad_b200 import cli, sequence, train_head
from test_head_module_cpu import _train_set, stub, trainer_stubs  # noqa: F401  (fixtures)
from test_strands_cpu import stub_emb

CLASSES = ("blue", "green", "red")


def _strand_set(path):
    """tests/test_head_module_cpu.py's training set plus a labelled record with 2 forward and 3 reverse windows: a run of
    4,400 N fills more than MAX_N of its second forward window but not of any reverse window but the first."""
    fa, lab, labels = _train_set(path)
    rng = np.random.default_rng(9)
    s = bytearray(np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 16000)].tobytes())
    s[6500:10900] = b"N" * 4400
    with open(fa, "ab") as f:
        f.write(b">skewed\n" + bytes(s) + b"\n")
    with open(lab, "a") as f:
        f.write("skewed\tgreen\n")
    labels["skewed"] = "green"
    return fa, lab, labels


def _used_windows(fa, labels):
    """(names, used record indices, forward windows, forward counts, reverse windows, reverse counts) of the used records."""
    pf = sequence.ParsedFasta(fa)
    wl = pf.windows(6000, False, reverse=True)
    try:
        idx = pf.index()
        names = list(idx.names)
        used = [i for i, n in enumerate(names) if n in labels and idx.offsets[i + 1] > idx.offsets[i]]
        roff = wl.spans()[0]

        def take(src, off):
            parts = [src.export_windows(int(off[i]), int(off[i + 1] - off[i]), np.empty((int(off[i + 1] - off[i]), 6000),
                                                                                         np.uint8)) for i in used]
            return np.concatenate(parts), np.array([int(off[i + 1] - off[i]) for i in used])
        fwd, nf = take(pf, idx.offsets)
        rev, nr = take(wl, roff)
    finally:
        wl.close()
        pf.close()
    return names, used, fwd, nf, rev, nr


def _held_out(steps, row_seq):
    train_rows = set(np.concatenate([s[0] for s in steps]).tolist())
    return set(range(row_seq.max() + 1)) - set(row_seq[list(train_rows)].tolist()), train_rows


def test_both_strands_rows_labels_and_split(tmp_path, stub, trainer_stubs):  # noqa: F811
    fa, lab, labels = _strand_set(tmp_path / "train.fna")
    kw = dict(epochs=2, batch_size=4, validation_fraction=0.34, seed=5, verbose=False)
    train_head.main(fa, lab, tmp_path / "one", **kw)
    n_plain = len(stub.windows_seen())
    train_head.main(fa, lab, tmp_path / "both", both_strands=True, **kw)
    plain, tr = trainer_stubs
    names, used, fwd, nf, rev, nr = _used_windows(fa, labels)
    assert (nf != nr).any()                                                  # the N rule: another count on one strand
    Nf, Nr = int(nf.sum()), int(nr.sum())
    # X: the forward rows as today, then the reverse rows; the classifier saw the forward windows, then the reverse ones
    assert tr.X.shape == (Nf + Nr, 512)
    assert np.array_equal(tr.X.numpy()[:Nf], plain.X.numpy())
    assert np.array_equal(tr.X.numpy()[Nf:], stub_emb(rev))
    seen = stub.windows_seen()[n_plain:]
    assert np.array_equal(seen, np.concatenate([fwd, rev]))
    # labels repeat per strand
    seq_cls = np.array([CLASSES.index(labels[names[i]]) for i in used])
    row_seq = np.concatenate([np.repeat(np.arange(len(used)), nf), np.repeat(np.arange(len(used)), nr)])
    row_class = seq_cls[row_seq]
    for r, l in tr.steps:
        assert np.array_equal(l, row_class[r])
    # the same sequences are held out; a training sequence trains on both strands, every row once per epoch
    held_plain, _ = _held_out(plain.steps, row_seq[:Nf])
    held, train_rows = _held_out(tr.steps, row_seq)
    assert held == held_plain and len(held) == 3
    assert train_rows == set(np.nonzero(~np.isin(row_seq, list(held)))[0].tolist())
    ep = tr.steps[: len(tr.steps) // 2]
    rows = np.concatenate([s[0] for s in ep])
    assert len(rows) == len(train_rows) == len(set(rows.tolist()))
    n = np.bincount(row_class[sorted(train_rows)], minlength=3)
    assert np.allclose(tr.cw.numpy(), n.sum() / (3 * n))
    # validation: loss and window accuracy over both strands' rows, sequence accuracy of both_strands(mean f, mean r)
    X = tr.X.numpy()
    probs = HS.stub_head_probs(X, 3)
    hv = sorted(held)
    vf = [np.nonzero((row_seq == s) & (np.arange(Nf + Nr) < Nf))[0] for s in hv]
    vr = [np.nonzero((row_seq == s) & (np.arange(Nf + Nr) >= Nf))[0] for s in hv]
    val_rows = np.concatenate(vf + vr)
    cw = tr.cw.numpy()
    p = np.clip(probs[val_rows, row_class[val_rows]].astype(np.float64), 1e-7, 1.0)
    loss = float((cw[row_class[val_rows]].astype(np.float64) * -np.log(p)).sum() / len(val_rows))
    win_acc = float((probs[val_rows].argmax(1) == row_class[val_rows]).mean())

    def run_mean(rs):
        s = np.zeros(3, np.float32)
        for r in rs:
            s = (s + probs[r]).astype(np.float32)
        return s / np.float32(len(rs))
    both = np.stack([(run_mean(a) + run_mean(b)) * np.float32(0.5) for a, b in zip(vf, vr)])
    seq_acc = float((both.argmax(1) == seq_cls[hv]).mean())
    line = (tmp_path / "both" / "train_head_training.tsv").read_text().split("\n")[1].split("\t")
    assert line[2:] == [f"{loss:.6f}", f"{win_acc:.6f}", f"{seq_acc:.6f}"]
    log = (tmp_path / "both" / "train_head_training.log").read_text()
    assert "Training on both strands" in log and "Training on both strands" not in \
        (tmp_path / "one" / "train_head_training.log").read_text()
    # the head file's format is unchanged
    assert (tmp_path / "both" / "train_head.npz").read_bytes() == (tmp_path / "one" / "train_head.npz").read_bytes()


def test_without_the_option_the_trainer_sees_todays_rows(tmp_path, stub, trainer_stubs):  # noqa: F811
    fa, lab, labels = _strand_set(tmp_path / "train.fna")
    kw = dict(epochs=2, batch_size=4, validation_fraction=0.34, seed=5, verbose=False)
    train_head.main(fa, lab, tmp_path / "a", **kw)
    train_head.main(fa, lab, tmp_path / "b", both_strands=False, **kw)
    a, b = trainer_stubs
    assert np.array_equal(a.X.numpy(), b.X.numpy()) and len(a.steps) == len(b.steps)
    assert all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(a.steps, b.steps))
    assert (tmp_path / "a" / "train_head_training.tsv").read_bytes() == (tmp_path / "b" / "train_head_training.tsv").read_bytes()


def test_cli_flag(tmp_path, monkeypatch):
    from click.testing import CliRunner
    fa, lab, _ = _train_set(tmp_path / "train.fna")
    seen = []
    monkeypatch.setattr(train_head, "main", lambda *a, **k: seen.append(k))
    r = CliRunner().invoke(cli.cli, ["train-head", "--both-strands", str(fa), str(lab), str(tmp_path / "o")])
    assert r.exit_code == 0, r.output
    r = CliRunner().invoke(cli.cli, ["train-head", str(fa), str(lab), str(tmp_path / "o")])
    assert r.exit_code == 0, r.output
    assert seen == [{"both_strands": True}, {}]


def test_memory_check_counts_both_strands(tmp_path, stub, trainer_stubs, monkeypatch):  # noqa: F811
    fa, lab, labels = _strand_set(tmp_path / "train.fna")
    _, _, _, nf, _, nr = _used_windows(fa, labels)
    need = int(nf.sum() + nr.sum()) * train_head.EMBED_BYTES
    monkeypatch.setattr(train_head, "_free_bytes", lambda clf: int(need / 0.9) - 1024)     # room for the forward rows only
    train_head.main(fa, lab, tmp_path / "one", epochs=1, verbose=False)
    with pytest.raises(SystemExit):
        train_head.main(fa, lab, tmp_path / "both", epochs=1, verbose=False, both_strands=True)
    assert "do not fit in the GPU's free memory" in (tmp_path / "both" / "train_head_training.log").read_text()
