"""
CPU tests of `nn-classification --head HEAD --write-novelty-attributions` and `--write-window-novelty` with stub classifier and
head (tests/window_stub.py, tests/head_stub.py, tests/test_novelty_cpu.py) behind the module's real chunk loop: the files'
keys and dtypes; each window attributed against its sequence's nearest class, whose per-sequence mean distance is bitwise the
novelty file's novelty; the window novelty rows at stride 6000 (the contig pass's own, whose per-sequence means are bitwise the
novelty file's distances) and at stride 1000 (the profile pass's); every other file unchanged; the refusals before any work;
restart and skip; the provirus twins; the log and the CLI.
"""
import shutil

import numpy as np
import pytest
import torch
from click.testing import CliRunner

import head_stub as HS
import window_stub as WS
from genomad_b200 import _paths, cli, nn_classification, sequence
from test_novelty_cpu import CLASSES, StubNoveltyHead, model, stub_novelty, write_novelty_head
from test_strands_cpu import EmbedStub, _all_files, stub_emb
from test_window_scores_cpu import _module_fasta, _run

TOK = 5997


def stub_nov_attr(win, tg, steps=0, baseline="zero"):
    w = win[:, :TOK].astype(np.float64)
    return ((w * (np.asarray(tg)[:, None] + 1) + np.arange(TOK) % 7 + steps + (baseline == "N")) / 1000.0).astype(np.float32)


class NovAttrHead(StubNoveltyHead):
    def __init__(self, clf, head_file):
        super().__init__(clf, head_file)
        self.clf = clf
        clf.nov_calls = getattr(clf, "nov_calls", [])

    def _common(self, d_win, tg):
        win = d_win.numpy().copy()
        self.clf.seen.append(win)
        tg = np.asarray(tg)
        assert tg.dtype == np.int32 and tg.shape == (len(win),) and ((tg >= 0) & (tg < self.n_classes)).all()
        return win, torch.from_numpy(WS.stub_probs(win)), torch.from_numpy(stub_novelty(stub_emb(win), self.n_classes))

    def attribute_novelty_ascii(self, d_win, tg):
        win, p, d = self._common(d_win, tg)
        self.clf.nov_calls.append(0)
        return p, d, torch.from_numpy(stub_nov_attr(win, tg))

    def integrated_gradients_novelty_ascii(self, d_win, tg, steps, baseline):
        win, p, d = self._common(d_win, tg)
        self.clf.nov_calls.append(steps)
        dt = np.stack([d.numpy()[np.arange(len(win)), tg], -1.0 - np.asarray(tg, np.float32)], 1).astype(np.float32)
        return p, d, torch.from_numpy(dt), torch.from_numpy(stub_nov_attr(win, tg, steps, baseline))


@pytest.fixture
def stub(monkeypatch):
    clf = EmbedStub()
    WS.install(monkeypatch.setattr, nn_classification, clf)
    monkeypatch.setattr(nn_classification, "_make_head", NovAttrHead)
    for k in ("GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS", "GENOMAD_B200_ATTRIBUTIONS",
              "GENOMAD_B200_BOTH_STRANDS", "GENOMAD_B200_HEAD_ATTRIBUTIONS", "GENOMAD_B200_NOVELTY_ATTRIBUTIONS",
              "GENOMAD_B200_WINDOW_NOVELTY", "GENOMAD_B200_ATTRIBUTION_STEPS", "GENOMAD_B200_ATTRIBUTION_BASELINE",
              "RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    return clf


def _windows(fa, single_window=False, stride=None):
    pf = sequence.ParsedFasta(fa, single_window)
    try:
        src = pf if stride is None else pf.windows(stride)
        win = src.export_windows(0, src.n_windows, np.empty((src.n_windows, 6000), np.uint8))
        offsets = np.asarray(pf.index().offsets) if stride is None else src.spans()[0]
        if stride is not None:
            src.close()
    finally:
        pf.close()
    return win, np.asarray(offsets)


def _segment_mean(rows, offsets):
    return WS.running_mean(np.asarray(rows, np.float32).reshape(len(rows), -1), offsets)


@pytest.mark.parametrize("single_window", [False, True])
@pytest.mark.parametrize("steps,baseline", [(0, "zero"), (4, "N")])
def test_novelty_attributions_file(tmp_path, stub, single_window, steps, baseline):
    hp = write_novelty_head(tmp_path / "h.npz")
    fa = _module_fasta(tmp_path / "sample.fna")
    o0 = _run(fa, tmp_path / "plain", head=hp, single_window=single_window)
    o = _run(fa, tmp_path / "out", head=hp, single_window=single_window, write_novelty_attributions=True,
             attribution_steps=steps, attribution_baseline=baseline)
    assert _all_files(tmp_path / "plain") == _all_files(tmp_path / "out")       # every other file keeps its bytes
    for a, b in ((o0.nn_classification_head_novelty_npz_output, o.nn_classification_head_novelty_npz_output),
                 (o0.nn_classification_head_npz_output, o.nn_classification_head_npz_output)):
        za, zb = np.load(a), np.load(b)
        assert all(np.array_equal(za[k], zb[k], equal_nan=za[k].dtype.kind == "f") for k in za.files)
    z = np.load(o.nn_classification_head_novelty_attributions_output)
    keys = {"contig_names", "window_contig", "window_start", "window_length", "target", "attributions", "target_class",
            "distance", "class_names", "head_sha256"}
    assert set(z.files) == keys | ({"method", "steps", "baseline", "distance_target"} if steps else set())
    win, offsets = _windows(fa, single_window)
    nv = np.load(o.nn_classification_head_novelty_npz_output)
    counts = np.diff(offsets)
    want_tg = np.repeat(nv["nearest_class"], counts)
    assert str(z["target"]) == "nearest_class" and z["target_class"].dtype == np.int32
    assert np.array_equal(z["target_class"], want_tg)
    d = stub_novelty(stub_emb(win), 3)
    assert z["distance"].dtype == np.float32 and z["distance"].tobytes() == d[np.arange(len(win)), want_tg].tobytes()
    assert z["attributions"].dtype == np.float32 and np.array_equal(z["attributions"], stub_nov_attr(win, want_tg, steps, baseline))
    has = counts > 0
    assert np.array_equal(_segment_mean(z["distance"], offsets)[has, 0], nv["novelty"][has])
    assert np.array_equal(z["window_contig"], np.repeat(np.arange(len(counts), dtype=np.int32), counts))
    if steps:
        assert str(z["method"]) == "integrated_gradients" and int(z["steps"]) == steps and str(z["baseline"]) == baseline
        assert z["distance_target"].dtype == np.float32 and np.array_equal(z["distance_target"][:, 0], z["distance"])
    assert stub.nov_calls and set(stub.nov_calls) == {steps}
    log = o.nn_classification_log.read_text()
    assert "nn_classification_head_novelty_attributions.npz" in log


@pytest.mark.parametrize("stride", [6000, 1000])
def test_window_novelty_files(tmp_path, stub, stride):
    hp = write_novelty_head(tmp_path / "h.npz")
    fa = _module_fasta(tmp_path / "sample.fna")
    kw = {} if stride == 6000 else {"window_stride": stride}
    o0 = _run(fa, tmp_path / "plain", head=hp, **kw)
    o = _run(fa, tmp_path / "out", head=hp, write_window_novelty=True, **kw)
    assert _all_files(tmp_path / "plain").items() <= _all_files(tmp_path / "out").items()
    z = np.load(o.nn_classification_head_novelty_windows_npz_output)
    assert set(z.files) == {"contig_names", "window_contig", "window_start", "window_length", "window_stride", "distances",
                            "novelty", "nearest_class", "class_names", "head_sha256"}
    win, offsets = _windows(fa, stride=None if stride == 6000 else stride)
    d = stub_novelty(stub_emb(win), 3)
    assert z["distances"].dtype == np.float32 and z["distances"].tobytes() == d.tobytes()
    assert np.array_equal(z["novelty"], d.min(1)) and z["nearest_class"].dtype == np.int32
    assert np.array_equal(z["nearest_class"], d.argmin(1)) and int(z["window_stride"]) == stride
    if stride == 6000:
        nv = np.load(o.nn_classification_head_novelty_npz_output)
        has = np.diff(offsets) > 0
        assert np.array_equal(_segment_mean(z["distances"], offsets)[has], nv["distances"][has])
    else:
        zw = np.load(o.nn_classification_windows_npz_output)            # --window-stride still implies the window scores
        assert np.array_equal(zw["window_start"], z["window_start"])
    lines = o.nn_classification_head_novelty_windows_output.read_text().split("\n")
    assert lines[0] == "seq_name\tstart\tend\tnovelty\t" + "\t".join(f"{c}_distance" for c in CLASSES)
    assert len(lines) == len(d) + 2
    first = lines[1].split("\t")
    assert first[3] == f"{float(z['novelty'][0]):.4f}" and first[4] == f"{float(d[0, 0]):.4f}"


def test_refusals_before_any_work(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    hp = write_novelty_head(tmp_path / "h.npz")
    with pytest.raises(ValueError, match="needs --head"):
        _run(fa, tmp_path / "a", write_novelty_attributions=True)
    with pytest.raises(ValueError, match="needs --head"):
        _run(fa, tmp_path / "b", write_window_novelty=True)
    for other in ({"write_attributions": "virus"}, {"write_head_attributions": "gc35"}):
        with pytest.raises(ValueError, match="one attribution file"):
            _run(fa, tmp_path / "c", head=hp, write_novelty_attributions=True, **other)
    plain = HS.write_head(tmp_path / "plain.npz", 3, 1, names=CLASSES)
    for opt in ("write_novelty_attributions", "write_window_novelty"):
        with pytest.raises(SystemExit):
            _run(fa, tmp_path / opt, head=plain, **{opt: True})
        o = _paths.NNOutputs("sample", tmp_path / opt)
        assert "carries no novelty model" in o.nn_classification_log.read_text()
        assert not o.nn_classification_npz_output.exists()


def test_restart_and_skip(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    hp = write_novelty_head(tmp_path / "h.npz")
    o = _run(fa, tmp_path / "out", head=hp, write_novelty_attributions=True, write_window_novelty=True)
    n = len(stub.nov_calls)
    _run(fa, tmp_path / "out", head=hp, write_novelty_attributions=True, write_window_novelty=True)
    assert len(stub.nov_calls) == n                                    # current: skipped
    _run(fa, tmp_path / "out", head=hp, write_novelty_attributions=True, write_window_novelty=True, attribution_steps=2)
    assert len(stub.nov_calls) > n and int(np.load(o.nn_classification_head_novelty_attributions_output)["steps"]) == 2
    n = len(stub.nov_calls)
    h2 = write_novelty_head(tmp_path / "h2.npz", nov_seed=5)                    # another head: redone
    _run(fa, tmp_path / "out", head=h2, write_novelty_attributions=True, write_window_novelty=True, attribution_steps=2)
    assert len(stub.nov_calls) > n
    sha = np.load(o.nn_classification_head_novelty_windows_npz_output)["head_sha256"]
    assert str(sha) == str(np.load(o.nn_classification_head_novelty_attributions_output)["head_sha256"])
    _run(fa, tmp_path / "out", head=h2, write_window_novelty=True, window_stride=2000)
    assert int(np.load(o.nn_classification_head_novelty_windows_npz_output)["window_stride"]) == 2000


def test_provirus_twins(tmp_path, stub, golden_dir):
    inp = golden_dir / "reference_module" / "input"
    out = tmp_path / "out"
    shutil.copytree(inp / "toy_find_proviruses", out / "toy_find_proviruses")
    hp = write_novelty_head(tmp_path / "h.npz")
    nn_classification.main(inp / "toy.fna", out, False, 128, False, 2, False, False, head=hp,
                           write_novelty_attributions=True, write_window_novelty=True)
    o = _paths.NNOutputs("toy", out)
    za = np.load(o.provirus_nn_classification_head_novelty_attributions_output)
    zw = np.load(o.provirus_nn_classification_head_novelty_windows_npz_output)
    assert len(za["provirus_names"]) > 0 and len(zw["provirus_names"]) == len(za["provirus_names"])
    assert o.provirus_nn_classification_head_novelty_windows_output.exists()
    nv = np.load(o.provirus_nn_classification_head_novelty_npz_output)
    counts = np.bincount(za["window_contig"], minlength=len(nv["provirus_names"]))
    assert np.array_equal(za["target_class"], np.repeat(nv["nearest_class"], counts))


def test_environment_and_cli(tmp_path, stub, monkeypatch):
    fa = _module_fasta(tmp_path / "sample.fna")
    hp = write_novelty_head(tmp_path / "h.npz")
    monkeypatch.setenv("GENOMAD_B200_WINDOW_NOVELTY", "1")
    o = _run(fa, tmp_path / "env", head=hp)
    assert o.nn_classification_head_novelty_windows_npz_output.exists()
    monkeypatch.delenv("GENOMAD_B200_WINDOW_NOVELTY")
    res = CliRunner().invoke(cli.cli, ["nn-classification", str(fa), str(tmp_path / "cli"), "--head", str(hp),
                                       "--write-novelty-attributions", "--write-window-novelty"])
    assert res.exit_code == 0, res.output
    oc = _paths.NNOutputs("sample", tmp_path / "cli")
    assert oc.nn_classification_head_novelty_attributions_output.exists()
    assert oc.nn_classification_head_novelty_windows_output.exists()
    assert model(3)["novelty_calibration"].size > 0


def test_sequence_without_a_nearest_class_is_refused_by_name():
    dist = np.array([[1.0, 2.0], [np.nan, 1.0], [0.0, 0.0]], np.float32)
    with pytest.raises(Exception, match="^beta: its window distances"):
        nn_classification._novelty_window_targets(dist, [2, 3, 0], np.zeros(0, np.float32), ["alpha", "beta", "gamma"])
    tg = nn_classification._novelty_window_targets(dist[[0, 2]], [2, 0], np.zeros(0, np.float32), ["alpha", "gamma"])
    assert tg.dtype == np.int32 and list(tg) == [0, 0]
