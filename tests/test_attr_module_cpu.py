"""
CPU tests of `nn-classification --write-attributions` with a stub classifier (tests/window_stub.py) behind the module's real
chunk loop: the file's name, keys, dtypes and window coordinates, that the contig pass itself runs through the attribution calls
(no second pass, unchanged predictions), the re-run rules, and byte-identical outputs with the option off.
"""
import json

import numpy as np
import pytest
import torch

import window_stub as WS
from genomad_b200 import _paths, nn_classification, sequence
from test_window_scores_cpu import _contig_outputs, _module_fasta, _run

TOK = 5997


def stub_attr(win: np.ndarray, target: str) -> np.ndarray:
    """uint8 [m, 6000] -> float32 [m, 5997], a function of the window's bytes, the position and the class."""
    c = ("chromosome", "plasmid", "virus").index(target) + 1
    w = win[:, :TOK].astype(np.float64)
    return ((w * c + np.arange(TOK) % 7) / 1000.0).astype(np.float32)


class AttrStub(WS.StubClassifier):
    """Also answers attribute_ascii: probabilities as classify_host_into, attributions stub_attr."""

    def __init__(self):
        super().__init__()
        self.attr_calls = 0

    def attribute_ascii(self, d_win, target):
        win = d_win.numpy().copy()
        self.seen.append(win)
        self.attr_calls += 1
        return torch.from_numpy(WS.stub_probs(win)), torch.from_numpy(stub_attr(win, target))


@pytest.fixture
def stub(monkeypatch):
    clf = AttrStub()
    WS.install(monkeypatch.setattr, nn_classification, clf)
    for k in ("GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS", "GENOMAD_B200_ATTRIBUTIONS"):
        monkeypatch.delenv(k, raising=False)
    return clf


def _all_files(out):
    return {p.relative_to(out).as_posix(): p.read_bytes() for p in sorted(out.rglob("*")) if p.is_file() and p.suffix != ".log"}


@pytest.mark.parametrize("single_window", [False, True])
def test_attributions_file_is_the_contig_pass(tmp_path, stub, single_window):
    fa = _module_fasta(tmp_path / "sample.fna")
    o_off = _run(fa, tmp_path / "off", single_window=single_window)
    n = len(stub.windows_seen())
    o_on = _run(fa, tmp_path / "on", single_window=single_window, write_attributions="plasmid")
    assert len(stub.windows_seen()) == 2 * n and stub.attr_calls > 0            # one pass, through the attribution calls
    assert _contig_outputs(o_off) == _contig_outputs(o_on)                      # predictions bitwise unchanged
    assert not o_off.nn_classification_attributions_output.exists()
    j_off, j_on = (json.loads(o.nn_classification_execution_info.read_text()) for o in (o_off, o_on))
    assert j_on["parameters"] == j_off["parameters"] == {"single_window": single_window}
    z = np.load(o_on.nn_classification_attributions_output)
    assert set(z.files) == {"contig_names", "window_contig", "window_start", "window_length", "target", "attributions"}
    assert z["window_contig"].dtype == np.int32 and z["window_start"].dtype == np.int64
    assert z["window_length"].dtype == np.int32 and z["attributions"].dtype == np.float32
    assert str(z["target"]) == "plasmid" and z["attributions"].shape == (n, TOK)
    seen = stub.windows_seen()[n:]
    assert np.array_equal(z["attributions"], stub_attr(seen, "plasmid"))
    preds = np.load(o_on.nn_classification_npz_output)
    assert list(z["contig_names"]) == list(preds["contig_names"])
    raw = {sequence.accession(h): s for h, s in sequence.iter_fasta(fa, strip_n=False)}
    names = list(z["contig_names"])
    for i, (c, s, ln) in enumerate(zip(z["window_contig"], z["window_start"], z["window_length"])):
        assert raw[names[c]][s: s + ln].upper().ljust(6000, b"N") == seen[i].tobytes()
    assert "sample_nn_classification_attributions.npz" in o_on.nn_classification_log.read_text()
    assert "_attributions.npz" not in o_off.nn_classification_log.read_text()


def test_with_window_scores_one_pass(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    o = _run(fa, tmp_path / "on", write_window_scores=True, write_attributions="virus")
    n = len(stub.windows_seen())
    zw, za = np.load(o.nn_classification_windows_npz_output), np.load(o.nn_classification_attributions_output)
    assert len(za["attributions"]) == len(zw["predictions"]) == n
    for k in ("window_contig", "window_start", "window_length"):
        assert np.array_equal(zw[k], za[k]), k
    assert np.array_equal(za["attributions"], stub_attr(stub.windows_seen(), "virus"))


def test_option_off_is_byte_identical(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    a = _run(fa, tmp_path / "a")
    b = _run(fa, tmp_path / "b", write_attributions=None)
    fa_, fb_ = _all_files(tmp_path / "a"), _all_files(tmp_path / "b")
    assert fa_.keys() == fb_.keys()
    # text outputs byte for byte; NPZ members by content (a zip member's timestamp is not part of the result); the JSON's
    # parameters (it also records the run's time)
    assert all(fa_[k] == fb_[k] for k in fa_ if k.endswith(".tsv"))
    for k in (k for k in fa_ if k.endswith(".npz")):
        za, zb = np.load(tmp_path / "a" / k), np.load(tmp_path / "b" / k)
        assert za.files == zb.files and all(np.array_equal(za[m], zb[m]) for m in za.files), k
    assert _contig_outputs(a) == _contig_outputs(b)
    assert (json.loads(a.nn_classification_execution_info.read_text())["parameters"]
            == json.loads(b.nn_classification_execution_info.read_text())["parameters"])
    la = [ln.split(" ", 1)[-1] for ln in a.nn_classification_log.read_text().replace(str(tmp_path / "a"), "X").splitlines()]
    lb = [ln.split(" ", 1)[-1] for ln in b.nn_classification_log.read_text().replace(str(tmp_path / "b"), "X").splitlines()]
    assert len(la) == len(lb)
    assert stub.attr_calls == 0


def test_restart_rules(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    out = tmp_path / "out"
    o = _run(fa, out, write_attributions="virus")
    before, n1 = _contig_outputs(o), len(stub.windows_seen())
    _run(fa, out, write_attributions="virus")                                 # everything found: skipped
    assert len(stub.windows_seen()) == n1
    _run(fa, out, write_attributions="plasmid")                               # another class: classified again
    assert len(stub.windows_seen()) == 2 * n1 and _contig_outputs(o) == before
    assert str(np.load(o.nn_classification_attributions_output)["target"]) == "plasmid"
    o.nn_classification_attributions_output.unlink()                         # missing file: classified again
    _run(fa, out, write_attributions="plasmid")
    assert len(stub.windows_seen()) == 3 * n1 and _contig_outputs(o) == before
    _run(fa, out, write_attributions="plasmid", cleanup=True)                # --cleanup keeps the file
    assert len(stub.windows_seen()) == 3 * n1 and o.nn_classification_attributions_output.exists()
    _run(fa, out)                                                             # option off: nothing redone, file left alone
    assert len(stub.windows_seen()) == 3 * n1 and o.nn_classification_attributions_output.exists()


def test_environment_variable_and_cli(tmp_path, stub, monkeypatch):
    fa = _module_fasta(tmp_path / "sample.fna")
    monkeypatch.setenv("GENOMAD_B200_ATTRIBUTIONS", "chromosome")
    o = _run(fa, tmp_path / "env")
    assert str(np.load(o.nn_classification_attributions_output)["target"]) == "chromosome"
    monkeypatch.setenv("GENOMAD_B200_ATTRIBUTIONS", "0")
    o = _run(fa, tmp_path / "env0")
    assert not o.nn_classification_attributions_output.exists()
    monkeypatch.delenv("GENOMAD_B200_ATTRIBUTIONS")
    with pytest.raises(ValueError):
        _run(fa, tmp_path / "bad", write_attributions="phage")
    from click.testing import CliRunner
    from genomad_b200 import cli
    seen = {}
    monkeypatch.setattr(nn_classification, "main", lambda *a, **k: seen.update(k))
    r = CliRunner().invoke(cli.cli, ["nn-classification", "--write-attributions", "virus", str(fa), str(tmp_path / "o")])
    assert r.exit_code == 0, r.output
    assert seen == {"write_embeddings": None, "write_attributions": "virus"}
    r = CliRunner().invoke(cli.cli, ["nn-classification", "--write-attributions", "phage", str(fa), str(tmp_path / "o")])
    assert r.exit_code != 0
    r = CliRunner().invoke(cli.cli, ["nn-classification", "--help"])
    assert "24 KB per window" in r.output


def test_provirus_twin(tmp_path, stub, golden_dir):
    import shutil
    inp = golden_dir / "reference_module" / "input"
    out = tmp_path / "out"
    shutil.copytree(inp / "toy_find_proviruses", out / "toy_find_proviruses")
    nn_classification.main(inp / "toy.fna", out, False, 128, False, 2, False, False, write_attributions="virus")
    o = _paths.NNOutputs("toy", out)
    zp = np.load(o.provirus_nn_classification_attributions_output)
    assert "provirus_names" in zp.files and str(zp["target"]) == "virus"
    assert zp["attributions"].shape[1] == TOK and len(zp["window_contig"]) == len(zp["attributions"])
    assert o.nn_classification_attributions_output.exists()
