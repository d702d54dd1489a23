"""
CPU tests of `nn-classification --write-attributions CLASS --attribution-steps N [--attribution-baseline {zero,N}]` with a
stub classifier (tests/window_stub.py) behind the module's real chunk loop: the contig pass runs through the
integrated-gradients calls (no second pass, unchanged predictions), the NPZ keys and dtypes, the re-run rules on a target,
steps, baseline or method change, byte-identical gradient x input files, the environment variables, the CLI, the provirus twin.
"""
import json

import numpy as np
import pytest
import torch

import window_stub as WS
from genomad_b200 import _paths, nn_classification
from test_attr_module_cpu import AttrStub, stub_attr
from test_window_scores_cpu import _contig_outputs, _module_fasta, _run

TOK = 5997


def stub_logp(win: np.ndarray, target: str, baseline: str) -> np.ndarray:
    """uint8 [m, 6000] -> float32 [m, 2]: (log p of the stub's probabilities, a constant per target and baseline)"""
    c = ("chromosome", "plasmid", "virus").index(target)
    p = WS.stub_probs(win)[:, c].astype(np.float64)
    return np.stack([np.log(p), np.full(len(win), -1.0 - c - (baseline == "N"))], 1).astype(np.float32)


def stub_ig(win: np.ndarray, target: str, steps: int, baseline: str) -> np.ndarray:
    return stub_attr(win, target) * np.float32(steps) + np.float32(baseline == "N")


class IGStub(AttrStub):
    """Also answers integrated_gradients_ascii."""

    def __init__(self):
        super().__init__()
        self.ig_calls = []

    def integrated_gradients_ascii(self, d_win, target, steps, baseline):
        win = d_win.numpy().copy()
        self.seen.append(win)
        self.ig_calls.append((target, steps, baseline))
        return (torch.from_numpy(WS.stub_probs(win)), torch.from_numpy(stub_logp(win, target, baseline)),
                torch.from_numpy(stub_ig(win, target, steps, baseline)))


@pytest.fixture
def stub(monkeypatch):
    clf = IGStub()
    WS.install(monkeypatch.setattr, nn_classification, clf)
    for k in ("GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS", "GENOMAD_B200_ATTRIBUTIONS",
              "GENOMAD_B200_ATTRIBUTION_STEPS", "GENOMAD_B200_ATTRIBUTION_BASELINE"):
        monkeypatch.delenv(k, raising=False)
    return clf


@pytest.mark.parametrize("single_window", [False, True])
def test_ig_file_is_the_contig_pass(tmp_path, stub, single_window):
    fa = _module_fasta(tmp_path / "sample.fna")
    o_off = _run(fa, tmp_path / "off", single_window=single_window)
    n = len(stub.windows_seen())
    o_on = _run(fa, tmp_path / "on", single_window=single_window, write_attributions="virus", attribution_steps=8,
                attribution_baseline="N")
    assert len(stub.windows_seen()) == 2 * n and stub.attr_calls == 0                # one pass, through the IG calls
    assert stub.ig_calls and set(stub.ig_calls) == {("virus", 8, "N")}
    assert _contig_outputs(o_off) == _contig_outputs(o_on)
    j_off, j_on = (json.loads(o.nn_classification_execution_info.read_text()) for o in (o_off, o_on))
    assert j_on["parameters"] == j_off["parameters"] == {"single_window": single_window}
    z = np.load(o_on.nn_classification_attributions_output)
    assert set(z.files) == {"contig_names", "window_contig", "window_start", "window_length", "target", "attributions",
                            "method", "steps", "baseline", "log_p_target"}
    assert str(z["method"]) == "integrated_gradients" and z["steps"].dtype == np.int32 and int(z["steps"]) == 8
    assert str(z["baseline"]) == "N" and str(z["target"]) == "virus"
    assert z["attributions"].dtype == np.float32 and z["log_p_target"].dtype == np.float32
    seen = stub.windows_seen()[n:]
    assert z["attributions"].shape == (n, TOK) and z["log_p_target"].shape == (n, 2)
    assert np.array_equal(z["attributions"], stub_ig(seen, "virus", 8, "N"))
    assert np.array_equal(z["log_p_target"], stub_logp(seen, "virus", "N"))
    log = o_on.nn_classification_log.read_text()
    assert "integrated gradients, 8 steps, baseline N" in log


def test_gradient_x_input_file_unchanged(tmp_path, stub):
    """Steps 0 (the default) is today's gradient x input: the same calls and the same keys and bytes."""
    fa = _module_fasta(tmp_path / "sample.fna")
    a = _run(fa, tmp_path / "a", write_attributions="plasmid")
    b = _run(fa, tmp_path / "b", write_attributions="plasmid", attribution_steps=0, attribution_baseline="N")
    assert not stub.ig_calls and stub.attr_calls > 0
    za, zb = np.load(a.nn_classification_attributions_output), np.load(b.nn_classification_attributions_output)
    assert za.files == zb.files == ["contig_names", "window_contig", "window_start", "window_length", "target", "attributions"]
    assert all(np.array_equal(za[k], zb[k]) and za[k].dtype == zb[k].dtype for k in za.files)
    la = [ln.split(" ", 1)[-1] for ln in a.nn_classification_log.read_text().replace(str(tmp_path / "a"), "X").splitlines()]
    lb = [ln.split(" ", 1)[-1] for ln in b.nn_classification_log.read_text().replace(str(tmp_path / "b"), "X").splitlines()]
    assert [x for x in la if "attributions" in x] == [x for x in lb if "attributions" in x]
    assert "integrated" not in a.nn_classification_log.read_text()


def test_restart_rules(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    out = tmp_path / "out"
    o = _run(fa, out, write_attributions="virus", attribution_steps=8)
    before, n1 = _contig_outputs(o), len(stub.windows_seen())
    k = 1
    _run(fa, out, write_attributions="virus", attribution_steps=8, attribution_baseline="zero")     # found: skipped
    assert len(stub.windows_seen()) == k * n1
    for kw in ({"attribution_steps": 16}, {"attribution_steps": 16, "attribution_baseline": "N"},
               {"attribution_steps": 16, "attribution_baseline": "N", "write_attributions": "plasmid"},
               {"write_attributions": "plasmid"},                                  # gradient x input now: classified again
               {"write_attributions": "plasmid", "attribution_steps": 16, "attribution_baseline": "N"}):
        kw = {"write_attributions": "virus", **kw}
        _run(fa, out, **kw)
        k += 1
        assert len(stub.windows_seen()) == k * n1, kw
        assert _contig_outputs(o) == before
        _run(fa, out, **kw)                                                         # the same again: skipped
        assert len(stub.windows_seen()) == k * n1, kw
    z = np.load(o.nn_classification_attributions_output)
    assert int(z["steps"]) == 16 and str(z["baseline"]) == "N" and str(z["target"]) == "plasmid"
    _run(fa, out, write_attributions="plasmid", attribution_steps=16, attribution_baseline="N", cleanup=True)
    assert len(stub.windows_seen()) == k * n1 and o.nn_classification_attributions_output.exists()


def test_environment_variables_and_cli(tmp_path, stub, monkeypatch):
    fa = _module_fasta(tmp_path / "sample.fna")
    monkeypatch.setenv("GENOMAD_B200_ATTRIBUTIONS", "chromosome")
    monkeypatch.setenv("GENOMAD_B200_ATTRIBUTION_STEPS", "4")
    monkeypatch.setenv("GENOMAD_B200_ATTRIBUTION_BASELINE", "N")
    o = _run(fa, tmp_path / "env")
    z = np.load(o.nn_classification_attributions_output)
    assert (str(z["target"]), int(z["steps"]), str(z["baseline"])) == ("chromosome", 4, "N")
    monkeypatch.setenv("GENOMAD_B200_ATTRIBUTION_STEPS", "0")
    o = _run(fa, tmp_path / "env0")
    assert "method" not in np.load(o.nn_classification_attributions_output).files
    for k in ("GENOMAD_B200_ATTRIBUTIONS", "GENOMAD_B200_ATTRIBUTION_STEPS", "GENOMAD_B200_ATTRIBUTION_BASELINE"):
        monkeypatch.delenv(k)
    with pytest.raises(ValueError):
        _run(fa, tmp_path / "bad", write_attributions="virus", attribution_steps=4, attribution_baseline="shuffled")
    with pytest.raises(ValueError):
        _run(fa, tmp_path / "bad2", write_attributions="virus", attribution_steps=-1)
    from click.testing import CliRunner
    from genomad_b200 import cli
    seen = {}
    monkeypatch.setattr(nn_classification, "main", lambda *a, **k: seen.update(k))
    r = CliRunner().invoke(cli.cli, ["nn-classification", "--write-attributions", "virus", "--attribution-steps", "8",
                                     "--attribution-baseline", "N", str(fa), str(tmp_path / "o")])
    assert r.exit_code == 0, r.output
    assert seen == {"write_embeddings": None, "write_attributions": "virus", "attribution_steps": 8,
                    "attribution_baseline": "N"}
    seen.clear()
    r = CliRunner().invoke(cli.cli, ["nn-classification", "--write-attributions", "virus", str(fa), str(tmp_path / "o")])
    assert r.exit_code == 0 and seen == {"write_embeddings": None, "write_attributions": "virus"}
    for bad in (["--attribution-steps", "-1"], ["--attribution-baseline", "shuffled"]):
        r = CliRunner().invoke(cli.cli, ["nn-classification", *bad, str(fa), str(tmp_path / "o")])
        assert r.exit_code != 0, bad
    r = CliRunner().invoke(cli.cli, ["nn-classification", "--help"])
    assert "--attribution-steps" in r.output and "--attribution-baseline" in r.output


def test_provirus_twin(tmp_path, stub, golden_dir):
    import shutil
    inp = golden_dir / "reference_module" / "input"
    out = tmp_path / "out"
    shutil.copytree(inp / "toy_find_proviruses", out / "toy_find_proviruses")
    nn_classification.main(inp / "toy.fna", out, False, 128, False, 2, False, False, write_attributions="virus",
                           attribution_steps=4)
    o = _paths.NNOutputs("toy", out)
    zp = np.load(o.provirus_nn_classification_attributions_output)
    assert "provirus_names" in zp.files and str(zp["method"]) == "integrated_gradients" and int(zp["steps"]) == 4
    assert zp["log_p_target"].shape == (len(zp["attributions"]), 2) and len(zp["window_contig"]) == len(zp["attributions"])
    assert "log_p_target" in np.load(o.nn_classification_attributions_output).files


def test_steps_checked_against_the_attribution_context(tmp_path, stub):
    """The steps must fit the attribution context (min(ATTR_MAX_BATCH, the classifier's windows per step); the stub's step is
    16): a larger value fails before the input is indexed or anything is classified."""
    fa = _module_fasta(tmp_path / "sample.fna")
    with pytest.raises(ValueError, match="at most 16"):
        _run(fa, tmp_path / "big", write_attributions="virus", attribution_steps=17)
    assert len(stub.windows_seen()) == 0 and not _paths.NNOutputs("sample", tmp_path / "big").nn_classification_npz_output.exists()
    _run(fa, tmp_path / "fits", write_attributions="virus", attribution_steps=16)
    assert set(stub.ig_calls) == {("virus", 16, "zero")}


def test_options_without_effect_are_reported(tmp_path, stub, monkeypatch):
    fa = _module_fasta(tmp_path / "sample.fna")
    o = _run(fa, tmp_path / "a", attribution_steps=8, attribution_baseline="N")
    assert not o.nn_classification_attributions_output.exists() and not stub.ig_calls and stub.attr_calls == 0
    assert "have no effect without --write-attributions" in o.nn_classification_log.read_text()
    o = _run(fa, tmp_path / "b", write_attributions="virus", attribution_baseline="N")
    assert "method" not in np.load(o.nn_classification_attributions_output).files
    assert "has no effect with --attribution-steps 0" in o.nn_classification_log.read_text()
    o = _run(fa, tmp_path / "c")
    assert "no effect" not in o.nn_classification_log.read_text()
    monkeypatch.setenv("GENOMAD_B200_ATTRIBUTION_STEPS", "eight")                 # invalid even when attributions are off
    with pytest.raises(ValueError, match="integer"):
        _run(fa, tmp_path / "d")
    monkeypatch.setenv("GENOMAD_B200_ATTRIBUTION_STEPS", "0")
    monkeypatch.setenv("GENOMAD_B200_ATTRIBUTION_BASELINE", "shuffled")
    with pytest.raises(ValueError, match="baseline"):
        _run(fa, tmp_path / "e")
