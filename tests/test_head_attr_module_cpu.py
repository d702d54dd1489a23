"""
CPU tests of `nn-classification --head HEAD --write-head-attributions CLASS` with stub classifier and head (tests/window_stub.py,
tests/head_stub.py) behind the module's real chunk loop: the contig pass runs through the head's attribution calls, which also
give the main predictions and the --head scores (bitwise those of runs without the option); the file's keys; the refusals
before any work (no --head, a class the head does not have, combined with --write-attributions); the re-run rules on a class,
head, method, steps or baseline change; the environment variable and the CLI.
"""
import hashlib
import json

import numpy as np
import pytest
import torch

import head_stub as HS
import window_stub as WS
from genomad_b200 import _paths, nn_classification
from test_strands_cpu import EmbedStub, stub_emb
from test_window_scores_cpu import _contig_outputs, _module_fasta, _run

TOK = 5997
NAMES = ("alpha", "beta", "gamma")


def stub_head_attr(win: np.ndarray, c: int, steps: int = 0, baseline: str = "zero") -> np.ndarray:
    """uint8 [m, 6000] -> float32 [m, 5997], a function of the window's bytes, the position, the class and the method"""
    w = win[:, :TOK].astype(np.float64)
    return ((w * (c + 1) + np.arange(TOK) % 5 + steps + (baseline == "N")) / 1000.0).astype(np.float32)


def stub_head_logp(win: np.ndarray, c: int, C: int, baseline: str) -> np.ndarray:
    p = HS.stub_head_probs(stub_emb(win), C)[:, c].astype(np.float64)
    return np.stack([np.log(p), np.full(len(win), -2.0 - c - (baseline == "N"))], 1).astype(np.float32)


class AttrHead(HS.StubHead):
    """Also answers the head's attribution calls; the windows they see are recorded by the classifier stub."""

    def __init__(self, clf, head_file):
        super().__init__(clf, head_file)
        self.clf = clf
        clf.head_calls = getattr(clf, "head_calls", [])

    def _common(self, d_win):
        win = d_win.numpy().copy()
        self.clf.seen.append(win)
        return win, torch.from_numpy(WS.stub_probs(win)), torch.from_numpy(HS.stub_head_probs(stub_emb(win), self.n_classes))

    def attribute_ascii(self, d_win, target):
        c = self.class_names.index(target)
        win, p, hp = self._common(d_win)
        self.clf.head_calls.append((target, 0, None))
        return p, hp, torch.from_numpy(stub_head_attr(win, c))

    def integrated_gradients_ascii(self, d_win, target, steps, baseline):
        c = self.class_names.index(target)
        win, p, hp = self._common(d_win)
        self.clf.head_calls.append((target, steps, baseline))
        return (p, hp, torch.from_numpy(stub_head_logp(win, c, self.n_classes, baseline)),
                torch.from_numpy(stub_head_attr(win, c, steps, baseline)))


@pytest.fixture
def stub(monkeypatch):
    clf = EmbedStub()
    clf.head_calls = []
    WS.install(monkeypatch.setattr, nn_classification, clf)
    monkeypatch.setattr(nn_classification, "_make_head", AttrHead)
    for k in ("GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS", "GENOMAD_B200_ATTRIBUTIONS",
              "GENOMAD_B200_HEAD_ATTRIBUTIONS", "GENOMAD_B200_ATTRIBUTION_STEPS", "GENOMAD_B200_ATTRIBUTION_BASELINE",
              "GENOMAD_B200_BOTH_STRANDS", "RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    return clf


def _head(tmp_path, name="h.npz", seed=1, names=NAMES):
    return HS.write_head(tmp_path / name, len(names), seed, names=names)


def _npz(path):
    z = np.load(path)
    return {k: (z[k].dtype.str, z[k].tobytes()) for k in z.files}


@pytest.mark.parametrize("steps", [0, 4])
def test_file_keys_and_unchanged_outputs(tmp_path, stub, steps):
    fa = _module_fasta(tmp_path / "sample.fna")
    hp = _head(tmp_path)
    plain = _run(fa, tmp_path / "plain")
    only_head = _run(fa, tmp_path / "head", head=hp)
    n = len(stub.windows_seen()) // 2
    kw = {"attribution_steps": steps, "attribution_baseline": "N"} if steps else {}
    o = _run(fa, tmp_path / "on", head=hp, write_head_attributions="beta", **kw)
    assert len(stub.windows_seen()) == 3 * n                         # one pass, through the head's attribution calls
    assert set(stub.head_calls) == {("beta", steps, "N" if steps else None)}
    assert _contig_outputs(o) == _contig_outputs(plain)
    assert _npz(o.nn_classification_head_npz_output) == _npz(only_head.nn_classification_head_npz_output)
    assert o.nn_classification_head_output.read_bytes() == only_head.nn_classification_head_output.read_bytes()
    assert not o.nn_classification_attributions_output.exists()
    j = json.loads(o.nn_classification_execution_info.read_text())
    assert j["parameters"] == {"single_window": False}
    z = np.load(o.nn_classification_head_attributions_output)
    keys = {"contig_names", "window_contig", "window_start", "window_length", "target", "attributions", "head_sha256",
            "class_names"}
    if steps:
        keys |= {"method", "steps", "baseline", "log_p_target"}
    assert set(z.files) == keys
    assert str(z["target"]) == "beta" and list(z["class_names"]) == list(NAMES)
    assert str(z["head_sha256"]) == hashlib.sha256(hp.read_bytes()).hexdigest()
    seen = stub.windows_seen()[2 * n:]
    assert z["attributions"].dtype == np.float32 and np.array_equal(z["attributions"], stub_head_attr(seen, 1, steps, "N" if steps else "zero"))
    zw = np.load(plain.nn_classification_npz_output)
    assert len(z["window_contig"]) == n and len(np.unique(z["window_contig"])) <= len(zw["contig_names"])
    if steps:
        assert str(z["method"]) == "integrated_gradients" and int(z["steps"]) == steps and str(z["baseline"]) == "N"
        assert np.array_equal(z["log_p_target"], stub_head_logp(seen, 1, 3, "N"))
    assert "window attributions of the head (beta" in o.nn_classification_log.read_text()


def test_refusals_before_any_work(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    hp = _head(tmp_path)
    with pytest.raises(ValueError, match="needs --head"):
        _run(fa, tmp_path / "a", write_head_attributions="beta")
    with pytest.raises(ValueError, match="cannot be combined"):
        _run(fa, tmp_path / "b", head=hp, write_head_attributions="beta", write_attributions="virus")
    with pytest.raises(SystemExit) as e:
        _run(fa, tmp_path / "c", head=hp, write_head_attributions="virus")
    assert e.value.code == 1
    assert "not a class of" in _paths.NNOutputs("sample", tmp_path / "c").nn_classification_log.read_text()
    assert len(stub.windows_seen()) == 0
    for d in "abc":
        assert not _paths.NNOutputs("sample", tmp_path / d).nn_classification_npz_output.exists()


def test_restart_rules(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    ha, hb = _head(tmp_path, "a.npz", 1), _head(tmp_path, "b.npz", 2)
    out = tmp_path / "out"
    o = _run(fa, out, head=ha, write_head_attributions="beta")
    n = len(stub.windows_seen())
    before = _contig_outputs(o)
    k = 1
    _run(fa, out, head=ha, write_head_attributions="beta")                       # the same: skipped
    assert len(stub.windows_seen()) == k * n
    o.nn_classification_head_attributions_output.unlink()                          # missing: classified again
    _run(fa, out, head=ha, write_head_attributions="beta")
    k += 1
    assert len(stub.windows_seen()) == k * n
    for kw in ({"write_head_attributions": "gamma"},                                # another class
               {"write_head_attributions": "gamma", "head": hb},                   # another head, same class names
               {"write_head_attributions": "gamma", "head": hb, "attribution_steps": 4},
               {"write_head_attributions": "gamma", "head": hb, "attribution_steps": 4, "attribution_baseline": "N"},
               {"write_head_attributions": "gamma", "head": hb, "attribution_steps": 8, "attribution_baseline": "N"}):
        kw = {"head": ha, **kw}
        _run(fa, out, **kw)
        k += 1
        assert len(stub.windows_seen()) == k * n, kw
        assert _contig_outputs(o) == before
        _run(fa, out, **kw)                                                       # the same again: skipped
        assert len(stub.windows_seen()) == k * n, kw
    z = np.load(o.nn_classification_head_attributions_output)
    assert (str(z["target"]), int(z["steps"]), str(z["baseline"])) == ("gamma", 8, "N")
    assert str(z["head_sha256"]) == hashlib.sha256(hb.read_bytes()).hexdigest()
    _run(fa, out, head=hb, write_head_attributions="gamma", attribution_steps=8, attribution_baseline="N", cleanup=True)
    assert len(stub.windows_seen()) == k * n and o.nn_classification_head_attributions_output.exists()


def test_provirus_twin(tmp_path, stub, golden_dir):
    import shutil
    inp = golden_dir / "reference_module" / "input"
    out = tmp_path / "out"
    shutil.copytree(inp / "toy_find_proviruses", out / "toy_find_proviruses")
    hp = _head(tmp_path)
    nn_classification.main(inp / "toy.fna", out, False, 128, False, 2, False, False, head=hp,
                           write_head_attributions="alpha", attribution_steps=4)
    o = _paths.NNOutputs("toy", out)
    zp = np.load(o.provirus_nn_classification_head_attributions_output)
    assert "provirus_names" in zp.files and str(zp["target"]) == "alpha" and int(zp["steps"]) == 4
    assert zp["log_p_target"].shape == (len(zp["attributions"]), 2) and list(zp["class_names"]) == list(NAMES)
    assert o.nn_classification_head_attributions_output.exists()


def test_environment_variable_cli_and_notes(tmp_path, stub, monkeypatch):
    fa = _module_fasta(tmp_path / "sample.fna")
    hp = _head(tmp_path)
    monkeypatch.setenv("GENOMAD_B200_HEAD_ATTRIBUTIONS", "gamma")
    o = _run(fa, tmp_path / "env", head=hp)
    assert str(np.load(o.nn_classification_head_attributions_output)["target"]) == "gamma"
    monkeypatch.delenv("GENOMAD_B200_HEAD_ATTRIBUTIONS")
    o = _run(fa, tmp_path / "notes", head=hp, attribution_steps=4)
    assert "no effect without --write-attributions or --write-head-attributions" in o.nn_classification_log.read_text()
    assert not o.nn_classification_head_attributions_output.exists()
    from click.testing import CliRunner
    from genomad_b200 import cli
    seen = {}
    monkeypatch.setattr(nn_classification, "main", lambda *a, **k: seen.update(k))
    r = CliRunner().invoke(cli.cli, ["nn-classification", "--head", str(hp), "--write-head-attributions", "beta",
                                     "--attribution-steps", "8", str(fa), str(tmp_path / "o")])
    assert r.exit_code == 0, r.output
    assert seen == {"write_embeddings": None, "head": hp, "write_head_attributions": "beta", "attribution_steps": 8}
    r = CliRunner().invoke(cli.cli, ["nn-classification", "--help"])
    assert "--write-head-attributions" in r.output
