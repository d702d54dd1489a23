"""
CPU tests of nn-classification's output surface over its options: with stub classifier and head objects (tests/window_stub.py,
tests/head_stub.py and the attribution stubs of the module tests) behind the real chunk loop and main(), on the toy input with
its find-proviruses directory (so the provirus job runs too), the header lists exactly the files that the run leaves in the
output directory, and a second run without --restart skips both classifications.
"""
import re
import shutil
from pathlib import Path

import numpy as np
import pytest
import torch

import head_stub as HS
import window_stub as WS
from genomad_b200 import _paths, nn_classification
from test_head_attr_module_cpu import stub_head_attr, stub_head_logp
from test_ig_module_cpu import IGStub
from test_novelty_attr_module_cpu import NovAttrHead
from test_novelty_cpu import CLASSES, write_novelty_head
from test_strands_cpu import EmbedStub, stub_emb

INPUT = Path(__file__).resolve().parent / "golden" / "reference_module" / "input"


class Classifier(IGStub, EmbedStub):
    """Answers every classifier call of the chunk loop: the plain, embedding and attribution routes and embed_ascii."""

    def embed_ascii(self, d_win):
        win = d_win.numpy()
        return torch.from_numpy(WS.stub_probs(win)), torch.from_numpy(stub_emb(win))


class Head(NovAttrHead):
    """A head with a novelty model and every head attribution call."""

    def _scores(self, d_win, target):
        win = d_win.numpy().copy()
        self.clf.seen.append(win)
        return (win, self.class_names.index(target), torch.from_numpy(WS.stub_probs(win)),
                torch.from_numpy(HS.stub_head_probs(stub_emb(win), self.n_classes)))

    def attribute_ascii(self, d_win, target):
        win, c, p, hp = self._scores(d_win, target)
        return p, hp, torch.from_numpy(stub_head_attr(win, c))

    def integrated_gradients_ascii(self, d_win, target, steps, baseline):
        win, c, p, hp = self._scores(d_win, target)
        return (p, hp, torch.from_numpy(stub_head_logp(win, c, self.n_classes, baseline)),
                torch.from_numpy(stub_head_attr(win, c, steps, baseline)))


@pytest.fixture
def stub(monkeypatch):
    clf = Classifier()
    WS.install(monkeypatch.setattr, nn_classification, clf)
    monkeypatch.setattr(nn_classification, "_make_head", Head)
    for k in ("GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS", "GENOMAD_B200_ATTRIBUTIONS",
              "GENOMAD_B200_BOTH_STRANDS", "GENOMAD_B200_HEAD_ATTRIBUTIONS", "GENOMAD_B200_NOVELTY_ATTRIBUTIONS",
              "GENOMAD_B200_WINDOW_NOVELTY", "GENOMAD_B200_ATTRIBUTION_STEPS", "GENOMAD_B200_ATTRIBUTION_BASELINE",
              "GENOMAD_B200_CONTIG_REDUCE", "GENOMAD_B200_TFRECORDS", "RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    return clf


# (name, main() options); "head" is "plain" (a head file without a novelty model) or "novelty"
CASES = [
    ("plain", {}),
    ("embeddings", {"write_embeddings": True}),
    ("windows_6000", {"window_stride": 6000}),
    ("windows_2000", {"window_stride": 2000}),
    ("attributions", {"write_attributions": "virus"}),
    ("attributions_ig", {"write_attributions": "plasmid", "attribution_steps": 3, "attribution_baseline": "N"}),
    ("attributions_embeddings_head", {"write_attributions": "plasmid", "write_embeddings": True, "head": "novelty"}),
    ("strands", {"both_strands": True, "write_embeddings": True}),
    ("head", {"head": "plain"}),
    ("head_novelty", {"head": "novelty"}),
    ("head_everything", {"head": "novelty", "both_strands": True, "window_stride": 2000, "write_embeddings": True}),
    ("head_attributions", {"head": "plain", "write_head_attributions": "k1"}),
    ("head_attributions_ig", {"head": "novelty", "write_head_attributions": CLASSES[2], "attribution_steps": 2}),
    ("novelty_attributions", {"head": "novelty", "write_novelty_attributions": True}),
    ("novelty_attributions_ig", {"head": "novelty", "write_novelty_attributions": True, "attribution_steps": 2}),
    ("window_novelty", {"head": "novelty", "write_window_novelty": True}),
    ("window_novelty_2000", {"head": "novelty", "write_window_novelty": True, "window_stride": 2000}),
    ("single_window", {"single_window": True, "head": "novelty", "window_stride": 6000, "both_strands": True,
                       "write_window_novelty": True, "write_novelty_attributions": True}),
    ("cleanup", {"cleanup": True, "write_embeddings": True, "window_stride": 3000, "head": "plain"}),
    ("provirus_without_windows", {"provirus_without_windows": True, "head": "novelty", "window_stride": 2000,
                                  "both_strands": True, "write_embeddings": True, "write_novelty_attributions": True,
                                  "write_window_novelty": True}),
    ("provirus_without_windows_attributions", {"provirus_without_windows": True, "write_attributions": "chromosome",
                                               "attribution_steps": 2}),
]


def run_case(root: Path, kw: dict) -> _paths.NNOutputs:
    """The toy input and its find-proviruses directory under root, then one main() run with the case's options."""
    kw = dict(kw)
    out = root / "out"
    if not out.exists():
        shutil.copytree(INPUT / "toy_find_proviruses", out / "toy_find_proviruses")
        shutil.copy(INPUT / "toy.fna", root / "toy.fna")
        if kw.get("provirus_without_windows"):           # every provirus record is dropped by the N rule
            (out / "toy_find_proviruses" / "toy_provirus.fna").write_text(">toy_provirus_1\n" + "N" * 7000 + "\n")
    kw.pop("provirus_without_windows", None)
    head = kw.pop("head", None)
    if head == "plain":
        kw["head"] = HS.write_head(root / "plain_head.npz", 3, 1)
    elif head == "novelty":
        kw["head"] = write_novelty_head(root / "novelty_head.npz")
    nn_classification.main(root / "toy.fna", out, kw.pop("single_window", False), 128, False, 2, False,
                           kw.pop("cleanup", False), **kw)
    return _paths.NNOutputs("toy", out)


def header_files(log: str) -> list:
    """The names the log's header lists under the output directory."""
    lines = log.split("Outputs:\n", 1)[1].splitlines()
    return [m.group(1) for m in map(re.compile(r"^ {4}(\S+) \(").match, lines[1:]) if m]


@pytest.mark.parametrize("name,kw", CASES, ids=[c[0] for c in CASES])
def test_header_lists_the_outputs_and_a_rerun_skips(tmp_path, stub, name, kw):
    o = run_case(tmp_path, kw)
    listed = header_files(o.nn_classification_log.read_text())
    assert len(listed) == len(set(listed))
    present = {p.name for p in o.nn_classification_dir.iterdir()}
    if kw.get("cleanup"):                                  # the encoded-data directories are listed, then deleted
        assert not {o.encoded_sequences_dir.name, o.encoded_proviruses_dir.name} & present
        present |= {o.encoded_sequences_dir.name, o.encoded_proviruses_dir.name}
    assert set(listed) == present
    assert o.provirus_nn_classification_output.name in listed
    if kw.get("provirus_without_windows"):
        assert len(np.load(o.provirus_nn_classification_npz_output)["provirus_names"]) == 0

    run_case(tmp_path, kw)
    log = o.nn_classification_log.read_text()
    assert f"{o.nn_classification_npz_output.name} was found. Skipping sequence classification." in log
    assert f"{o.provirus_nn_classification_npz_output.name} was found. Skipping provirus classification." in log
    assert set(header_files(log)) == set(listed)
