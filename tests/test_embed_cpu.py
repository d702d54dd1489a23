"""
CPU tests of the encoder-embedding feature: the CPU encoder restatement (tests/encoder_ref.py) against the reference encoder's
golden outputs, the `--write-embeddings` / GENOMAD_B200_EMBEDDINGS plumbing of the module (stubbed classifier), its restart rule,
and what ptxas made of the new kernel and the changed dense epilogue.
"""
import json
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from genomad_b200 import _paths, nn_classification
from genomad_b200 import build as B
from oracle import igloo_model as M
import encoder_ref as E

GOLD = Path(__file__).resolve().parent / "golden"
ROOT = GOLD.parents[1]


# ------------------------------------------------------------------------------------------ CPU encoder vs the reference encoder
@pytest.fixture(scope="module")
def enc_gold():
    return np.load(GOLD / "reference_encoder_golden.npz")


@pytest.fixture(scope="module")
def weights():
    w = M.load_npz_weights(ROOT / "genomad_b200" / "data" / "nn_classifier.npz")
    return {"shipped": w, "synthetic": M.synthetic_igloo_weights(w)}


@pytest.mark.parametrize("inputs", ["graph", "tokens"])
@pytest.mark.parametrize("variant", ["shipped", "synthetic"])
def test_encoder_ref_matches_reference_encoder(enc_gold, weights, inputs, variant):
    tok = enc_gold[f"{inputs}_tokens"]
    ref64 = enc_gold[f"{inputs}_{variant}_fp64"]
    assert ref64.shape == (len(tok), 512) and np.abs(ref64).max() > 5          # the values reach about 10
    o64 = E.encoder(tok, weights[variant], torch.float64)
    assert np.abs(o64 - ref64).max() <= 1e-11
    o32 = E.encoder(tok, weights[variant], torch.float32)
    bar = 1e-4 * np.maximum(1.0, np.abs(ref64).max(axis=1))
    assert (np.abs(o32 - ref64).max(axis=1) <= bar).all()
    assert np.abs(enc_gold[f"{inputs}_{variant}"] - ref64).max() <= 1e-4 * np.abs(ref64).max()


def test_encoder_ref_is_the_first_layer_of_the_oracle_head(enc_gold, weights):
    """The oracle's forward() (which encoder_ref builds on) still matches the reference graph golden, and dense0() followed by
    the rest of the head gives exactly the oracle's probabilities."""
    g = np.load(GOLD / "reference_graph_golden.npz")
    tok = g["tokens"][:8]
    p, im = M.forward(tok, weights["shipped"], torch.float64, return_intermediates=True)
    assert np.abs(p - g["shipped_fp64"][:8]).max() <= 1e-12
    e = E.dense0(im["h0"], weights["shipped"], torch.float64)
    w = weights["shipped"]
    h2 = torch.relu((M._t(w, "bn1g", torch.float64) * (e @ M._t(w, "d1w", torch.float64) + M._t(w, "d1b", torch.float64)
                                                       - M._t(w, "bn1m", torch.float64))
                     / torch.sqrt(M._t(w, "bn1v", torch.float64) + M.BN_EPS) + M._t(w, "bn1b", torch.float64)))
    logits = h2 @ M._t(w, "d2w", torch.float64) + M._t(w, "d2b", torch.float64)
    assert np.array_equal(torch.softmax(logits, -1).numpy(), p)


# ------------------------------------------------------------------------------------------ module plumbing (stubbed GPU stage)
def _write_fasta(path, lengths, seed=0):
    rng = np.random.default_rng(seed)
    with open(path, "w") as fh:
        for i, ln in enumerate(lengths):
            s = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, ln)].tobytes().decode()
            fh.write(f">contig_{i:03d} d\n" + "\n".join(s[k:k + 60] for k in range(0, ln, 60)) + "\n")


def _stub_emb(offsets):
    n = len(offsets) - 1
    return (np.arange(n, dtype=np.float32)[:, None] + np.arange(512, dtype=np.float32)[None] / 512).astype(np.float32)


@pytest.fixture
def stub(monkeypatch):
    calls = []
    monkeypatch.setattr(nn_classification, "_make_classifier", lambda batch_size, device: object())

    def fake_classify(clf, parsed, offsets, info, contig_reduce="gather", embeddings=False):
        calls.append(embeddings)
        n = len(offsets) - 1
        preds = np.tile(np.array([[0.2, 0.3, 0.5]], np.float32), (n, 1))
        return (preds, _stub_emb(offsets)) if embeddings else preds
    monkeypatch.setattr(nn_classification, "_classify_parsed", fake_classify)
    monkeypatch.delenv("GENOMAD_B200_EMBEDDINGS", raising=False)
    return calls


def _snapshot(o):
    return {p.name: p.read_bytes() for p in (o.nn_classification_output, o.nn_classification_npz_output)}


def test_flag_writes_embeddings_and_keeps_everything_else(tmp_path, stub):
    fa = tmp_path / "sample.fna"
    _write_fasta(fa, [10000, 7000, 3000])
    o_off, o_on = _paths.NNOutputs("sample", tmp_path / "off"), _paths.NNOutputs("sample", tmp_path / "on")
    nn_classification.main(fa, tmp_path / "off", False, 128, False, 2, False, False)
    nn_classification.main(fa, tmp_path / "on", False, 128, False, 2, False, False, write_embeddings=True)
    assert stub == [False, True]
    assert not o_off.nn_classification_embeddings_output.exists()
    assert _snapshot(o_off) == _snapshot(o_on)
    j_off, j_on = (json.loads(o.nn_classification_execution_info.read_text()) for o in (o_off, o_on))
    assert j_on["parameters"] == j_off["parameters"] == {"single_window": False}      # the flag is not a reference parameter
    z = np.load(o_on.nn_classification_embeddings_output)
    assert set(z.files) == {"contig_names", "embeddings"}
    assert z["embeddings"].dtype == np.float32 and z["embeddings"].shape == (3, 512)
    assert list(z["contig_names"]) == list(np.load(o_on.nn_classification_npz_output)["contig_names"])
    with open(o_on.nn_classification_embeddings_output, "rb") as fh:
        assert fh.read(4) == b"PK\x03\x04"
    log_on = o_on.nn_classification_log.read_text()
    assert "sample_nn_classification_embeddings.npz" in log_on
    assert "_embeddings.npz" not in o_off.nn_classification_log.read_text()


def test_environment_variable_reaches_main(tmp_path, stub, monkeypatch):
    fa = tmp_path / "sample.fna"
    _write_fasta(fa, [9000])
    monkeypatch.setenv("GENOMAD_B200_EMBEDDINGS", "1")
    nn_classification.main(fa, tmp_path / "out", False, 128, False, 2, False, False)
    assert stub == [True]
    assert _paths.NNOutputs("sample", tmp_path / "out").nn_classification_embeddings_output.exists()


def test_cli_flag_reaches_main(tmp_path, monkeypatch):
    from click.testing import CliRunner
    from genomad_b200 import cli
    seen = {}
    monkeypatch.setattr(nn_classification, "main", lambda *a, **k: seen.update(k))
    fa = tmp_path / "x.fna"
    _write_fasta(fa, [100])
    r = CliRunner().invoke(cli.cli, ["nn-classification", "--write-embeddings", str(fa), str(tmp_path / "o")])
    assert r.exit_code == 0, r.output
    assert seen == {"write_embeddings": True}
    r = CliRunner().invoke(cli.cli, ["nn-classification", str(fa), str(tmp_path / "o")])
    assert r.exit_code == 0 and seen == {"write_embeddings": None}            # off: the environment variable decides


def test_missing_embeddings_file_reruns_only_that_classification(tmp_path, stub):
    fa = tmp_path / "sample.fna"
    _write_fasta(fa, [10000, 7000])
    out = tmp_path / "out"
    o = _paths.NNOutputs("sample", out)
    nn_classification.main(fa, out, False, 128, False, 2, False, False)                 # flag off: no embeddings file
    before = _snapshot(o)
    nn_classification.main(fa, out, False, 128, False, 2, False, False, write_embeddings=True)
    assert stub == [False, True]                                                         # classification redone for the file
    assert o.nn_classification_embeddings_output.exists() and _snapshot(o) == before
    nn_classification.main(fa, out, False, 128, False, 2, False, False, write_embeddings=True)
    assert stub == [False, True]                                                         # now everything is found: skipped
    nn_classification.main(fa, out, False, 128, False, 2, False, True, write_embeddings=True)   # --cleanup keeps the file
    assert o.nn_classification_embeddings_output.exists()


# ------------------------------------------------------------------------------------------ ptxas report
KERNELS = {"segment_sum_rows_kernel": "_ZN3gnm23segment_sum_rows_kernelEPKfPKiS1_Pf",
           "splitk_reduce_epi_kernel": "_ZN3gnm24splitk_reduce_epi_kernelEPKfPfS2_S2_S2_iiiS1_S1_S1_i"}


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_embedding_kernels_do_not_spill(kernel):
    B.build()
    log = (B.PKG / "build.log").read_text()
    assert f"Compiling entry function '{KERNELS[kernel]}' for 'sm_90a'" in log
    m = re.search(r"Function properties for " + re.escape(KERNELS[kernel]) +
                  r"\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert m, f"no ptxas resource report for {kernel} in build.log"
    assert tuple(map(int, m.groups())) == (0, 0, 0), f"{kernel}: stack frame / spills {m.groups()}"
