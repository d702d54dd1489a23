"""
CPU tests of the reverse strand (`nn-classification --both-strands`): the native reader's reverse window lists and exports against
the reference's own rc() / seq_windows / N rule / ljust (tests/golden/reference_rc_golden.npz) and, at every stride, against
their pure-Python statement; the module's strand files with a stub classifier (tests/window_stub.py) behind its real chunk loop:
file set, keys, dtypes, the strand invariants, byte-identical outputs with the option off, restart, skip and cleanup, the
provirus twin, --single-window, the environment variable and the CLI; the embedding tools' --both-strands input key.
"""
import ctypes as C
import json
import shutil
from pathlib import Path

import numpy as np
import pytest
import torch

import window_stub as WS
from genomad_b200 import _paths, engine, nn_classification, sequence
from test_window_scores_cpu import STRIDES, _contig_outputs, _module_fasta, _run, write_edge_fasta

GOLDEN = Path(__file__).resolve().parent / "golden" / "reference_rc_golden.npz"
EMBED = 512


@pytest.fixture(scope="module")
def golden(tmp_path_factory):
    z = dict(np.load(GOLDEN))
    path = tmp_path_factory.mktemp("rc") / "rc.fna"
    path.write_bytes(z["fasta"].tobytes())
    return z, path


# ------------------------------------------------------------------------------------------ the reader's reverse lists
@pytest.mark.parametrize("threads", [1, 7])
@pytest.mark.parametrize("single_window", [False, True])
def test_reverse_list_is_the_reference(golden, threads, single_window):
    z, path = golden
    sfx = "_single" if single_window else ""
    pf = sequence.ParsedFasta(path, single_window, threads=threads)
    wl = pf.windows(6000, single_window, reverse=True)
    try:
        assert pf.n_contigs == len(z["names" + sfx]) and wl.n_windows == len(z["windows" + sfx])
        assert list(pf.index().names) == list(z["names" + sfx])
        offsets, starts, lengths = wl.spans()
        assert np.array_equal(offsets, z["offsets" + sfx])
        assert np.array_equal(starts, z["starts" + sfx]) and np.array_equal(lengths, z["lengths" + sfx])
        got = wl.export_windows(0, wl.n_windows, np.empty((wl.n_windows, 6000), np.uint8))
        assert np.array_equal(got, z["windows" + sfx])
        part = np.empty((5, 6000), np.uint8)                                # any block of the list
        assert np.array_equal(wl.export_windows(3, 5, part), z["windows" + sfx][3:8])
    finally:
        wl.close()
        pf.close()


def test_golden_covers_the_edges(golden):
    """The fixture holds windows the N rule drops on one strand only, and the forward list differs from the reverse one."""
    z, path = golden
    names = list(z["names"])
    fwd_counts = {}
    pf = sequence.ParsedFasta(path)
    enc = pf.encode()
    pf.close()
    for i, n in enumerate(enc.names):
        fwd_counts[n] = int(enc.offsets[i + 1] - enc.offsets[i])
    rev_counts = {n: int(z["offsets"][i + 1] - z["offsets"][i]) for i, n in enumerate(names)}
    assert fwd_counts["n_rule_forward_only"] == 1 and rev_counts["n_rule_forward_only"] == 2
    assert fwd_counts["n_rule_reverse_only"] == 2 and rev_counts["n_rule_reverse_only"] == 1
    assert fwd_counts["n_rule_lowercase_n"] == rev_counts["n_rule_lowercase_n"] == 2
    assert "all_n" not in names and "empty" not in names
    assert any(fwd_counts[n] != rev_counts[n] for n in names if n == "long_many_windows")


def expected_rc_windows(path, stride, single_window=False):
    """Pure-Python statement: per kept record, rc_spans + the N rule on the forward segment + reverse_complement."""
    out, names = [], []
    for header, raw in sequence.iter_fasta(path, strip_n=False):
        seq = raw.strip(b"nN")
        if not seq:
            continue
        lead = len(raw) - len(raw.lstrip(b"nN"))
        for k, (s, e) in enumerate(sequence.rc_spans(len(seq), stride, single_window)):
            if k > 0 and seq[s:e].count(b"N") > sequence.MAX_N:
                continue
            out.append((len(names), lead + s, e - s, sequence.reverse_complement(seq[s:e]).upper().ljust(6000, b"N")))
        names.append(sequence.accession(header))
    return names, out


@pytest.mark.parametrize("stride", STRIDES)
def test_reverse_list_at_any_stride(tmp_path, stride):
    fa = write_edge_fasta(tmp_path / "edge.fna", stride, seed=stride + 1)
    names, exp = expected_rc_windows(fa, stride)
    pf = sequence.ParsedFasta(fa, threads=4)
    wl = pf.windows(stride, reverse=True)
    try:
        assert wl.n_contigs == len(names) and wl.n_windows == len(exp)
        offsets, starts, lengths = wl.spans()
        cid = np.array([e[0] for e in exp], np.int64)
        assert np.array_equal(offsets, np.concatenate([[0], np.cumsum(np.bincount(cid, minlength=len(names)))]))
        assert np.array_equal(starts, [e[1] for e in exp]) and np.array_equal(lengths, [e[2] for e in exp])
        buf = np.empty((len(exp), 6000), np.uint8)
        got = wl.export_windows(0, len(exp), buf)
        assert all(got[i].tobytes() == e[3] for i, e in enumerate(exp))
    finally:
        wl.close()
        pf.close()


def test_reverse_complement_is_the_reference_table():
    assert sequence.reverse_complement(b"ACTGNactgnRYUuX-") == b"-XuUYRncagtNCAGT"
    assert sequence.rc_spans(10000) == [(4000, 10000), (0, 4000)]
    assert sequence.rc_spans(10000, single_window=True) == [(4000, 10000)]
    assert sequence.rc_spans(8000) == [(2000, 8000)]                        # a 2,000-nt tail is not a window
    pf = sequence.ParsedFasta(GOLDEN.parent / "reference_module" / "input" / "toy.fna")
    try:
        for bad in (0, 6001):
            with pytest.raises(RuntimeError, match="gnm_fasta_windows_plan_rc: stride must be in"):
                pf.windows(bad, reverse=True)
    finally:
        pf.close()


def test_both_strands_helper():
    a = np.array([[0.1, 0.2, 0.7]], np.float32)
    b = np.array([[0.3, 0.3, 0.4]], np.float32)
    got = engine.both_strands(a, b)
    assert got.dtype == np.float32 and np.array_equal(got, (a + b) * np.float32(0.5))
    assert np.array_equal(engine.both_strands(b, a), got)
    t = engine.both_strands(torch.from_numpy(a), torch.from_numpy(b))
    assert t.dtype == torch.float32 and np.array_equal(t.numpy(), got)


# ------------------------------------------------------------------------------------------ module (stubbed classifier)
def stub_emb(win: np.ndarray) -> np.ndarray:
    """uint8 [m, 6000] -> float32 [m, 512], a function of the window's bytes."""
    x = win[:, :EMBED].astype(np.float32) + win[:, EMBED: 2 * EMBED].astype(np.float32) * np.float32(0.37)
    return (x * np.linspace(0.01, 1.0, EMBED, dtype=np.float32)).astype(np.float32)


def np_segment_sum_rows(rows, offsets, carry=None):
    k = len(offsets) - 1
    sums = np.zeros((k, rows.shape[1]), np.float32)
    for c in range(k):
        s = np.array(carry, np.float32).copy() if (c == 0 and carry is not None) else np.zeros(rows.shape[1], np.float32)
        for i in range(offsets[c], offsets[c + 1]):
            s = (s + rows[i]).astype(np.float32)
        sums[c] = s
    return sums, (sums[k - 1].copy() if k else np.zeros(rows.shape[1], np.float32))


class EmbedStub(WS.StubClassifier):
    """Also answers the embedding calls: embed_host_into (probabilities as classify_host_into, rows stub_emb) and
    segment_sum_rows (gnm_segment_sum_rows' fp32 running sums)."""

    def embed_host_into(self, ascii_ptr, n, probs_ptr, d_embed_ptr):
        self.classify_host_into(ascii_ptr, n, probs_ptr)
        emb = np.ctypeslib.as_array((C.c_float * (n * EMBED)).from_address(d_embed_ptr)).reshape(n, EMBED)
        emb[:] = stub_emb(self.seen[-1])

    def segment_sum_rows(self, rows, offsets, carry=None):
        s, c = np_segment_sum_rows(rows.numpy(), offsets.numpy(), None if carry is None else carry.numpy())
        return torch.from_numpy(s), torch.from_numpy(c)


@pytest.fixture
def stub(monkeypatch):
    clf = EmbedStub()
    WS.install(monkeypatch.setattr, nn_classification, clf)
    for k in ("GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS", "GENOMAD_B200_ATTRIBUTIONS",
              "GENOMAD_B200_BOTH_STRANDS"):
        monkeypatch.delenv(k, raising=False)
    return clf


def _all_files(out):
    return {p.relative_to(out).as_posix(): p.read_bytes() for p in sorted(out.rglob("*"))
            if p.is_file() and p.suffix not in (".log", ".npz", ".json")}          # the JSON and the log carry times


def _npz(path):
    z = np.load(path)
    return {k: (z[k].dtype.str, z[k].shape, z[k].tobytes()) for k in z.files}


def _rc_fasta(src, dst):
    """Every record of src reverse-complemented with the 10-letter table, 60 per line."""
    with open(dst, "wb") as fh:
        for h, s in sequence.iter_fasta(src, strip_n=False):
            r = sequence.reverse_complement(s)
            fh.write(f">{h}\n".encode() + b"\n".join(r[i:i + 60] for i in range(0, len(r), 60)) + b"\n")
    return dst


@pytest.mark.parametrize("single_window", [False, True])
def test_strand_files_and_invariants(tmp_path, stub, single_window):
    fa = _module_fasta(tmp_path / "sample.fna")
    (tmp_path / "rc").mkdir()
    fr = _rc_fasta(fa, tmp_path / "rc" / "sample.fna")
    o_off = _run(fa, tmp_path / "off", single_window=single_window, write_embeddings=True)
    o = _run(fa, tmp_path / "on", single_window=single_window, write_embeddings=True, both_strands=True)
    o_rc = _run(fr, tmp_path / "rc_on", single_window=single_window, write_embeddings=True, both_strands=True)
    o_rc_plain = _run(fr, tmp_path / "rc_off", single_window=single_window, write_embeddings=True)
    # the main outputs do not change, nor does the embeddings file's "embeddings" array
    assert _contig_outputs(o_off) == _contig_outputs(o)
    assert json.loads(o.nn_classification_execution_info.read_text())["parameters"] == {"single_window": single_window}
    e_off, e_on = np.load(o_off.nn_classification_embeddings_output), np.load(o.nn_classification_embeddings_output)
    assert set(e_on.files) == {"contig_names", "embeddings", "embeddings_reverse", "embeddings_both_strands"}
    assert e_on["embeddings"].tobytes() == e_off["embeddings"].tobytes()
    assert not o_off.nn_classification_strands_npz_output.exists()
    z = np.load(o.nn_classification_strands_npz_output)
    assert set(z.files) == {"contig_names", "forward", "reverse", "both_strands"}
    assert all(z[k].dtype == np.float32 and z[k].shape == (len(z["contig_names"]), 3) for k in nn_classification.STRANDS)
    assert z["forward"].tobytes() == np.load(o.nn_classification_npz_output)["predictions"].tobytes()
    # reverse(F) == forward(F') == a plain run on F'; both(F) == both(F'); the same for embeddings; all bitwise
    zr = np.load(o_rc.nn_classification_strands_npz_output)
    er = np.load(o_rc.nn_classification_embeddings_output)
    assert np.array_equal(z["reverse"], zr["forward"]) and np.array_equal(zr["reverse"], z["forward"])
    assert np.array_equal(z["reverse"], np.load(o_rc_plain.nn_classification_npz_output)["predictions"])
    assert np.array_equal(z["both_strands"], zr["both_strands"])
    assert np.array_equal(z["both_strands"], (z["forward"] + z["reverse"]) * np.float32(0.5))
    assert np.array_equal(e_on["embeddings_reverse"], er["embeddings"])
    assert np.array_equal(e_on["embeddings_reverse"], np.load(o_rc_plain.nn_classification_embeddings_output)["embeddings"])
    assert np.array_equal(e_on["embeddings_both_strands"], er["embeddings_both_strands"])
    assert not np.array_equal(z["forward"], z["reverse"])
    # the TSV: nine scores with the digits of f"{x:.4f}"
    lines = o.nn_classification_strands_output.read_text().split("\n")
    assert lines[0].split("\t") == ["seq_name"] + [f"{c}_score_{s}" for s in nn_classification.STRANDS
                                                   for c in ("chromosome", "plasmid", "virus")]
    assert lines[-1] == "" and len(lines) == len(z["contig_names"]) + 2
    for i, name in enumerate(z["contig_names"]):
        vals = np.concatenate([z[k][i] for k in nn_classification.STRANDS])
        assert lines[1 + i] == name + "".join(f"\t{float(v):.4f}" for v in vals)
    log = o.nn_classification_log.read_text()
    assert "sample_nn_classification_strands.tsv" in log and "_strands" not in o_off.nn_classification_log.read_text()


def test_flag_off_changes_no_file(tmp_path, stub, monkeypatch):
    fa = _module_fasta(tmp_path / "sample.fna")
    _run(fa, tmp_path / "a", write_embeddings=True)
    _run(fa, tmp_path / "b", write_embeddings=True, both_strands=False)
    monkeypatch.setenv("GENOMAD_B200_BOTH_STRANDS", "0")
    _run(fa, tmp_path / "c", write_embeddings=True)
    fa_ = _all_files(tmp_path / "a")
    assert fa_ == _all_files(tmp_path / "b") == _all_files(tmp_path / "c")
    for rel in ("sample_nn_classification/sample_nn_classification.npz",
                "sample_nn_classification/sample_nn_classification_embeddings.npz"):
        assert _npz(tmp_path / "a" / rel) == _npz(tmp_path / "b" / rel) == _npz(tmp_path / "c" / rel)
    names = {p.name for p in (tmp_path / "a").rglob("*")}
    assert not any("strands" in n for n in names)


def test_restart_skip_and_cleanup(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    out = tmp_path / "out"
    o = _run(fa, out, both_strands=True)
    n1 = len(stub.windows_seen())
    before = _npz(o.nn_classification_strands_npz_output)
    _run(fa, out, both_strands=True)                                       # everything found: skipped
    assert len(stub.windows_seen()) == n1
    o.nn_classification_strands_output.unlink()                            # a strand file missing: classified again
    _run(fa, out, both_strands=True)
    assert len(stub.windows_seen()) == 2 * n1 and _npz(o.nn_classification_strands_npz_output) == before
    _run(fa, out, both_strands=True, write_embeddings=True)                # embeddings file missing: again
    n2 = len(stub.windows_seen())
    assert n2 == 3 * n1
    e = np.load(o.nn_classification_embeddings_output)
    np.savez(o.nn_classification_embeddings_output, contig_names=e["contig_names"], embeddings=e["embeddings"])
    _run(fa, out, both_strands=True, write_embeddings=True)                # embeddings file without the keys: again
    assert len(stub.windows_seen()) == 4 * n1
    assert "embeddings_both_strands" in np.load(o.nn_classification_embeddings_output).files
    _run(fa, out, both_strands=True, write_embeddings=True, cleanup=True)  # --cleanup keeps the files
    assert len(stub.windows_seen()) == 4 * n1
    assert o.nn_classification_strands_npz_output.exists() and o.nn_classification_strands_output.exists()
    assert not o.encoded_sequences_dir.exists()
    _run(fa, out)                                                          # flag off: nothing redone, files left alone
    assert len(stub.windows_seen()) == 4 * n1 and o.nn_classification_strands_npz_output.exists()
    _run(fa, out, both_strands=True, restart=True)                         # --restart
    assert len(stub.windows_seen()) == 5 * n1 and _npz(o.nn_classification_strands_npz_output) == before


def test_reverse_pass_sees_the_reverse_windows(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    _run(fa, tmp_path / "on", both_strands=True)
    seen = stub.windows_seen()
    pf = sequence.ParsedFasta(fa)
    n = pf.n_windows
    wl = pf.windows(6000, reverse=True)
    try:
        exp = wl.export_windows(0, wl.n_windows, np.empty((wl.n_windows, 6000), np.uint8))
    finally:
        wl.close()
        pf.close()
    assert len(seen) == n + len(exp) and np.array_equal(seen[n:], exp)


def test_provirus_twin(tmp_path, stub, golden_dir):
    inp = golden_dir / "reference_module" / "input"
    out = tmp_path / "out"
    shutil.copytree(inp / "toy_find_proviruses", out / "toy_find_proviruses")
    nn_classification.main(inp / "toy.fna", out, False, 128, False, 2, False, False, both_strands=True)
    o = _paths.NNOutputs("toy", out)
    zp = np.load(o.provirus_nn_classification_strands_npz_output)
    assert set(zp.files) == {"provirus_names", "forward", "reverse", "both_strands"}
    assert zp["forward"].tobytes() == np.load(o.provirus_nn_classification_npz_output)["predictions"].tobytes()
    assert o.provirus_nn_classification_strands_output.read_text().startswith("seq_name\tchromosome_score_forward\t")
    assert o.nn_classification_strands_npz_output.exists()


def test_environment_variable_and_cli(tmp_path, stub, monkeypatch):
    fa = _module_fasta(tmp_path / "sample.fna")
    monkeypatch.setenv("GENOMAD_B200_BOTH_STRANDS", "1")
    o = _run(fa, tmp_path / "env")
    assert o.nn_classification_strands_npz_output.exists() and o.nn_classification_strands_output.exists()
    monkeypatch.delenv("GENOMAD_B200_BOTH_STRANDS")
    from click.testing import CliRunner
    from genomad_b200 import cli, embedding_clusters, embedding_neighbours
    seen = {}
    monkeypatch.setattr(nn_classification, "main", lambda *a, **k: seen.update(k))
    r = CliRunner().invoke(cli.cli, ["nn-classification", "--both-strands", str(fa), str(tmp_path / "o")])
    assert r.exit_code == 0, r.output
    assert seen == {"write_embeddings": None, "both_strands": True}
    seen.clear()
    r = CliRunner().invoke(cli.cli, ["nn-classification", str(fa), str(tmp_path / "o")])
    assert r.exit_code == 0 and seen == {"write_embeddings": None}
    emb = tmp_path / "x_nn_classification_embeddings.npz"
    np.savez(emb, contig_names=np.array(["a"]), embeddings=np.ones((1, EMBED), np.float32))
    for mod, args in ((embedding_neighbours, ["embedding-neighbours", "--both-strands", str(emb), str(tmp_path / "n")]),
                      (embedding_clusters, ["embedding-clusters", "--both-strands", "--min-similarity", "0.9", str(emb),
                                            str(tmp_path / "c")])):
        got = {}
        monkeypatch.setattr(mod, "main", lambda *a, **k: got.update(k))
        r = CliRunner().invoke(cli.cli, args)
        assert r.exit_code == 0, r.output
        assert got == {"both_strands": True}


# ------------------------------------------------------------------------------------------ embedding tools' input key
def test_embedding_tools_read_the_both_strands_key(tmp_path):
    from genomad_b200 import embedding_neighbours as EN
    names = np.array(["a", "b"])
    fwd = np.ones((2, EMBED), np.float32)
    both = np.full((2, EMBED), 2.0, np.float32)
    p = tmp_path / "s_nn_classification_embeddings.npz"
    np.savez(p, contig_names=names, embeddings=fwd, embeddings_reverse=fwd, embeddings_both_strands=both)
    assert np.array_equal(EN.read_embeddings(p)[1], fwd)
    assert np.array_equal(EN.read_embeddings(p, EN.BOTH_STRANDS_KEY)[1], both)
    q = tmp_path / "t_nn_classification_embeddings.npz"
    np.savez(q, contig_names=names, embeddings=fwd)
    with pytest.raises(EN.EmbeddingsFileError, match="--both-strands"):
        EN.read_embeddings(q, EN.BOTH_STRANDS_KEY)
    from genomad_b200 import embedding_clusters as EC
    for call in (lambda: EN.main(q, None, tmp_path / "o", 1, False, both_strands=True),
                 lambda: EN.main(p, q, tmp_path / "o", 1, False, both_strands=True),
                 lambda: EC.main(q, tmp_path / "o", 0.9, False, both_strands=True)):
        with pytest.raises(EN.EmbeddingsFileError, match="--write-embeddings --both-strands"):
            call()
