"""
CPU tests of the head's strand and window files (`nn-classification --head` with `--both-strands` / `--write-window-scores`)
with stub classifiers (tests/window_stub.py, tests/head_stub.py) behind the real module code: keys, dtypes, shapes and TSV
headers, the values the stubs give for the reverse list and the profile windows, `forward` bitwise the head file, the
windows bitwise those of the window-score file, the provirus twin, the restart rules, the empty-input branch, and every other
file byte-identical to a run without the pairing.  Also the n-column window table writer against Python's formatting.
"""
import ctypes as C
import hashlib
import shutil

import numpy as np
import pytest

import head_stub as HS
import window_stub as WS
from genomad_b200 import _paths, engine, nn_classification, sequence
from test_strands_cpu import EmbedStub, _all_files, _npz, stub_emb
from test_window_scores_cpu import _module_fasta, _run

CLASSES = ("alpha", "beta", "gamma.1", "d-4")


@pytest.fixture
def stub(monkeypatch):
    clf = EmbedStub()
    WS.install(monkeypatch.setattr, nn_classification, clf)
    monkeypatch.setattr(nn_classification, "_make_head", HS.StubHead)
    for k in ("GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS", "GENOMAD_B200_ATTRIBUTIONS",
              "GENOMAD_B200_BOTH_STRANDS", "GENOMAD_B200_HEAD_ATTRIBUTIONS", "RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    return clf


@pytest.fixture
def head(tmp_path):
    return HS.write_head(tmp_path / "h.npz", len(CLASSES), 1, names=CLASSES)


def _sha(p):
    return hashlib.sha256(p.read_bytes()).hexdigest()


def _list_windows(wl):
    return wl.export_windows(0, wl.n_windows, np.empty((wl.n_windows, 6000), np.uint8))


def _reverse_expected(fa, single_window=False):
    """The stub head's per-contig running means over the reverse list's windows."""
    pf = sequence.ParsedFasta(fa, single_window)
    wl = pf.windows(6000, single_window, reverse=True)
    try:
        offsets = wl.spans()[0]
        win = _list_windows(wl)
    finally:
        wl.close()
        pf.close()
    return WS.running_mean(HS.stub_head_probs(stub_emb(win), len(CLASSES)), offsets)


def _check_strands_tsv(path, z, names_key="contig_names"):
    lines = path.read_text().split("\n")
    assert lines[0].split("\t") == ["seq_name"] + [f"{c}_score_{s}" for s in nn_classification.STRANDS for c in CLASSES]
    assert lines[-1] == "" and len(lines) == len(z[names_key]) + 2
    for i, name in enumerate(z[names_key]):
        vals = np.concatenate([z[k][i] for k in nn_classification.STRANDS])
        assert lines[1 + i] == name + "".join(f"\t{float(v):.4f}" for v in vals)


@pytest.mark.parametrize("single_window", [False, True])
def test_head_strands_file(tmp_path, stub, head, single_window):
    fa = _module_fasta(tmp_path / "sample.fna")
    o = _run(fa, tmp_path / "out", head=head, both_strands=True, single_window=single_window)
    z = np.load(o.nn_classification_head_strands_npz_output)
    assert set(z.files) == {"contig_names", "forward", "reverse", "both_strands", "class_names", "head_sha256"}
    n = len(z["contig_names"])
    assert all(z[k].dtype == np.float32 and z[k].shape == (n, len(CLASSES)) for k in nn_classification.STRANDS)
    assert list(z["class_names"]) == list(CLASSES) and str(z["head_sha256"]) == _sha(head)
    zh = np.load(o.nn_classification_head_npz_output)
    assert list(z["contig_names"]) == list(zh["contig_names"])
    assert z["forward"].tobytes() == zh["predictions"].tobytes()
    assert np.array_equal(z["reverse"], _reverse_expected(fa, single_window))
    assert z["both_strands"].tobytes() == ((z["forward"] + z["reverse"]) * np.float32(0.5)).tobytes()
    assert not np.array_equal(z["forward"], z["reverse"])
    _check_strands_tsv(o.nn_classification_head_strands_output, z)
    assert "sample_nn_classification_head_strands.tsv" in o.nn_classification_log.read_text()


def _check_windows_tsv(path, z, names_key="contig_names"):
    lines = path.read_text().split("\n")
    assert lines[0] == "seq_name\tstart\tend\t" + "\t".join(f"{c}_score" for c in CLASSES) and lines[-1] == ""
    assert len(lines) == len(z["predictions"]) + 2
    names = z[names_key]
    for i, (c, s, n, p) in enumerate(zip(z["window_contig"], z["window_start"], z["window_length"], z["predictions"])):
        assert lines[1 + i] == f"{names[c]}\t{s + 1}\t{s + n}" + "".join(f"\t{float(x):.4f}" for x in p)


@pytest.mark.parametrize("stride,single_window", [(6000, False), (1000, False), (6000, True)])
def test_head_windows_file(tmp_path, stub, head, stride, single_window):
    fa = _module_fasta(tmp_path / "sample.fna")
    o = _run(fa, tmp_path / "out", head=head, write_window_scores=True, window_stride=stride, single_window=single_window)
    z = np.load(o.nn_classification_head_windows_npz_output)
    zw = np.load(o.nn_classification_windows_npz_output)
    assert set(z.files) == set(zw.files) | {"class_names", "head_sha256"}
    for k in ("contig_names", "window_contig", "window_start", "window_length", "window_stride"):
        assert z[k].dtype == zw[k].dtype and z[k].shape == zw[k].shape and np.array_equal(z[k], zw[k]), k
    assert z["predictions"].dtype == np.float32 and z["predictions"].shape == (len(zw["predictions"]), len(CLASSES))
    assert list(z["class_names"]) == list(CLASSES) and str(z["head_sha256"]) == _sha(head)
    # the rows are the stub head's scores of the stub's embeddings of the profile's own windows
    pf = sequence.ParsedFasta(fa, single_window)
    try:
        if stride == 6000 and not single_window:
            win, offsets = pf.export_windows(0, pf.n_windows, np.empty((pf.n_windows, 6000), np.uint8)), pf.index().offsets
        else:
            wl = pf.windows(stride)
            try:
                win, offsets = _list_windows(wl), wl.spans()[0]
            finally:
                wl.close()
    finally:
        pf.close()
    assert np.array_equal(z["predictions"], HS.stub_head_probs(stub_emb(win), len(CLASSES)))
    assert np.array_equal(zw["predictions"], WS.stub_probs(win))
    if stride == 6000 and not single_window:         # the contig pass's own rows: the head file is their per-contig mean
        assert np.array_equal(WS.running_mean(z["predictions"], offsets),
                              np.load(o.nn_classification_head_npz_output)["predictions"])
        assert len(stub.windows_seen()) == len(win)   # no second pass
    _check_windows_tsv(o.nn_classification_head_windows_output, z)
    assert "sample_nn_classification_head_windows.tsv" in o.nn_classification_log.read_text()


def test_provirus_twins(tmp_path, stub, head, golden_dir):
    inp = golden_dir / "reference_module" / "input"
    out = tmp_path / "out"
    shutil.copytree(inp / "toy_find_proviruses", out / "toy_find_proviruses")
    nn_classification.main(inp / "toy.fna", out, False, 128, False, 2, False, False, both_strands=True, head=head,
                           write_window_scores=True, window_stride=1000)
    o = _paths.NNOutputs("toy", out)
    zp = np.load(o.provirus_nn_classification_head_strands_npz_output)
    assert set(zp.files) == {"provirus_names", "forward", "reverse", "both_strands", "class_names", "head_sha256"}
    assert zp["forward"].tobytes() == np.load(o.provirus_nn_classification_head_npz_output)["predictions"].tobytes()
    _check_strands_tsv(o.provirus_nn_classification_head_strands_output, zp, "provirus_names")
    zw = np.load(o.provirus_nn_classification_head_windows_npz_output)
    zs = np.load(o.provirus_nn_classification_windows_npz_output)
    assert "provirus_names" in zw.files and len(zw["predictions"]) == len(zs["predictions"]) > 0
    assert all(np.array_equal(zw[k], zs[k]) for k in ("provirus_names", "window_contig", "window_start", "window_length"))
    _check_windows_tsv(o.provirus_nn_classification_head_windows_output, zw, "provirus_names")
    assert o.nn_classification_head_strands_npz_output.exists() and o.nn_classification_head_windows_npz_output.exists()


def test_empty_provirus_input_writes_zero_rows(tmp_path, stub, head, golden_dir):
    inp = golden_dir / "reference_module" / "input"
    out = tmp_path / "out"
    shutil.copytree(inp / "toy_find_proviruses", out / "toy_find_proviruses")
    (out / "toy_find_proviruses" / "toy_provirus.fna").write_text(">p1|provirus_1_500\n" + "N" * 500 + "\n")
    nn_classification.main(inp / "toy.fna", out, False, 128, False, 2, False, False, both_strands=True, head=head,
                           write_window_scores=True)
    o = _paths.NNOutputs("toy", out)
    zp = np.load(o.provirus_nn_classification_head_strands_npz_output)
    assert all(zp[k].shape == (len(zp["provirus_names"]), len(CLASSES)) and not zp[k].any()
               for k in nn_classification.STRANDS)
    zw = np.load(o.provirus_nn_classification_head_windows_npz_output)
    assert zw["predictions"].shape == (0, len(CLASSES)) and zw["predictions"].dtype == np.float32
    assert zw["window_start"].shape == (0,) and int(zw["window_stride"]) == 6000
    assert o.provirus_nn_classification_head_windows_output.read_text() == \
        "seq_name\tstart\tend\t" + "\t".join(f"{c}_score" for c in CLASSES) + "\n"


def test_restart_rules(tmp_path, stub, head):
    fa = _module_fasta(tmp_path / "sample.fna")
    other = HS.write_head(tmp_path / "other.npz", 3, 7)
    out = tmp_path / "out"
    kw = dict(both_strands=True, write_window_scores=True, window_stride=1000)
    o = _run(fa, out, head=head, **kw)
    n1 = len(stub.windows_seen())
    before = {p: _npz(p) for p in (o.nn_classification_head_strands_npz_output, o.nn_classification_head_windows_npz_output)}
    _run(fa, out, head=head, **kw)                                             # everything found: skipped
    assert len(stub.windows_seen()) == n1
    for p in (o.nn_classification_head_strands_output, o.nn_classification_head_strands_npz_output,
              o.nn_classification_head_windows_output, o.nn_classification_head_windows_npz_output):
        p.unlink()                                                             # one file missing: classified again
        _run(fa, out, head=head, **kw)
        n2 = len(stub.windows_seen())
        assert n2 > n1 and p.exists()
        n1 = n2
    assert all(_npz(p) == b for p, b in before.items())
    # a head strands / head windows file of another head: classified again
    for p in (o.nn_classification_head_strands_npz_output, o.nn_classification_head_windows_npz_output):
        z = dict(np.load(p))
        z["head_sha256"] = np.str_(_sha(other))
        np.savez(p, **z)
        _run(fa, out, head=head, **kw)
        n2 = len(stub.windows_seen())
        assert n2 > n1 and str(np.load(p)["head_sha256"]) == _sha(head)
        n1 = n2
    z = dict(np.load(o.nn_classification_head_windows_npz_output))             # written at another stride: again
    z["window_stride"] = np.int32(2000)
    np.savez(o.nn_classification_head_windows_npz_output, **z)
    _run(fa, out, head=head, **kw)
    assert len(stub.windows_seen()) > n1 and _npz(o.nn_classification_head_windows_npz_output) == \
        before[o.nn_classification_head_windows_npz_output]
    n1 = len(stub.windows_seen())
    _run(fa, out, head=head, **kw, cleanup=True)                               # --cleanup leaves them alone
    assert len(stub.windows_seen()) == n1 and all(p.exists() for p in before)
    _run(fa, out, head=other, **kw)                                            # another head: again, all four replaced
    assert len(stub.windows_seen()) > n1
    assert all(str(np.load(p)["head_sha256"]) == _sha(other) and np.load(p)["class_names"].shape == (3,) for p in before)


def _same_files(a, b):
    """Every file of run a is in run b with the same bytes (NPZ: the same arrays; a zip member's date is not a result)."""
    fa_, fb = _all_files(a), _all_files(b)
    assert all(fb.get(k) == v for k, v in fa_.items()), [k for k, v in fa_.items() if fb.get(k) != v]
    for p in a.rglob("*.npz"):
        assert _npz(p) == _npz(b / p.relative_to(a)), p.name


@pytest.mark.parametrize("single_window", [False, True])
def test_other_files_unchanged_by_the_pairings(tmp_path, stub, head, single_window):
    fa = _module_fasta(tmp_path / "sample.fna")
    sw = dict(single_window=single_window)
    runs = {name: tmp_path / name for name in ("head", "strands", "head_strands", "windows", "head_windows", "all")}
    _run(fa, runs["head"], head=head, **sw)
    _run(fa, runs["strands"], both_strands=True, write_embeddings=True, **sw)
    _run(fa, runs["head_strands"], head=head, both_strands=True, write_embeddings=True, **sw)
    _run(fa, runs["windows"], write_window_scores=True, window_stride=1000, **sw)
    _run(fa, runs["head_windows"], head=head, write_window_scores=True, window_stride=1000, **sw)
    _run(fa, runs["all"], head=head, both_strands=True, write_window_scores=True, **sw)
    _same_files(runs["head"], runs["head_strands"])
    _same_files(runs["strands"], runs["head_strands"])
    _same_files(runs["head"], runs["head_windows"])
    _same_files(runs["windows"], runs["head_windows"])
    _same_files(runs["head"], runs["all"])
    new = {p.name for p in runs["head_strands"].rglob("*")} - {p.name for p in runs["head"].rglob("*")} \
        - {p.name for p in runs["strands"].rglob("*")}
    assert new == {"sample_nn_classification_head_strands.tsv", "sample_nn_classification_head_strands.npz"}
    new = {p.name for p in runs["head_windows"].rglob("*")} - {p.name for p in runs["head"].rglob("*")} \
        - {p.name for p in runs["windows"].rglob("*")}
    assert new == {"sample_nn_classification_head_windows.tsv", "sample_nn_classification_head_windows.npz"}
    assert not any("head_" in p.name for p in runs["head"].rglob("*") if p.suffix in (".tsv", ".npz"))


# ------------------------------------------------------------------------------------------ the n-column table writer
@pytest.fixture(scope="module")
def lib():
    return engine.load_library()


def _table(rng, n_cols):
    names = ["a", "contig_2|provirus_1_9000", "x" * 300, "empty", "z"]
    counts = [3, 70000, 2, 0, 1]                                                  # more rows than one formatting block
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    n = int(offsets[-1])
    starts = rng.integers(0, 10 ** 9, n).astype(np.int64)
    lengths = rng.integers(1, 6001, n).astype(np.int32)
    probs = rng.random((n, n_cols), dtype=np.float32)
    probs[:50] = np.float32(rng.standard_normal((50, n_cols)) * 1e6)              # long scores too
    return names, offsets, starts, lengths, probs


def _write_cols(lib, path, header, names, offsets, starts, lengths, probs, threads):
    blobs = [x.encode() for x in names]
    name_off = np.zeros(len(blobs) + 1, np.int64)
    np.cumsum([len(b) for b in blobs], out=name_off[1:])
    probs = np.ascontiguousarray(probs, np.float32)
    return lib.gnm_write_window_tsv_cols(str(path).encode(), header.encode(), b"".join(blobs), name_off.ctypes.data,
                                         len(blobs), offsets.ctypes.data, starts.ctypes.data, lengths.ctypes.data,
                                         probs.ctypes.data, probs.shape[1], threads)


def test_three_columns_are_the_window_score_writer(tmp_path, lib):
    names, offsets, starts, lengths, probs = _table(np.random.default_rng(4), 3)
    header = nn_classification._WINDOW_HEADER
    nn_classification._write_window_tsv(tmp_path / "a.tsv", names, offsets, starts, lengths, probs, threads=3)
    assert _write_cols(lib, tmp_path / "b.tsv", header, names, offsets, starts, lengths, probs, 3) == 0
    assert (tmp_path / "a.tsv").read_bytes() == (tmp_path / "b.tsv").read_bytes()


@pytest.mark.parametrize("n_cols", [1, 7, 32])
def test_n_columns_match_python(tmp_path, lib, n_cols):
    rng = np.random.default_rng(n_cols)
    names, offsets, starts, lengths, probs = _table(rng, n_cols)
    header = "seq_name\tstart\tend\t" + "\t".join(f"k{i}_score" for i in range(n_cols)) + "\n"
    nn_classification._write_window_tsv(tmp_path / "w.tsv", names, offsets, starts, lengths, probs, threads=2,
                                        header=header, n_cols=n_cols)
    lines = (tmp_path / "w.tsv").read_text().split("\n")
    assert lines[0] + "\n" == header and lines[-1] == "" and len(lines) == len(starts) + 2
    cid = np.repeat(np.arange(len(names)), np.diff(offsets))
    for i in list(range(0, 60)) + list(range(len(starts) - 20, len(starts))) + rng.integers(0, len(starts), 1000).tolist():
        assert lines[1 + i] == (f"{names[cid[i]]}\t{starts[i] + 1}\t{starts[i] + lengths[i]}"
                                + "".join(f"\t{float(x):.4f}" for x in probs[i]))


def test_n_columns_out_of_range_are_refused(tmp_path, lib):
    names, offsets, starts, lengths, probs = ["a"], np.array([0, 1], np.int32), np.zeros(1, np.int64), \
        np.ones(1, np.int32), np.zeros((1, 33), np.float32)
    assert _write_cols(lib, tmp_path / "w.tsv", "h\n", names, offsets, starts, lengths, probs, 1) != 0
    assert b"n_cols" in lib.gnm_tsv_last_error()
    assert _write_cols(lib, tmp_path / "w.tsv", "h\n", names, offsets, starts, lengths, probs[:, :0], 1) != 0
    assert not (tmp_path / "w.tsv").exists()
