"""
CPU tests of the per-window score export (`--write-window-scores`, `--window-stride`): the native FASTA window lists at any
stride against their pure-Python statement (sequence.profile_spans), the stride-6000 list against the reference's window list,
the score-table writer against Python's f-string formatting, and the module's outputs, restart rules and bytes handed to the
classifier (stubbed).
"""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from genomad_b200 import _paths, engine, nn_classification, sequence
import window_stub as WS

STRIDES = [1, 7, 8, 999, 1000, 2500, 5999, 6000]


# ------------------------------------------------------------------------------------------ pure-Python statement
def expected_windows(path, stride, single_window=False):
    """Per kept record, from the record's joined lines: [(record index, start in the unstripped sequence, length, 6000 bytes)]."""
    out, names = [], []
    for header, raw in sequence.iter_fasta(path, strip_n=False):
        seq = raw.strip(b"nN")
        if not seq:
            continue
        lead = len(raw) - len(raw.lstrip(b"nN"))
        spans = sequence.profile_spans(len(seq), stride)
        if single_window:
            spans = spans[:1]
        for k, (s, e) in enumerate(spans):
            if k > 0 and seq[s:e].count(b"N") > sequence.MAX_N:
                continue
            out.append((len(names), lead + s, e - s, seq[s:e].upper().ljust(sequence.WINDOW, b"N")))
        names.append(sequence.accession(header))
    return names, out


@pytest.mark.parametrize("length", list(range(0, 2600, 97)) + [2499, 2500, 2501, 5999, 6000, 6001, 8499, 8500, 8501,
                                                                12000, 14500, 14501, 60000, 123457])
def test_profile_spans_at_6000_are_the_reference_windows(length):
    assert sequence.profile_spans(length, 6000) == sequence.window_spans(length)


@pytest.mark.parametrize("stride", STRIDES)
@pytest.mark.parametrize("length", [1, 2499, 2500, 2501, 5999, 6000, 6001, 9000, 17777])
def test_profile_spans_count_is_closed_form(stride, length):
    spans = sequence.profile_spans(length, stride)
    assert len(spans) == 1 + max(0, (length - 2500) // stride)
    assert all(s == k * stride and e == min(s + 6000, length) for k, (s, e) in enumerate(spans))
    assert all(e - s >= 2500 for s, e in spans[1:])


def test_profile_spans_rejects_bad_stride():
    for s in (0, -1, 6001):
        with pytest.raises(ValueError):
            sequence.profile_spans(100, s)


# ------------------------------------------------------------------------------------------ seeded FASTA with the edge cases
def _rand(rng, n, alphabet=b"ACGTacgt"):
    return np.frombuffer(alphabet, np.uint8)[rng.integers(0, len(alphabet), n)].tobytes()


def write_edge_fasta(path, stride, seed=0):
    rng = np.random.default_rng(seed)
    recs = []
    for k in (1, 2, 3):                                   # lengths k*s - 1, k*s, k*s + 1 plus 2500
        for d in (-1, 0, 1):
            recs.append(_rand(rng, k * stride + 2500 + d))
    recs.append(_rand(rng, 1800))                         # shorter than 2500
    recs.append(_rand(rng, 4700))                         # shorter than 6000
    nrun = bytearray(_rand(rng, 13000))                   # an N run that the N rule drops, and lower-case n that it ignores
    nrun[5000:9700] = b"N" * 4700
    nrun[1000:5500] = b"n" * 4500
    nrun[11000:11500] = b"N" * 500
    recs.append(b"nNnN" + bytes(nrun) + b"NNnn")          # leading and trailing n/N are stripped
    recs.append(b"N" * 7000)                              # all N: dropped
    recs.append(b"")                                      # empty: dropped
    recs.append(b"NNN" + _rand(rng, 2600) + b"n")
    with open(path, "wb") as fh:
        fh.write(b"; text before the first record is ignored\n")
        for i, r in enumerate(recs):
            if i % 4 == 1:                                # CRLF, 70 per line
                fh.write(f">r{i} crlf\r\n".encode() + b"\r\n".join(r[k:k + 70] for k in range(0, len(r), 70)) + b"\r\n")
            elif i % 4 == 2:                              # irregular line lengths
                cuts, k = [], 0
                while k < len(r):
                    step = int(rng.integers(1, 150))
                    cuts.append(r[k:k + step])
                    k += step
                fh.write(f">r{i} irregular\n".encode() + b"\n".join(cuts) + b"\n")
            else:
                fh.write(f">r{i}\n".encode() + b"\n".join(r[k:k + 61] for k in range(0, len(r), 61)) + b"\n")
    return path


@pytest.fixture(scope="module")
def lib():
    return engine.load_library()


@pytest.mark.parametrize("stride", STRIDES)
def test_native_window_list_matches_profile_spans(tmp_path, lib, stride):
    fa = write_edge_fasta(tmp_path / "edge.fna", stride, seed=stride)
    names, exp = expected_windows(fa, stride)
    pf = sequence.ParsedFasta(fa, threads=4)
    wl = pf.windows(stride)
    try:
        assert wl.n_contigs == pf.n_contigs == len(names) and wl.n_windows == len(exp)
        offsets, starts, lengths = wl.spans()
        cid = np.array([e[0] for e in exp], np.int64)
        assert np.array_equal(offsets, np.concatenate([[0], np.cumsum(np.bincount(cid, minlength=len(names)))]))
        assert np.array_equal(starts, np.array([e[1] for e in exp], np.int64))
        assert np.array_equal(lengths, np.array([e[2] for e in exp], np.int32))
        if stride < 6000:
            assert wl.n_windows > pf.n_windows                                # overlapping windows
        buf = np.empty((min(512, len(exp)), 6000), np.uint8)
        for a in range(0, len(exp), 512):                                     # any block, on 4 threads
            got = wl.export_windows(a, min(512, len(exp) - a), buf)
            want = np.frombuffer(b"".join(e[3] for e in exp[a:a + 512]), np.uint8).reshape(-1, 6000)
            assert np.array_equal(got, want)
        wl.release_before(wl.n_windows // 2)                                  # mmap: pages behind the cursor go back
        got = wl.export_windows(len(exp) - 1, 1, buf)
        assert np.array_equal(got[0], np.frombuffer(exp[-1][3], np.uint8))
    finally:
        wl.close()
        pf.close()


def _mapping_rss_kb(path) -> int:
    """Resident kB of this process' mappings of `path` (/proc/self/smaps)."""
    import re
    rss, hit = 0, False
    with open("/proc/self/smaps") as fh:
        for line in fh:
            if re.match(r"^[0-9a-f]+-[0-9a-f]+ ", line):
                hit = line.rstrip().endswith(str(path))
            elif hit and line.startswith("Rss:"):
                rss += int(line.split()[1])
    return rss


def _stream(src, chunk):
    """The module's chunk loop (nn_classification._classify_parsed): export chunk i, release what lies before chunk i - 1."""
    buf = np.empty((chunk, 6000), np.uint8)
    for i, a in enumerate(range(0, src.n_windows, chunk)):
        if i >= 2:
            src.release_before(a - chunk)
        src.export_windows(a, min(chunk, src.n_windows - a), buf)


@pytest.mark.skipif(not os.path.exists("/proc/self/smaps"), reason="needs /proc/self/smaps")
def test_each_window_list_releases_the_pages_behind_its_cursor(tmp_path):
    """A profile pass re-reads the file after the contig pass has released it: its own list must release the pages again,
    so the resident part of the mapping stays a few chunks, not the file."""
    rng = np.random.default_rng(21)
    fa = tmp_path / "big.fna"
    with open(fa, "wb") as fh:
        for i in range(400):                                                  # 400 records of 100 kb: 40 MB
            r = _rand(rng, 100_000, b"ACGT")
            fh.write(f">r{i}\n".encode() + b"\n".join(r[k:k + 80] for k in range(0, len(r), 80)) + b"\n")
    size_kb = fa.stat().st_size // 1024
    pf = sequence.ParsedFasta(fa, threads=4)
    wl = None
    try:
        _stream(pf, 512)                                                      # contig pass: 3 MB chunks
        assert _mapping_rss_kb(fa) < size_kb // 3
        wl = pf.windows(1000)
        _stream(wl, 512)                                                      # profile pass: 0.5 MB chunks
        rss = _mapping_rss_kb(fa)
        assert rss < 8 * 1024, f"{rss} kB of the {size_kb} kB mapping resident after the profile pass"
    finally:
        if wl is not None:
            wl.close()
        pf.close()


@pytest.mark.parametrize("single_window", [False, True])
def test_stride_6000_list_is_the_reference_list(tmp_path, single_window):
    fa = write_edge_fasta(tmp_path / "edge.fna", 6000, seed=3)
    pf = sequence.ParsedFasta(fa, single_window=single_window, threads=3)
    wl = pf.windows(6000, single_window=single_window)
    try:
        enc = pf.encode()
        offsets, starts, lengths = wl.spans()
        assert np.array_equal(offsets, enc.offsets)
        full = np.empty((wl.n_windows, 6000), np.uint8)
        assert np.array_equal(wl.export_windows(0, wl.n_windows, full), enc.windows)
        assert np.array_equal(enc.windows, sequence.encode_fasta_py(fa, single_window).windows)
        _names, exp = expected_windows(fa, 6000, single_window)
        assert np.array_equal(starts, [e[1] for e in exp]) and np.array_equal(lengths, [e[2] for e in exp])
    finally:
        wl.close()
        pf.close()


def test_window_list_from_caller_memory_and_bad_stride(tmp_path, lib):
    fa = write_edge_fasta(tmp_path / "edge.fna", 999, seed=9)
    text = fa.read_bytes()
    h = C.c_void_p()
    assert lib.gnm_fasta_parse(C.cast(C.c_char_p(text), C.c_void_p), len(text), 0, 2, C.byref(h)) == 0
    try:
        for bad in (0, 6001):
            w = C.c_void_p()
            assert lib.gnm_fasta_windows_plan(h, bad, 0, 2, C.byref(w)) != 0
            assert b"stride must be in [1, 6000]" in lib.gnm_fasta_last_error()
        w = C.c_void_p()
        assert lib.gnm_fasta_windows_plan(h, 999, 0, 2, C.byref(w)) == 0
        nc, nw = C.c_int64(), C.c_int64()
        lib.gnm_fasta_windows_info(w, C.byref(nc), C.byref(nw))
        _names, exp = expected_windows(fa, 999)
        assert nw.value == len(exp)
        buf = np.empty((nw.value, 6000), np.uint8)
        assert lib.gnm_fasta_windows_export(w, 0, nw.value, buf.ctypes.data, 2) == 0
        assert buf.tobytes() == b"".join(e[3] for e in exp)
        assert lib.gnm_fasta_windows_export(w, 1, nw.value, buf.ctypes.data, 2) != 0       # out of range
        lib.gnm_fasta_windows_free(w)
    finally:
        lib.gnm_fasta_free(h)


# ------------------------------------------------------------------------------------------ score formatting
def _format_native(lib, x):
    x = np.ascontiguousarray(x, np.float32)
    out = C.create_string_buffer(50 * max(1, len(x)))
    n = C.c_int64()
    assert lib.gnm_format_scores(x.ctypes.data, len(x), out, C.byref(n)) == 0
    return out.raw[: n.value].decode().split("\n")[:-1]


def test_score_format_matches_python_fstring(lib):
    rng = np.random.default_rng(11)
    x = np.concatenate([
        rng.random(200000, dtype=np.float32),                                       # probabilities
        (np.arange(0, 20001) / 20000).astype(np.float32),                           # every x.xxxx5 neighbourhood
        np.nextafter((np.arange(1, 20001, 2) / 20000).astype(np.float32), np.float32(2)),
        np.nextafter((np.arange(1, 20001, 2) / 20000).astype(np.float32), np.float32(-1)),
        np.array([0.03125, 0.09375, 0.15625, 0.21875, 0.28125, 0.0, -0.0, 1.0, 0.99995, 0.99994999, 1e-30, 1e-45, -1e-7,
                  -0.5, 3.5, 1234.56789, -42.00005, 2.0 ** 24, -2.0 ** 30, 3e38, np.inf, -np.inf, np.nan, -np.nan],
                 np.float32),
        rng.standard_normal(20000).astype(np.float32) * 1000,
    ])
    got = _format_native(lib, x)
    want = [f"{float(v):.4f}" for v in x]
    bad = [(float(v), g, w) for v, g, w in zip(x, got, want) if g != w]
    assert not bad, bad[:10]
    assert _format_native(lib, [0.03125, 0.09375]) == ["0.0312", "0.0938"]          # exact ties go to even, as in Python


def test_window_tsv_writer_longest_rows(tmp_path, lib):
    """The public writer takes any float: rows of long names, 19-digit coordinates and 45-character scores."""
    n = 5000
    names = ["n" * 1000, "m"]
    offsets = np.array([0, n - 1, n], np.int32)
    starts = np.full(n, 2 ** 62, np.int64)
    lengths = np.full(n, 6000, np.int32)
    probs = np.tile(np.array([[-3.4e38, 3.4e38, -1.5e38]], np.float32), (n, 1))
    path = tmp_path / "w.tsv"
    nn_classification._write_window_tsv(path, names, offsets, starts, lengths, probs, threads=2)
    lines = path.read_text().split("\n")
    assert len(lines) == n + 2
    for i in (0, n - 2, n - 1):
        p = probs[i]
        assert lines[1 + i] == (f"{names[0 if i < n - 1 else 1]}\t{2 ** 62 + 1}\t{2 ** 62 + 6000}"
                                f"\t{float(p[0]):.4f}\t{float(p[1]):.4f}\t{float(p[2]):.4f}")


def test_window_tsv_writer_matches_fstring_rows(tmp_path, lib):
    rng = np.random.default_rng(4)
    names = ["a", "contig_2|provirus_1_9000", "x" * 300, "empty", "z"]
    counts = [3, 70000, 2, 0, 1]                                                  # more rows than one formatting block
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    n = int(offsets[-1])
    starts = rng.integers(0, 10 ** 9, n).astype(np.int64)
    lengths = rng.integers(1, 6001, n).astype(np.int32)
    probs = rng.random((n, 3), dtype=np.float32)
    path = tmp_path / "w.tsv"
    nn_classification._write_window_tsv(path, names, offsets, starts, lengths, probs, threads=3)
    lines = path.read_text().split("\n")
    assert lines[0] == "seq_name\tstart\tend\tchromosome_score\tplasmid_score\tvirus_score" and lines[-1] == ""
    cid = np.repeat(np.arange(len(names)), counts)
    for i in list(range(0, 20)) + list(range(n - 20, n)) + rng.integers(0, n, 2000).tolist():
        p = probs[i]
        assert lines[1 + i] == (f"{names[cid[i]]}\t{starts[i] + 1}\t{starts[i] + lengths[i]}"
                                f"\t{float(p[0]):.4f}\t{float(p[1]):.4f}\t{float(p[2]):.4f}")
    assert len(lines) == n + 2


# ------------------------------------------------------------------------------------------ module (stubbed classifier)
@pytest.fixture
def stub(monkeypatch):
    clf = WS.StubClassifier()
    WS.install(monkeypatch.setattr, nn_classification, clf)
    monkeypatch.delenv("GENOMAD_B200_WINDOW_SCORES", raising=False)
    monkeypatch.delenv("GENOMAD_B200_EMBEDDINGS", raising=False)
    return clf


def _module_fasta(path):
    """Contigs of several windows, one that loses a window to the N rule, leading / trailing n/N, irregular lines."""
    rng = np.random.default_rng(7)
    recs = {"c0": _rand(rng, 20000), "c1": _rand(rng, 3000), "c2": b"nnNN" + _rand(rng, 14000) + b"NNN",
            "c3": _rand(rng, 6100), "c4": b"N" * 100}
    r = bytearray(_rand(rng, 19000))
    r[6500:11200] = b"N" * 4700
    recs["c5"] = bytes(r)
    with open(path, "wb") as fh:
        for i, (k, v) in enumerate(recs.items()):
            w = 60 if i % 2 else 77
            fh.write(f">{k} desc\n".encode() + b"\n".join(v[j:j + w] for j in range(0, len(v), w)) + b"\n")
    return path


def _run(fa, out, **kw):
    nn_classification.main(fa, out, kw.pop("single_window", False), 128, kw.pop("restart", False), 2, False,
                           kw.pop("cleanup", False), **kw)
    return _paths.NNOutputs("sample", out)


def _contig_outputs(o):
    """The contig table's bytes and the predictions NPZ's arrays (a zip member's timestamp is not part of the result)."""
    z = np.load(o.nn_classification_npz_output)
    return (o.nn_classification_output.read_bytes(), {k: (z[k].dtype.str, z[k].tobytes()) for k in z.files})


def _check_tsv_matches_npz(o):
    z = np.load(o.nn_classification_windows_npz_output)
    lines = o.nn_classification_windows_output.read_text().split("\n")
    assert lines[0] == "seq_name\tstart\tend\tchromosome_score\tplasmid_score\tvirus_score" and lines[-1] == ""
    assert len(lines) == len(z["predictions"]) + 2
    names = z["contig_names"]
    for i, (c, s, n, p) in enumerate(zip(z["window_contig"], z["window_start"], z["window_length"], z["predictions"])):
        assert lines[1 + i] == f"{names[c]}\t{s + 1}\t{s + n}\t{float(p[0]):.4f}\t{float(p[1]):.4f}\t{float(p[2]):.4f}"


def test_window_scores_at_6000_are_the_contig_pass(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    o_off = _run(fa, tmp_path / "off")
    n_contig_windows = len(stub.windows_seen())
    o_on = _run(fa, tmp_path / "on", write_window_scores=True)
    assert len(stub.windows_seen()) == 2 * n_contig_windows                 # no second classification
    assert _contig_outputs(o_off) == _contig_outputs(o_on)
    assert not o_off.nn_classification_windows_npz_output.exists() and not o_off.nn_classification_windows_output.exists()
    j_off, j_on = (json.loads(o.nn_classification_execution_info.read_text()) for o in (o_off, o_on))
    assert j_on["parameters"] == j_off["parameters"] == {"single_window": False}
    z = np.load(o_on.nn_classification_windows_npz_output)
    assert set(z.files) == {"contig_names", "window_contig", "window_start", "window_length", "predictions", "window_stride"}
    assert z["window_contig"].dtype == np.int32 and z["window_start"].dtype == np.int64
    assert z["window_length"].dtype == np.int32 and z["predictions"].dtype == np.float32
    assert z["predictions"].shape == (n_contig_windows, 3) and int(z["window_stride"]) == 6000
    preds = np.load(o_on.nn_classification_npz_output)
    assert list(z["contig_names"]) == list(preds["contig_names"])
    offsets = np.concatenate([[0], np.cumsum(np.bincount(z["window_contig"], minlength=len(z["contig_names"])))])
    # The stub reduces with the same fp32 running mean, so this shows that the NPZ holds exactly the rows the contig pass
    # reduced, in its order and grouping (an fp32 running sum changes bits when rows move); that gnm_segment_mean itself is
    # that running mean is tested on the GPU (test_gpu_window_scores.py).  The rows are also each window's own scores:
    assert np.array_equal(WS.running_mean(z["predictions"], offsets), preds["predictions"])      # bitwise
    assert np.array_equal(z["predictions"], WS.stub_probs(stub.windows_seen()[n_contig_windows:]))
    _check_tsv_matches_npz(o_on)
    assert "sample_nn_classification_windows.tsv" in o_on.nn_classification_log.read_text()
    assert "_windows" not in o_off.nn_classification_log.read_text()


@pytest.mark.parametrize("stride,single_window", [(1000, False), (999, False), (6000, True), (2500, True)])
def test_profile_windows_are_the_bytes_the_classifier_received(tmp_path, stub, stride, single_window):
    fa = _module_fasta(tmp_path / "sample.fna")
    o_ref = _run(fa, tmp_path / "ref", single_window=single_window)
    n_contig = len(stub.windows_seen())
    o = _run(fa, tmp_path / "on", single_window=single_window, write_window_scores=True, window_stride=stride)
    assert _contig_outputs(o_ref) == _contig_outputs(o)
    seen = stub.windows_seen()[2 * n_contig:]                             # the second pass, in window order
    z = np.load(o.nn_classification_windows_npz_output)
    assert int(z["window_stride"]) == stride and len(seen) == len(z["predictions"])
    raw = {sequence.accession(h): s for h, s in sequence.iter_fasta(fa, strip_n=False)}
    names, exp = expected_windows(fa, stride)                             # a profile covers every contig whole
    assert list(z["contig_names"]) == names and len(exp) == len(seen)
    for i, (c, s, n) in enumerate(zip(z["window_contig"], z["window_start"], z["window_length"])):
        got = raw[names[c]][s: s + n].upper().ljust(6000, b"N")           # TSV [start - 1, end) of the raw record
        assert got == seen[i].tobytes() == exp[i][3]
    assert np.array_equal(z["predictions"], WS.stub_probs(seen))
    _check_tsv_matches_npz(o)


def test_restart_rules(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    out = tmp_path / "out"
    o = _run(fa, out, write_window_scores=True, window_stride=1000)
    before, n1 = _contig_outputs(o), len(stub.windows_seen())
    win_before = tmp_path / "before.npz"
    win_before.write_bytes(o.nn_classification_windows_npz_output.read_bytes())
    _run(fa, out, write_window_scores=True, window_stride=1000)           # everything found: skipped
    assert len(stub.windows_seen()) == n1
    _run(fa, out, write_window_scores=True, window_stride=2000)           # another stride: classified again
    assert len(stub.windows_seen()) > n1 and _contig_outputs(o) == before
    assert int(np.load(o.nn_classification_windows_npz_output)["window_stride"]) == 2000
    n2 = len(stub.windows_seen())
    o.nn_classification_windows_npz_output.unlink()                      # missing windows file: classified again
    _run(fa, out, write_window_scores=True, window_stride=1000)
    assert len(stub.windows_seen()) > n2 and _contig_outputs(o) == before
    z, zb = np.load(o.nn_classification_windows_npz_output), np.load(win_before)
    assert all(np.array_equal(z[k], zb[k]) for k in zb.files)
    n3 = len(stub.windows_seen())
    _run(fa, out, write_window_scores=True, window_stride=1000, cleanup=True)     # --cleanup keeps the files
    assert len(stub.windows_seen()) == n3
    assert o.nn_classification_windows_npz_output.exists() and o.nn_classification_windows_output.exists()
    _run(fa, out)                                                         # flag off: nothing redone, files left alone
    assert len(stub.windows_seen()) == n3 and o.nn_classification_windows_npz_output.exists()


def test_environment_variable_and_cli(tmp_path, stub, monkeypatch):
    fa = _module_fasta(tmp_path / "sample.fna")
    monkeypatch.setenv("GENOMAD_B200_WINDOW_SCORES", "1")
    o = _run(fa, tmp_path / "env")
    assert o.nn_classification_windows_npz_output.exists() and o.nn_classification_windows_output.exists()
    monkeypatch.delenv("GENOMAD_B200_WINDOW_SCORES")
    for bad in (0, 6001):
        with pytest.raises(ValueError):
            _run(fa, tmp_path / "bad", write_window_scores=True, window_stride=bad)
    o = _run(fa, tmp_path / "stride_only", window_stride=1500)               # a stride implies the window scores
    assert int(np.load(o.nn_classification_windows_npz_output)["window_stride"]) == 1500
    o = _run(fa, tmp_path / "stride_off", write_window_scores=False, window_stride=1500)   # unless switched off explicitly
    assert not o.nn_classification_windows_npz_output.exists()
    from click.testing import CliRunner
    from genomad_b200 import cli
    seen = {}
    monkeypatch.setattr(nn_classification, "main", lambda *a, **k: seen.update(k))
    r = CliRunner().invoke(cli.cli, ["nn-classification", "--write-window-scores", "--window-stride", "750", str(fa),
                                     str(tmp_path / "o")])
    assert r.exit_code == 0, r.output
    assert seen == {"write_embeddings": None, "write_window_scores": True, "window_stride": 750}
    seen.clear()
    r = CliRunner().invoke(cli.cli, ["nn-classification", "--window-stride", "750", str(fa), str(tmp_path / "o")])
    assert r.exit_code == 0 and seen == {"write_embeddings": None, "window_stride": 750}
    for bad in ("0", "6001"):
        r = CliRunner().invoke(cli.cli, ["nn-classification", "--window-stride", bad, str(fa), str(tmp_path / "o")])
        assert r.exit_code != 0
