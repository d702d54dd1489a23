"""
GPU tests of the reverse strand (run with `-m gpu` on an H100): gnm_contig_windows_rc against the native reader's reverse list,
gnm_gather_windows_rc against the reader's export (and so against the reference's rc() windows, tests/golden/
reference_rc_golden.npz), gnm_forward_windows_rc / gnm_embed_windows_rc bitwise against gnm_forward_ascii / gnm_embed_ascii on
those rows, the module's strand invariants with the real classifier, and embedding-clusters --both-strands on sequences paired
with their reverse complements.
"""
import numpy as np
import pytest
import torch

from genomad_b200 import _paths, embedding_clusters, engine, nn_classification, sequence
from test_gpu_contigs import adversarial_contigs, random_contigs, to_device

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def clf():
    c = engine.Classifier(None, device=0, max_batch=256)
    yield c
    c.close()


@pytest.fixture(scope="module")
def contig_set():
    return adversarial_contigs() + random_contigs(2000, seed=9)


def _reader_list(contigs, tmp_path, stride, single_window):
    """The native reader's reverse list over the same contigs written as FASTA: (offsets, starts, lengths, rows)."""
    p = tmp_path / "contigs.fna"
    p.write_bytes(b"".join(b">c%d\n%s\n" % (i, s) for i, s in enumerate(contigs)))
    pf = sequence.ParsedFasta(p, single_window)
    wl = pf.windows(stride, single_window, reverse=True)
    try:
        offsets, starts, lengths = wl.spans()
        rows = wl.export_windows(0, wl.n_windows, np.empty((wl.n_windows, 6000), np.uint8))
    finally:
        wl.close()
        pf.close()
    return offsets, starts, lengths, rows


@pytest.mark.parametrize("stride,single_window", [(6000, False), (6000, True), (1000, False), (2501, False)])
def test_device_plan_and_gather_are_the_reader(clf, contig_set, tmp_path, stride, single_window):
    seq, offs = to_device(contig_set)
    start, length, woff = clf.contig_windows(seq, offs, single_window, stride=stride if not single_window else 6000,
                                             reverse=True)
    r_off, r_start, r_len, r_rows = _reader_list(contig_set, tmp_path, stride, single_window)
    # the reader drops records that are empty after stripping; the device keeps them with zero windows
    counts = np.diff(woff.cpu().numpy().astype(np.int64))
    kept = np.array([len(s.strip(b"nN")) > 0 for s in contig_set])
    assert (counts[~kept] == 0).all() and np.array_equal(counts[kept], np.diff(r_off.astype(np.int64)))
    contig = np.repeat(np.arange(len(contig_set)), counts)
    rel = start.cpu().numpy() - offs.cpu().numpy()[contig]
    assert np.array_equal(rel, r_start) and np.array_equal(length.cpu().numpy(), r_len)
    rows = clf.gather_windows(seq, start, length, reverse=True)
    assert np.array_equal(rows.cpu().numpy(), r_rows)


def test_gather_rc_is_the_reference(clf, golden_dir):
    """gnm_gather_windows_rc on the golden records gives the reference's own rc() windows, byte for byte."""
    z = np.load(golden_dir / "reference_rc_golden.npz")
    recs = [s for _, s in _records(z["fasta"].tobytes())]
    seq, offs = to_device(recs)
    for single, sfx in ((False, ""), (True, "_single")):
        start, length, woff = clf.contig_windows(seq, offs, single, reverse=True)
        rows = clf.gather_windows(seq, start, length, reverse=True).cpu().numpy()
        assert np.array_equal(rows, z["windows" + sfx])


def _records(text: bytes):
    """(name, joined lines) of every record, empty ones included (the device drops nothing by itself)."""
    out = []
    for rec in (b"\n" + text.replace(b"\r\n", b"\n")).split(b"\n>")[1:]:
        h, _, body = rec.partition(b"\n")
        out.append((h.split()[0].decode() if h.split() else "", body.replace(b"\n", b"")))
    return out


def test_forward_and_embed_rc_are_the_ascii_step_bitwise(clf, contig_set):
    seq, offs = to_device(contig_set[:600])
    start, length, woff = clf.contig_windows(seq, offs, reverse=True)
    rows = clf.gather_windows(seq, start, length, reverse=True)
    assert rows.shape[0] > 2 * clf.max_batch                                   # several internal steps
    p_rc = clf.predict_windows(seq, start, length, reverse=True)
    assert torch.equal(p_rc, clf.predict_ascii(rows))
    pe, e = clf.embed_windows(seq, start, length, reverse=True)
    pa, ea = clf.embed_ascii(rows)
    assert torch.equal(pe, pa) and torch.equal(e, ea) and torch.equal(pe, p_rc)


def test_classify_contigs_reverse_is_forward_of_rc(clf, contig_set):
    cs = contig_set[:800]
    rc = [sequence.reverse_complement(s) for s in cs]
    for single in (False, True):
        m_r, c_r, e_r = clf.classify_contigs(cs, single, return_embeddings=True, strand="reverse")
        m_f, c_f, e_f = clf.classify_contigs(rc, single, return_embeddings=True)
        assert torch.equal(m_r, m_f) and torch.equal(c_r, c_f) and torch.equal(e_r, e_f)
        m_a, _, e_a = clf.classify_contigs(cs, single, return_embeddings=True)
        m_b, _, e_b = clf.classify_contigs(rc, single, return_embeddings=True, strand="reverse")
        assert torch.equal(engine.both_strands(m_a, m_r), engine.both_strands(m_f, m_b))
        assert torch.equal(engine.both_strands(e_a, e_r), engine.both_strands(e_f, e_b))
    with pytest.raises(ValueError):
        clf.classify_contigs(cs[:2], strand="both")


def _module_input(path, seed=3, n=60):
    rng = np.random.default_rng(seed)
    with open(path, "wb") as fh:
        for i, L in enumerate(np.exp(rng.uniform(np.log(500), np.log(40000), n)).astype(int)):
            s = bytearray(np.frombuffer(b"ACGTacgt", np.uint8)[rng.integers(0, 8, L)].tobytes())
            if i % 7 == 3 and L > 14000:
                s[7000:11500] = b"N" * 4500                                       # dropped on one strand at most
            s = b"nN" * (i % 3) + bytes(s) + b"N" * (i % 4)
            fh.write(f">s{i} d\n".encode() + b"\n".join(s[j:j + 70] for j in range(0, len(s), 70)) + b"\n")
    return path


def _rc_file(src, dst):
    with open(dst, "wb") as fh:
        for h, s in sequence.iter_fasta(src, strip_n=False):
            r = sequence.reverse_complement(s)
            fh.write(f">{h}\n".encode() + b"\n".join(r[j:j + 60] for j in range(0, len(r), 60)) + b"\n")
    return dst


@pytest.mark.parametrize("single_window", [False, True])
def test_module_strand_invariants(tmp_path, single_window):
    fa = _module_input(tmp_path / "sample.fna")
    (tmp_path / "rc").mkdir()
    fr = _rc_file(fa, tmp_path / "rc" / "sample.fna")
    outs = {}
    for key, src, both in (("F", fa, True), ("R", fr, True), ("R_plain", fr, False), ("F_plain", fa, False)):
        nn_classification.main(src, tmp_path / key, single_window, 128, False, 4, False, False, write_embeddings=True,
                               both_strands=both)
        outs[key] = _paths.NNOutputs("sample", tmp_path / key)
    z = {k: np.load(o.nn_classification_strands_npz_output) for k, o in outs.items() if k in ("F", "R")}
    e = {k: np.load(o.nn_classification_embeddings_output) for k, o in outs.items()}
    preds = {k: np.load(o.nn_classification_npz_output)["predictions"] for k, o in outs.items()}
    assert np.array_equal(z["F"]["reverse"], z["R"]["forward"]) and np.array_equal(z["F"]["reverse"], preds["R_plain"])
    assert np.array_equal(z["F"]["forward"], preds["F_plain"]) and np.array_equal(preds["F"], preds["F_plain"])
    assert np.array_equal(z["F"]["both_strands"], z["R"]["both_strands"])
    assert np.array_equal(e["F"]["embeddings_reverse"], e["R_plain"]["embeddings"])
    assert np.array_equal(e["F"]["embeddings_both_strands"], e["R"]["embeddings_both_strands"])
    assert e["F"]["embeddings"].tobytes() == e["F_plain"]["embeddings"].tobytes()
    assert not np.array_equal(z["F"]["forward"], z["F"]["reverse"])


def test_clusters_pair_each_sequence_with_its_reverse_complement(tmp_path):
    rng = np.random.default_rng(21)
    fa = tmp_path / "pairs.fna"
    with open(fa, "wb") as fh:
        for i in range(40):
            L = int(rng.integers(3000, 30000))
            s = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, L)].tobytes()
            fh.write(f">p{i}\n".encode() + s + b"\n" + f">p{i}_rc\n".encode() + sequence.reverse_complement(s) + b"\n")
    nn_classification.main(fa, tmp_path / "nn", False, 128, False, 4, False, False, write_embeddings=True, both_strands=True)
    emb = _paths.NNOutputs("pairs", tmp_path / "nn").nn_classification_embeddings_output
    embedding_clusters.main(emb, tmp_path / "cl", 0.999, False, both_strands=True)
    z = np.load(tmp_path / "cl" / "pairs_embedding_clusters.npz")
    rep = z["representative_index"]
    assert len(z["representatives"]) == 40
    assert all(rep[2 * i] == 2 * i and rep[2 * i + 1] == 2 * i for i in range(40))
    assert (z["similarity"][1::2] >= np.float32(0.999)).all()
