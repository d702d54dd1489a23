"""
GPU tests of the contig -> window path (run with `-m gpu` on an H100): gnm_contig_windows / gnm_gather_windows /
gnm_forward_windows and Classifier.classify_contigs, against

  * the pure-Python statement of the windowing rules (sequence.window_spans + the N rule, in NumPy),
  * the native FASTA reader on the same contigs written as FASTA text (gnm_fasta_parse / gnm_fasta_export),
  * gnm_forward_ascii on the gathered windows (bitwise), and the CPU oracle within the 1e-4 bar.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from genomad_b200 import engine, sequence
from oracle import igloo_model as M
from oracle import tokenizer as T

pytestmark = pytest.mark.gpu

TOL = 1e-4
ACGT = b"ACGT"


def _rnd(rng, n, alphabet=ACGT):
    return np.frombuffer(alphabet, np.uint8)[rng.integers(0, len(alphabet), n)].tobytes()


def _with_n(rng, body, k, ch):
    """body with k bytes (never the last one) replaced by ch"""
    b = bytearray(body)
    for p in rng.choice(len(b) - 1, k, replace=False):
        b[p] = ch[0]
    return bytes(b)


def adversarial_contigs():
    rng = np.random.default_rng(11)
    c = [b"", b"N" * 5000, b"n" * 7000, b"nNnN" * 3000, b"N" * 1_000_000, b"N", b"n"]
    c += [b"NNnn" + _rnd(rng, 9000) + b"nnNN", b"n" * 12345 + _rnd(rng, 14000) + b"N" * 6001 + b"nNnN"]
    c += [_rnd(rng, n) for n in (1, 3, 4, 2499, 2500, 5999, 6000, 6001, 8499, 8500, 12000 + 2499)]
    c += [b"nN" + _rnd(rng, n) + b"Nn" for n in (1, 2499, 2500, 8499, 8500)]
    # second windows with exactly 4000 / 4001 'N' (kept / dropped) and 4001 'n' (kept: the rule is case-sensitive)
    for k, ch in ((4000, b"N"), (4001, b"N"), (4001, b"n")):
        c.append(_rnd(rng, 6000) + _with_n(rng, _rnd(rng, 6000), k, ch) + _rnd(rng, 3000))
        c.append(_rnd(rng, 6000) + _with_n(rng, _rnd(rng, 3000), min(k, 2999), ch))      # short tail, same rule
    c.append(_rnd(rng, 6000) + b"N" * 6000 + _rnd(rng, 6000) + b"N" * 4001 + _rnd(rng, 1999))   # drops in the middle
    c.append(_rnd(rng, 20000, b"acgtACGT"))                                                      # lower case
    c.append(_rnd(rng, 15000, b"ACGTRYKMSWBDHVNacgtrykmswbdhvn"))                                # IUPAC codes
    c.append(_rnd(rng, 13000, bytes(b for b in range(256) if b not in b"\n\r>")))               # every other byte
    c.append(_rnd(rng, 9001, b"Nn") + _rnd(rng, 2) + _rnd(rng, 9001, b"Nn"))                    # two bases amid n/N
    return c


def random_contigs(n, seed):
    """Log-uniform lengths with N runs, n runs, lower-case stretches and stripped ends mixed in."""
    rng = np.random.default_rng(seed)
    out = []
    for L in np.exp(rng.uniform(np.log(1), np.log(40000), n)).astype(int):
        s = bytearray(_rnd(rng, L))
        for _ in range(rng.integers(0, 4)):
            a = int(rng.integers(0, L)); e = min(L, a + int(rng.integers(1, 7000)))
            s[a:e] = _rnd(rng, e - a, [b"N", b"n", b"acgt", b"NNNNn"][rng.integers(0, 4)])
        out.append(_rnd(rng, rng.integers(0, 50), b"nN") + bytes(s) + _rnd(rng, rng.integers(0, 50), b"nN"))
    return out


def expected_plan(contigs, single_window):
    """NumPy statement: read_fasta(strip_n=True) -> seq_windows(6000, 2500) -> N rule; starts are absolute offsets."""
    starts, lens, counts, pos = [], [], [], 0
    for s in contigs:
        st = s.strip(b"nN")
        lead = len(s) - len(s.lstrip(b"nN"))
        k = 0
        for wn, (a, e) in enumerate(sequence.window_spans(len(st), single_window)):
            if wn > 0 and st[a:e].count(b"N") > sequence.MAX_N:
                continue
            starts.append(pos + lead + a); lens.append(e - a); k += 1
        counts.append(k)
        pos += len(s)
    return np.array(starts, np.int64), np.array(lens, np.int32), np.array(counts, np.int64)


def to_device(contigs, odd=True):
    """Contigs back to back in a device buffer that starts at an odd address (odd=True), plus int64 offsets."""
    raw = np.frombuffer(b"".join(contigs), np.uint8)
    big = torch.zeros(raw.size + 17, dtype=torch.uint8, device="cuda")
    seq = big[1:1 + raw.size] if odd else big[:raw.size]
    if raw.size:
        seq.copy_(torch.from_numpy(raw.copy()))
    offs = np.zeros(len(contigs) + 1, np.int64)
    np.cumsum([len(s) for s in contigs], out=offs[1:])
    return seq, torch.from_numpy(offs).cuda()


def fasta_reference(contigs, tmp_path, single_window):
    p = tmp_path / "contigs.fna"
    p.write_bytes(b"".join(b">c%d\n%s\n" % (i, s) for i, s in enumerate(contigs)))
    return sequence.encode_fasta(p, single_window=single_window)


@pytest.fixture(scope="module")
def shipped(weights_npz):
    return M.load_npz_weights(weights_npz)


@pytest.fixture(scope="module")
def clf():
    c = engine.Classifier(None, device=0, max_batch=256)
    yield c
    c.close()


@pytest.fixture(scope="module")
def contig_set():
    return adversarial_contigs() + random_contigs(3000, seed=5)


# ------------------------------------------------------------------------------------------ plan + bytes
@pytest.mark.parametrize("single_window", [False, True])
def test_plan_and_bytes_match_numpy_and_fasta_reader(clf, contig_set, tmp_path, single_window):
    seq, offs = to_device(contig_set)
    assert seq.data_ptr() % 2 == 1
    start, length, woff = clf.contig_windows(seq, offs, single_window)
    exp_start, exp_len, exp_counts = expected_plan(contig_set, single_window)
    assert np.array_equal(start.cpu().numpy(), exp_start)
    assert np.array_equal(length.cpu().numpy(), exp_len)
    counts = np.diff(woff.cpu().numpy().astype(np.int64))
    assert np.array_equal(counts, exp_counts) and woff[0].item() == 0
    ref = fasta_reference(contig_set, tmp_path, single_window)
    assert np.array_equal(counts[counts > 0], np.diff(ref.offsets.astype(np.int64)))       # FASTA drops empty contigs
    ascii_w = clf.gather_windows(seq, start, length).cpu().numpy()
    assert ascii_w.shape == ref.windows.shape and np.array_equal(ascii_w, ref.windows)
    clf.check_status()


def test_plan_is_independent_of_the_buffer_address(clf, contig_set):
    seq_odd, offs = to_device(contig_set[:200], odd=True)
    seq_even, _ = to_device(contig_set[:200], odd=False)
    a = clf.contig_windows(seq_odd, offs)
    b = clf.contig_windows(seq_even, offs)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert torch.equal(clf.gather_windows(seq_odd, *a[:2]), clf.gather_windows(seq_even, *b[:2]))
    clf.check_status()


# ------------------------------------------------------------------------------------------ probabilities
@pytest.mark.parametrize("max_batch", [16, 1024])
def test_forward_windows_bitwise_equals_forward_ascii(contig_set, max_batch):
    c = engine.Classifier(None, device=0, max_batch=max_batch)
    try:
        seq, offs = to_device(contig_set)
        start, length, _ = c.contig_windows(seq, offs)
        if max_batch == 16:
            start, length = start[:200], length[:200]           # 13 steps; contigs straddle them
        ascii_w = c.gather_windows(seq, start, length)
        for overlap in (0, 1):
            c.set_option("tail_overlap", overlap)
            p_win = c.predict_windows(seq, start, length)
            p_asc = c.predict_ascii(ascii_w)
            c.check_status()
            assert torch.equal(p_win, p_asc), (max_batch, overlap)
    finally:
        c.close()


# ------------------------------------------------------------------------------------------ per-contig scores
def _fasta_path_scores(c, contigs, tmp_path):
    ref = fasta_reference(contigs, tmp_path, False)
    probs = c.predict_ascii(torch.from_numpy(ref.windows).cuda())
    return c.segment_mean(probs, torch.from_numpy(ref.offsets).cuda()), probs, ref


@pytest.mark.parametrize("weights", ["shipped", "synthetic"])
def test_classify_contigs_matches_fasta_path_and_oracle(shipped, tmp_path, weights):
    w = shipped if weights == "shipped" else M.synthetic_igloo_weights(shipped)
    c = engine.Classifier(None if weights == "shipped" else w, device=0, max_batch=64)
    try:
        contigs = adversarial_contigs() + random_contigs(400, seed=8)
        means, counts, probs = c.classify_contigs(contigs, return_window_probs=True)
        c.check_status()
        kept = counts.cpu().numpy() > 0
        ref_means, ref_probs, ref = _fasta_path_scores(c, contigs, tmp_path)
        assert torch.equal(probs, ref_probs)
        assert torch.equal(means[torch.from_numpy(kept).cuda()], ref_means)
        assert not means[torch.from_numpy(~kept).cuda()].any()                 # empty contigs: zeros
        # the same through a (device tensor, offsets) pair and a host (array, offsets) pair
        seq, offs = to_device(contigs)
        m2, n2 = c.classify_contigs((seq, offs))
        raw = np.frombuffer(b"".join(contigs), np.uint8).copy()
        m3, n3 = c.classify_contigs((raw, offs.cpu().numpy()))
        assert torch.equal(m2, means) and torch.equal(m3, means) and torch.equal(n2, counts) and torch.equal(n3, counts)
        # oracle on a small subset: contigs with one or two windows
        sub = [s for s in contigs if 0 < len(s.strip(b"nN")) <= 14000][:8]
        sm, sc, sp = c.classify_contigs(sub, return_window_probs=True)
        r = fasta_reference(sub, tmp_path, False)
        oracle = M.forward(T.tokenize_windows(r.windows), w, torch.float32)
        assert np.abs(sp.cpu().numpy() - oracle).max() <= TOL
        assert np.array_equal(sp.cpu().numpy().argmax(1), oracle.argmax(1))
        om = T.segment_mean(oracle, r.contig_ids, len(sub))
        assert np.abs(sm.cpu().numpy() - om).max() <= TOL
        top2 = np.sort(om, axis=1)[:, -2:]
        clear = top2[:, 1] - top2[:, 0] > 2 * TOL
        assert np.array_equal(sm.cpu().numpy().argmax(1)[clear], om.argmax(1)[clear])
    finally:
        c.close()


# ------------------------------------------------------------------------------------------ edges
def test_edges_empty_sets_capacity_and_bad_offsets(clf):
    t = torch
    seq = t.zeros(16, dtype=t.uint8, device="cuda")
    start, length, woff = clf.contig_windows(seq, t.zeros(1, dtype=t.int64, device="cuda"))
    assert start.numel() == 0 and woff.cpu().tolist() == [0]
    m, n = clf.classify_contigs([])
    assert m.shape == (0, 3) and n.shape == (0,)
    clf.check_status()

    m, n, p = clf.classify_contigs(["", "NNN", "nnnn", b"nNn", ""], return_window_probs=True)
    assert n.cpu().tolist() == [0] * 5 and p.shape == (0, 3) and not m.any()
    clf.check_status()

    contigs = adversarial_contigs()
    seq, offs = to_device(contigs)
    need = int(expected_plan(contigs, False)[2].sum())
    guard = 64
    for cap in (need - 1, 0):
        ws = t.full((cap + guard,), -5, dtype=t.int64, device="cuda")
        wl = t.full((cap + guard,), -5, dtype=t.int32, device="cuda")
        wo = t.empty(len(contigs) + 1, dtype=t.int32, device="cuda")
        nw = C.c_int64(-1)
        rc = clf.lib.gnm_contig_windows(clf._h, seq.data_ptr(), offs.data_ptr(), len(contigs), 0, ws.data_ptr(), wl.data_ptr(),
                                        cap, wo.data_ptr(), C.byref(nw), clf._stream())
        assert rc != 0 and "capacity" in clf.lib.gnm_last_error().decode()
        assert nw.value == need
        assert bool((ws == -5).all()) and bool((wl == -5).all())          # nothing written, guard region included
        clf.check_status()

    bad = offs.clone()
    bad[3], bad[4] = offs[4], offs[3]                    # contig 3 ends before it starts
    with pytest.raises(engine.GnmError, match="non-decreasing"):
        clf.contig_windows(seq, bad)
    clf.check_status()
