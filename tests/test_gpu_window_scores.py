"""
GPU tests of the per-window score export (run with `-m gpu` on an H100): gnm_contig_windows_stride against the pure-Python
statement (sequence.profile_spans + the N rule), the stride-6000 call against gnm_contig_windows, Classifier.window_scores
against gnm_forward_ascii on the gathered windows and against classify_contigs, the capacity failure, and the module's windows
NPZ on the GPU.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from genomad_b200 import _paths, engine, nn_classification, sequence
from test_gpu_contigs import adversarial_contigs, random_contigs
import window_stub as WS

pytestmark = pytest.mark.gpu

STRIDES = [1, 7, 8, 999, 1000, 2500, 5999, 6000]


@pytest.fixture(scope="module")
def clf():
    c = engine.Classifier(None, device=0, max_batch=256)
    yield c
    c.close()


def expected_profile(contigs, stride):
    """NumPy statement: strip n/N, profile_spans, N rule (prefix counts); starts are absolute offsets."""
    starts, lens, counts, pos = [], [], [], 0
    for s in contigs:
        st = s.strip(b"nN")
        lead = len(s) - len(s.lstrip(b"nN"))
        cum = np.concatenate([[0], np.cumsum(np.frombuffer(st, np.uint8) == ord("N"))]) if st else np.zeros(1, np.int64)
        k = 0
        for wn, (a, e) in enumerate(sequence.profile_spans(len(st), stride)):
            if wn > 0 and cum[e] - cum[a] > sequence.MAX_N:
                continue
            starts.append(pos + lead + a); lens.append(e - a); k += 1
        counts.append(k)
        pos += len(s)
    return np.array(starts, np.int64), np.array(lens, np.int32), np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)


def _contigs(stride):
    c = adversarial_contigs() + random_contigs(60, seed=stride)
    for k in (1, 2, 3):                                              # lengths k*s - 1, k*s, k*s + 1 plus 2500
        c += [bytes(np.frombuffer(b"ACGT", np.uint8)[np.random.default_rng(k).integers(0, 4, k * stride + 2500 + d)])
              for d in (-1, 0, 1)]
    return c


def _plan_stride(clf, seq, offs, stride, cap=None):
    n = offs.numel() - 1
    cap = n + seq.numel() // stride if cap is None else cap
    start = torch.empty(max(1, cap), dtype=torch.int64, device="cuda")
    length = torch.empty(max(1, cap), dtype=torch.int32, device="cuda")
    woff = torch.empty(n + 1, dtype=torch.int32, device="cuda")
    nw = C.c_int64()
    rc = clf.lib.gnm_contig_windows_stride(clf._h, seq.data_ptr(), offs.data_ptr(), n, stride, start.data_ptr(),
                                           length.data_ptr(), cap, woff.data_ptr(), C.byref(nw), clf._stream())
    return rc, start[:nw.value], length[:nw.value], woff, nw.value


@pytest.mark.parametrize("stride", STRIDES)
def test_device_planner_matches_profile_spans(clf, stride):
    contigs = _contigs(stride)
    seq, offs = clf.contig_buffers(contigs)
    want_s, want_l, want_o = expected_profile(contigs, stride)
    rc, start, length, woff, nw = _plan_stride(clf, seq, offs, stride)
    assert rc == 0, clf.lib.gnm_last_error()
    assert nw == len(want_s)
    assert np.array_equal(woff.cpu().numpy(), want_o)
    assert np.array_equal(start.cpu().numpy(), want_s) and np.array_equal(length.cpu().numpy(), want_l)
    s2, l2, o2 = clf.contig_windows(seq, offs, stride=stride)            # the Python entry point, same plan
    assert torch.equal(s2, start) and torch.equal(l2, length) and torch.equal(o2, woff)


def test_stride_6000_is_gnm_contig_windows(clf):
    contigs = _contigs(6000) + random_contigs(300, seed=99)
    seq, offs = clf.contig_buffers(contigs)
    rc, start, length, woff, nw = _plan_stride(clf, seq, offs, 6000)
    assert rc == 0
    s0, l0, o0 = clf.contig_windows(seq, offs)                           # gnm_contig_windows
    assert torch.equal(s0, start) and torch.equal(l0, length) and torch.equal(o0, woff)


def test_capacity_one_window_short_fails(clf):
    contigs = _contigs(1000)
    seq, offs = clf.contig_buffers(contigs)
    _rc, _s, _l, _o, nw = _plan_stride(clf, seq, offs, 1000)
    rc, *_ = _plan_stride(clf, seq, offs, 1000, cap=nw - 1)
    assert rc != 0
    msg = clf.lib.gnm_last_error().decode()
    assert msg == (f"gnm_contig_windows_stride: the contigs have {nw} windows, capacity is {nw - 1} "
                   f"(n_contigs + total_bytes / 1000 is always enough)")
    rc, *_ = _plan_stride(clf, seq, offs, 0, cap=nw)
    assert rc != 0 and "stride must be in [1, 6000]" in clf.lib.gnm_last_error().decode()


@pytest.mark.parametrize("stride", [1000, 2500, 5999])
def test_window_scores_are_forward_ascii_of_the_gathered_plan(clf, stride):
    contigs = adversarial_contigs() + random_contigs(40, seed=5)
    ws = clf.window_scores(contigs, stride=stride)
    seq, offs = clf.contig_buffers(contigs)
    start, length, woff = clf.contig_windows(seq, offs, stride=stride)
    ref = clf.predict_ascii(clf.gather_windows(seq, start, length))
    assert torch.equal(ws.probs, ref)
    assert torch.equal(ws.offsets, woff) and torch.equal(ws.length, length)
    cid = ws.contig.long()
    assert torch.equal(ws.start + offs[:-1][cid], start)
    assert torch.equal(torch.bincount(cid, minlength=len(contigs)).int(), woff[1:] - woff[:-1])
    assert ws.contig.dtype == torch.int32 and ws.start.dtype == torch.int64 and ws.length.dtype == torch.int32
    clf.check_status()


def test_window_scores_at_6000_are_classify_contigs(clf):
    contigs = adversarial_contigs() + random_contigs(80, seed=8)
    ws = clf.window_scores(contigs)
    means, counts, probs = clf.classify_contigs(contigs, return_window_probs=True)
    assert torch.equal(ws.probs, probs)
    assert torch.equal(clf.segment_mean(ws.probs, ws.offsets), means)
    assert torch.equal(ws.offsets[1:] - ws.offsets[:-1], counts)
    clf.check_status()


def test_module_windows_npz_reproduces_contig_predictions(tmp_path):
    rng = np.random.default_rng(3)
    fa = tmp_path / "sample.fna"
    with open(fa, "w") as fh:
        for i, ln in enumerate([20000, 3000, 47000, 6100, 1200, 31000, 9000]):
            s = np.frombuffer(b"ACGTacgt", np.uint8)[rng.integers(0, 8, ln)].tobytes().decode()
            fh.write(f">c{i}\n" + "\n".join(s[k:k + 60] for k in range(0, ln, 60)) + "\n")
    out = tmp_path / "out"
    nn_classification.main(fa, out, False, 128, False, 4, False, False, write_window_scores=True)
    o = _paths.NNOutputs("sample", out)
    z, p = np.load(o.nn_classification_windows_npz_output), np.load(o.nn_classification_npz_output)
    offsets = np.concatenate([[0], np.cumsum(np.bincount(z["window_contig"], minlength=len(p["contig_names"])))])
    assert np.array_equal(WS.running_mean(z["predictions"], offsets), p["predictions"])
    nn_classification.main(fa, tmp_path / "p1000", False, 128, False, 4, False, False, write_window_scores=True,
                           window_stride=1000)
    o2 = _paths.NNOutputs("sample", tmp_path / "p1000")
    assert np.array_equal(np.load(o2.nn_classification_npz_output)["predictions"], p["predictions"])
    z2 = np.load(o2.nn_classification_windows_npz_output)
    assert int(z2["window_stride"]) == 1000 and len(z2["predictions"]) > 3 * len(z["predictions"])
    at0 = z2["window_start"] % 6000 == 0                                   # windows that are also reference windows
    k = {(int(c), int(s)): i for i, (c, s) in enumerate(zip(z["window_contig"], z["window_start"]))}
    for i in np.nonzero(at0)[0]:
        j = k.get((int(z2["window_contig"][i]), int(z2["window_start"][i])))
        if j is not None:
            assert np.array_equal(z2["predictions"][i], z["predictions"][j])
