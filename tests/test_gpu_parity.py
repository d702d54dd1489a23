"""
GPU parity tests (run with `-m gpu` on an H100): the CUDA path, called through the C ABI of libgnm.so,
against the CPU oracle and the committed golden fixtures.

Tolerances: tokens are bit-exact; per-window probabilities are within 1e-4 (absolute) of the fp32 oracle
-- the bar BASELINE.json's north_star states -- and class calls (argmax) are identical.
"""
import hashlib
import json

import numpy as np
import pytest
import torch

from oracle import igloo_model as M
from oracle import tokenizer as T

pytestmark = pytest.mark.gpu

TOL = 1e-4


def _families(n, seed):
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tools"))
    import precision_study
    return precision_study.make_windows(n, seed)


@pytest.fixture(scope="module")
def shipped(weights_npz):
    return M.load_npz_weights(weights_npz)


@pytest.fixture(scope="module")
def clf():
    from genomad_b200 import engine
    c = engine.Classifier(None, device=0, max_batch=256)
    yield c
    c.close()


@pytest.fixture(scope="module")
def clf_syn(shipped):
    from genomad_b200 import engine
    c = engine.Classifier(M.synthetic_igloo_weights(shipped), device=0, max_batch=64)
    yield c
    c.close()


def _oracle_probs(tok, w, dtype=torch.float32, bs=32):
    return np.concatenate([M.forward(tok[i:i + bs], w, dtype) for i in range(0, len(tok), bs)])


# ------------------------------------------------------------------------------------------ encoder
def test_encode_bitexact_reference_golden(clf, golden_dir):
    enc = json.loads((golden_dir / "encoder_golden.json").read_text())
    ref = np.load(golden_dir / "encoder_batch_tokens.npz")["tokens"]       # produced by the REAL reference tokenizer
    a = np.frombuffer(b"".join(r.upper().encode("ascii").ljust(6000, b"N") for r in enc["batch"]["raw"]),
                      np.uint8).reshape(-1, 6000)
    tok = clf.encode(torch.from_numpy(a.copy()).cuda()).cpu().numpy()
    assert tok.dtype == np.uint16 and np.array_equal(tok, ref)
    assert hashlib.sha256(tok.tobytes()).hexdigest() == enc["batch"]["tokens_sha256"]


def test_encode_adversarial_bytes(clf):
    rng = np.random.default_rng(9)
    a = rng.integers(0, 256, (257, 6000), dtype=np.uint8)                # every byte value, incl. lowercase / IUPAC / NUL
    a[1] = ord("N"); a[2] = ord("A"); a[3, ::7] = ord("n"); a[4, :3] = ord("N"); a[5, -3:] = ord("N")
    tok = clf.encode(torch.from_numpy(a).cuda()).cpu().numpy()
    assert np.array_equal(tok, T.tokenize_windows(a))
    assert tok[1].max() == 0 and tok[2].min() == 1 == tok[2].max()
    assert clf.encode(torch.empty((0, 6000), dtype=torch.uint8, device="cuda")).shape == (0, 5997)


# ------------------------------------------------------------------------------------------ model
def test_forward_matches_frozen_golden(clf, golden_dir):
    g = np.load(golden_dir / "model_golden.npz")
    p = clf.predict_ascii(torch.from_numpy(g["ascii"]).cuda()).cpu().numpy()
    assert np.abs(p - g["shipped_fp32"]).max() <= TOL
    assert np.abs(p - g["shipped_fp64"]).max() <= TOL
    assert np.array_equal(p.argmax(1), g["shipped_fp64"].argmax(1))
    assert np.allclose(p.sum(1), 1.0, atol=1e-6)


def test_forward_synthetic_weights_match_frozen_golden(clf_syn, golden_dir):
    """Non-degenerate patch/attention weights: a wrong gather or softmax cannot hide here."""
    g = np.load(golden_dir / "model_golden.npz")
    p = clf_syn.predict_ascii(torch.from_numpy(g["ascii"]).cuda()).cpu().numpy()
    assert np.abs(p - g["synthetic_fp32"]).max() <= TOL
    assert np.array_equal(p.argmax(1), g["synthetic_fp64"].argmax(1))


def test_forward_parity_mixed_families(clf, shipped):
    a = _families(96, seed=21)                      # iid, GC-skew, tandem repeats, N tails, Markov, homopolymer, N islands
    tok = T.tokenize_windows(a)
    ref = _oracle_probs(tok, shipped)
    p = clf.predict_ascii(torch.from_numpy(a).cuda()).cpu().numpy()
    assert np.abs(p - ref).max() <= TOL
    assert np.array_equal(p.argmax(1), ref.argmax(1))
    p2 = clf.predict_tokens(torch.from_numpy(tok.view(np.int16)).cuda().view(torch.uint16)).cpu().numpy()
    assert np.array_equal(p, p2)                    # fused encode == separate encode, bitwise


def test_stagewise_parity_synthetic(clf_syn, shipped):
    w = M.synthetic_igloo_weights(shipped)
    a = _families(8, seed=5)
    tok = T.tokenize_windows(a)
    _, it = M.forward(tok, w, torch.float32, return_intermediates=True)
    da = torch.from_numpy(a).cuda()

    def close(name, got, ref, rel):
        ref = ref.numpy() if hasattr(ref, "numpy") else ref
        d = np.abs(got.cpu().numpy().astype(np.float64) - ref).max()
        assert d <= rel * max(1.0, np.abs(ref).max()), (name, d)

    try:
        clf_syn.set_option("debug_stop", 1); clf_syn.predict_ascii(da); torch.cuda.synchronize()
        close("y1", clf_syn.debug_fetch("buf0", 8), it["y1"], 2e-6)
        close("mpi0", clf_syn.debug_fetch("mpi0", 8), it["ig0"]["mpi"], 1e-5)
        clf_syn.set_option("debug_stop", 2); clf_syn.predict_ascii(da); torch.cuda.synchronize()
        close("y2", clf_syn.debug_fetch("buf1", 8), it["y2"], 6e-5)      # stored as hi16 + e4m3 correction (what conv3 reads)
        close("q0", clf_syn.debug_fetch("q0", 8), it["ig0"]["q"], 1e-5)
        clf_syn.set_option("debug_stop", 3); clf_syn.predict_ascii(da); torch.cuda.synchronize()
        close("y3", clf_syn.debug_fetch("buf0", 8), it["y3"], 2e-5)
    finally:
        clf_syn.set_option("debug_stop", 0)
    clf_syn.predict_ascii(da); torch.cuda.synchronize()
    close("q1", clf_syn.debug_fetch("q1", 8), it["ig1"]["q"], 1e-5)
    close("mpi1", clf_syn.debug_fetch("mpi1", 8), it["ig1"]["mpi"], 2e-5)
    close("h0", clf_syn.debug_fetch("h0", 8), it["h0"], 1e-5)


def test_tensor_core_path_vs_cuda_core_validation_kernels(clf):
    """512 windows: wgmma fp16x3 path vs the independent fp32 FFMA kernels, both on the GPU."""
    a = torch.from_numpy(_families(512, seed=33)).cuda()
    p_tc = clf.predict_ascii(a).clone()
    try:
        clf.set_option("conv_impl", 1)
        p_ref = clf.predict_ascii(a).clone()
    finally:
        clf.set_option("conv_impl", 0)
    assert (p_tc - p_ref).abs().max().item() <= 5e-5
    assert torch.equal(p_tc.argmax(1), p_ref.argmax(1))


def test_batching_invariance_and_host_path(clf):
    a = _families(300, seed=2)                                            # > max_batch (256): two internal steps
    da = torch.from_numpy(a).cuda()
    p_all = clf.predict_ascii(da).cpu().numpy()
    p_one = np.concatenate([clf.predict_ascii(da[i:i + 1]).cpu().numpy() for i in (0, 7, 255, 256, 299)])
    assert np.array_equal(p_one, p_all[[0, 7, 255, 256, 299]])            # position in the batch does not matter
    perm = np.random.default_rng(0).permutation(300)
    assert np.array_equal(clf.predict_ascii(da[torch.from_numpy(perm).cuda()]).cpu().numpy(), p_all[perm])
    assert np.array_equal(clf.classify_host(a), p_all)                    # host-buffer entry point == device entry point
    assert clf.classify_host(a[:0]).shape == (0, 3)
    n0 = clf.kernel_launches
    clf.predict_ascii(da[:4])
    assert clf.kernel_launches - n0 == 18                                 # our kernels really launched (1 + 2x2 + 2 + 2x3 + 5)


def test_segment_mean_and_sum(clf):
    rng = np.random.default_rng(4)
    counts = np.array([1, 167, 0, 2, 13, 1, 1, 40], np.int64)             # includes an empty segment
    W = int(counts.sum())
    probs = rng.random((W, 3)).astype(np.float32)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    dp, do = torch.from_numpy(probs).cuda(), torch.from_numpy(offsets).cuda()
    mean = clf.segment_mean(dp, do).cpu().numpy()
    ref = T.segment_mean(probs, np.repeat(np.arange(len(counts)), counts), len(counts))
    assert np.array_equal(mean, ref)                                      # same sequential fp32 order -> bitwise
    s4 = clf.segment_sum(dp, do).cpu().numpy()
    assert np.array_equal(s4[:, 3], counts.astype(np.float32))
    assert np.allclose(s4[:, :3] / np.maximum(s4[:, 3:4], 1), ref, atol=1e-6)


# ------------------------------------------------------------------------------------------ full-size properties
def test_config2_scale_properties():
    """BASELINE config 2 shape (batch 1024) at reduced length: 20 steps of 1024 windows drawn from a 1024-window
    pool in a different order each step -> results are a pure function of the window (idempotence), rows are
    probabilities, and the checksum of checksums is order-independent."""
    from genomad_b200 import engine
    c = engine.Classifier(None, device=0, max_batch=1024)
    pool = torch.from_numpy(_families(1024, seed=77)).cuda()
    base = c.predict_ascii(pool).clone()
    assert torch.all(base >= 0) and torch.all(base <= 1)
    assert (base.sum(1) - 1).abs().max().item() < 1e-5
    g = torch.Generator(device="cpu").manual_seed(0)
    total = torch.zeros(3, dtype=torch.float64, device="cuda")
    for _ in range(20):
        perm = torch.randperm(1024, generator=g).cuda()
        p = c.predict_ascii(pool[perm])
        assert torch.equal(p, base[perm])
        total += p.double().sum(0)
    assert torch.allclose(total, base.double().sum(0) * 20, rtol=0, atol=1e-9)
    c.close()


# ------------------------------------------------------------------------------------------ module on the GPU (config 1)
def test_cli_config1_end_to_end(tmp_path, shipped):
    """BASELINE config 1: 100 synthetic 10 kb contigs through the CLI; TSV/NPZ vs the CPU oracle pipeline."""
    from click.testing import CliRunner
    from genomad_b200 import cli, _paths
    rng = np.random.default_rng(0)
    fa = tmp_path / "cfg1.fna"
    with open(fa, "w") as fh:
        for i in range(100):
            s = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 10000)].tobytes().decode()
            fh.write(f">contig_{i:03d}\n")
            for k in range(0, 10000, 60):
                fh.write(s[k:k + 60] + "\n")
    out = tmp_path / "out"
    r = CliRunner().invoke(cli.cli, ["nn-classification", "--quiet", "--batch-size", "128", str(fa), str(out)])
    assert r.exit_code == 0, r.output
    o = _paths.NNOutputs("cfg1", out)
    z = np.load(o.nn_classification_npz_output)
    names, ids, ascii_arr, tok = T.encode_fasta(fa)
    assert len(ids) == 200 and list(z["contig_names"]) == list(names)
    ref = T.segment_mean(_oracle_probs(tok, shipped), ids)
    assert np.abs(z["predictions"] - ref).max() <= TOL
    assert np.array_equal(z["predictions"].argmax(1), ref.argmax(1))
    lines = o.nn_classification_output.read_text().splitlines()
    assert len(lines) == 101 and lines[0].split("\t") == ["seq_name", "chromosome_score", "plasmid_score", "virus_score"]
    for line, name, row in zip(lines[1:], names, ref):
        f = line.split("\t")
        assert f[0] == name and all(abs(float(x) - y) <= TOL + 5e-5 for x, y in zip(f[1:], row))


def test_conv_operand_scaling_rule(shipped):
    """The per-layer operand scaling chosen in gnm_create (conv_t.cuh): conv2 weights x4 (|W| > 0.78 -> smaller 2^d),
    conv3 weights / 4 (small weights in the e4m3 planes).  The network function changes, so compare with the oracle
    evaluated on the same modified weights."""
    from genomad_b200 import engine
    w = dict(shipped)
    w["c2w"] = (shipped["c2w"] * 4).astype(np.float32)
    w["c3w"] = (shipped["c3w"] / 4).astype(np.float32)
    a = _families(24, seed=9)
    tok = T.tokenize_windows(a)
    ref = _oracle_probs(tok, w)
    c = engine.Classifier(w, device=0, max_batch=32)
    try:
        p = c.predict_ascii(torch.from_numpy(a).cuda()).cpu().numpy()
    finally:
        c.close()
    assert np.abs(p - ref).max() <= TOL
    assert np.array_equal(p.argmax(1), ref.argmax(1))


def test_module_mixed_lengths_single_window_and_n_rich(tmp_path, shipped):
    """BASELINE config 5 shape in miniature: contig lengths 1 kb - 60 kb, lower-case and N-rich stretches, a contig that is
    dropped after stripping, CRLF line ends; multi-window and --single-window runs against the oracle pipeline."""
    from genomad_b200 import nn_classification, _paths
    rng = np.random.default_rng(12)
    recs = []
    for i, ln in enumerate([1000, 2499, 2500, 6000, 6001, 8500, 14499, 33000, 60000, 12000]):
        s = np.frombuffer(b"ACGTacgtN", np.uint8)[rng.choice(9, ln, p=[.22, .22, .22, .22, .025, .025, .025, .025, .02])].copy()
        if i == 7:
            s[6000:11000] = ord("N")          # window 1 has > 4000 N -> skipped by the reference's rule
        if i == 9:
            s[:700] = ord("N"); s[-900:] = ord("n")   # stripped before windowing
        recs.append(f">ctg{i} len={ln}\r\n" + "\r\n".join(s.tobytes().decode()[k:k + 70] for k in range(0, ln, 70)))
    recs.append(">all_n\r\nNNNNNNNNNNnnnnnnnn")
    fa = tmp_path / "mixed.fna"
    fa.write_text("\r\n".join(recs) + "\r\n", newline="")
    for single in (False, True):
        out = tmp_path / f"out{int(single)}"
        nn_classification.main(fa, out, single, 16, False, 2, False, True)
        z = np.load(_paths.NNOutputs("mixed", out).nn_classification_npz_output)
        names, ids, ascii_arr, tok = T.encode_fasta(fa, single_window=single)
        ref = T.segment_mean(_oracle_probs(tok, shipped), ids, len(names))
        assert list(z["contig_names"]) == list(names) and "all_n" not in list(names)
        assert np.abs(z["predictions"] - ref).max() <= TOL
        assert np.array_equal(z["predictions"].argmax(1), ref.argmax(1))
        assert not _paths.NNOutputs("mixed", out).encoded_sequences_dir.exists()      # --cleanup


@pytest.mark.gpu
def test_module_tfrecord_intermediates_and_aggregation(tmp_path, shipped, monkeypatch):
    """SURVEY §8f ranks 3-4 end to end on the GPU: with GENOMAD_B200_TFRECORDS=1 the encoded directory holds the
    reference's <cumulative count>.tfrec files (tokens bit-exact vs the oracle tokenizer, classifying them through
    gnm_forward_tokens reproduces the module's NPZ), and aggregated-classification consumes the module's NPZ."""
    import torch
    from genomad_b200 import nn_classification, aggregated_classification as agg, tfrecord, _paths, utils
    from genomad_b200.engine import Classifier
    monkeypatch.setenv("GENOMAD_B200_TFRECORDS", "1")
    monkeypatch.setattr(tfrecord, "RECORDS_PER_FILE", 7)          # several files from a small input
    rng = np.random.default_rng(3)
    lens = [30000, 9000, 2000, 48000]
    fa = tmp_path / "toy.fna"
    with open(fa, "w") as f:
        for i, ln in enumerate(lens):
            f.write(f">c{i}\n" + np.frombuffer(b"ACGTN", np.uint8)[rng.choice(5, ln, p=[.245, .245, .245, .245, .02])].tobytes().decode() + "\n")
    out = tmp_path / "out"
    nn_classification.main(fa, out, False, 8, False, 2, False, False)
    o = _paths.AggregatedOutputs("toy", out)
    names, ids, ascii_arr, tok = T.encode_fasta(fa)
    files = tfrecord.tfrecord_files(o.encoded_sequences_dir)
    n = len(tok)
    assert [int(p.stem) for p in files] == list(range(7, n, 7)) + [n]
    back = np.concatenate([tfrecord.read_tfrecord(p) for p in files])
    assert np.array_equal(back, tok.astype(np.uint16))
    clf = Classifier(max_batch=8)
    probs = clf.predict_tokens(torch.from_numpy(back).cuda()).cpu().numpy()
    z = np.load(o.nn_classification_npz_output)
    assert np.abs(T.segment_mean(probs, ids, len(names)) - z["predictions"]).max() <= 1e-6
    # downstream consumer: synthetic marker branch + this run's NPZ
    o.marker_classification_dir.mkdir()
    utils.write_execution_info("marker_classification", fa, {}, o.marker_classification_execution_info)
    feats = rng.random((len(names), 25)).astype(np.float32)
    mk = rng.random((len(names), 3)).astype(np.float32)
    np.savez_compressed(o.features_npz_output, contig_names=names, contig_features=feats)
    np.savez_compressed(o.marker_classification_npz_output, contig_names=names, predictions=mk)
    agg.main(fa, out, False, False)
    a = np.load(o.aggregated_classification_npz_output)
    assert list(a["contig_names"]) == list(names)
    assert np.array_equal(a["predictions"], agg.branch_attention(feats[:, 15:18].sum(1), mk, z["predictions"]))


@pytest.mark.gpu
def test_fused_layer1_wv_option(shipped):
    """Option fuse_l1=1 (layer 1 + w_v#0 in one wgmma kernel whose B operand is written by SIMT producers in the TMA
    swizzle layout) must reproduce the two separate kernels bit for bit: y1, q0 and the final probabilities, from ASCII
    and from tokens, incl. N-rich / padded windows and a batch that leaves the last unit of every window partial."""
    import torch
    from genomad_b200.engine import Classifier
    rng = np.random.default_rng(21)
    n = 9
    a = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, (n, 6000))].copy()
    a[1, 100:400] = ord("N"); a[2, 3000:] = ord("N"); a[3, :] = ord("N"); a[4, ::7] = ord("R")
    at = torch.from_numpy(a).cuda()
    clf = Classifier(max_batch=16)
    tok = clf.encode(at)
    res = {}
    for f in (0, 1):
        clf.set_option("fuse_l1", f)
        n0 = clf.kernel_launches
        p_ascii = clf.predict_ascii(at).cpu().numpy()
        assert clf.kernel_launches - n0 == (19 if f else 18)
        y1 = None
        clf.set_option("debug_stop", 1)
        clf.predict_ascii(at)
        y1 = clf.debug_fetch("buf0", n).cpu().numpy()
        q0 = clf.debug_fetch("q0", n).cpu().numpy()
        clf.set_option("debug_stop", 0)
        p_tok = clf.predict_tokens(tok).cpu().numpy()
        res[f] = (p_ascii, p_tok, y1, q0)
    for x, y in zip(res[0], res[1]):
        assert np.array_equal(x, y)
    assert np.array_equal(res[1][0], res[1][1])


# ------------------------------------------------------------------------------------------ BASELINE config 2 parity clause
def test_config2_subsample_batch1024_vs_oracle(golden_dir, shipped):
    """BASELINE.md config 2: "per-window probs vs oracle on a fixed 2,048-window subsample", batch 1024.  The 2,048 windows
    (counter-based stream of genomad_b200/synth.py, seed 1, incl. >= 32 windows of the N-run / IUPAC sub-stream) go through a
    max_batch = 1024 handle in two steps; the oracle's fp32 outputs are the committed fixture
    (tests/golden/make_config2_golden.py), re-derived live for a 48-window slice so a stale fixture cannot pass."""
    from genomad_b200 import engine, synth
    g = np.load(golden_dir / "config2_subsample.npz")
    idx = g["indices"]
    a = synth.windows_numpy(idx, seed=1)
    assert len(idx) == 2048 and int((a == ord("N")).any(1).sum()) == int(g["n_dirty"]) >= 32
    # the device generator bench.py uses is the same function of (seed, index)
    dev0 = synth.windows_torch(int(idx[5]), 3, 1, "cuda").cpu().numpy()
    assert np.array_equal(dev0, synth.windows_numpy(np.arange(idx[5], idx[5] + 3), seed=1))
    c = engine.Classifier(None, device=0, max_batch=1024)
    try:
        p = c.predict_ascii(torch.from_numpy(a).cuda()).cpu().numpy()
        p_host = c.classify_host(a)
    finally:
        c.close()
    ref = g["shipped_fp32"]
    d = np.abs(p - ref)
    assert d.max() <= TOL, d.max()
    assert np.array_equal(p.argmax(1), ref.argmax(1))
    assert np.array_equal(p_host, p)
    sl = slice(1000, 1048)
    live = _oracle_probs(T.tokenize_windows(a[sl]), shipped)
    assert np.abs(live - ref[sl]).max() <= 5e-6             # the fixture IS the oracle (fp32: reproducible to re-association level across hosts)
    print(f"config-2 subsample: max |dp| = {d.max():.2e}, mean = {d.mean():.2e}")


def test_live_igloo_weights_320_windows_vs_oracle(golden_dir, shipped):
    """>= 256 windows with synthetic O(1) patch / attention weights (the only inputs where the patch gather, the 3xTF32 logits
    GEMM and the softmax are numerically alive), batch 1024 handle, against the oracle fixture (fp32 and fp64)."""
    import sys
    from genomad_b200 import engine, synth
    g = np.load(golden_dir / "config2_subsample.npz")
    a = np.concatenate([synth.windows_numpy(g["syn_indices"], seed=1), _families(64, seed=int(g["syn_family_seed"]))])
    assert len(a) == 320
    c = engine.Classifier(M.synthetic_igloo_weights(shipped), device=0, max_batch=1024)
    try:
        p = c.predict_ascii(torch.from_numpy(a).cuda()).cpu().numpy()
    finally:
        c.close()
    d32, d64 = np.abs(p - g["synthetic_fp32"]), np.abs(p - g["synthetic_fp64"])
    assert d32.max() <= TOL and d64.max() <= TOL, (d32.max(), d64.max())
    assert np.array_equal(p.argmax(1), g["synthetic_fp64"].argmax(1))
    live = _oracle_probs(T.tokenize_windows(a[300:316]), M.synthetic_igloo_weights(shipped))
    assert np.abs(live - g["synthetic_fp32"][300:316]).max() <= 5e-6      # fp32 oracle: host-dependent summation order
    print(f"live IGLOO weights: max |dp| vs fp32 oracle = {d32.max():.2e}, vs fp64 = {d64.max():.2e}")


# ------------------------------------------------------------------------------------------ provirus twin + skip / restart on the GPU
def test_module_provirus_twin_skip_and_restart(tmp_path, shipped):
    """SURVEY 8(f) rank 2 with the REAL classifier: the provirus twin (reference nn_classification.py:248-281, 355-425),
    the skip rules (:176-197, :215-225, :284-292), --restart, and a parameter change, each against the oracle pipeline."""
    import time as _time
    from genomad_b200 import nn_classification, _paths, utils
    rng = np.random.default_rng(5)

    def seq(n):
        return np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)].tobytes().decode()

    fa = tmp_path / "meta.fna"
    with open(fa, "w") as fh:
        for i, ln in enumerate([30000, 7000, 2400, 13000]):
            s = seq(ln)
            fh.write(f">ctg_{i} x\n" + "\n".join(s[k:k + 80] for k in range(0, ln, 80)) + "\n")
    out = tmp_path / "out"
    out.mkdir()
    o = _paths.NNOutputs("meta", out)
    # a finished find-proviruses run on the same input with three proviruses (15 kb -> 3 windows, 3 kb, 9 kb)
    o.find_proviruses_dir.mkdir()
    utils.write_execution_info("find_proviruses", fa, {}, o.find_proviruses_execution_info)
    pv = {"ctg_0|provirus_1001_16000": seq(15000), "ctg_0|provirus_20001_23000": seq(3000), "ctg_3|provirus_1_9000": seq(9000)}
    o.find_proviruses_output.write_text("seq_name\tx\n" + "".join(f"{k}\t1\n" for k in pv))
    o.find_proviruses_nucleotide_output.write_text("".join(f">{k}\n{v}\n" for k, v in pv.items()))
    o.find_proviruses_proteins_output.write_text("")
    o.find_proviruses_genes_output.write_text("")

    def oracle_for(path, single):
        names, ids, _, tok = T.encode_fasta(path, single_window=single)
        return list(names), T.segment_mean(_oracle_probs(tok, shipped), ids, len(names))

    def check(single):
        for path, npz, key, tsv in ((fa, o.nn_classification_npz_output, "contig_names", o.nn_classification_output),
                                    (o.find_proviruses_nucleotide_output, o.provirus_nn_classification_npz_output,
                                     "provirus_names", o.provirus_nn_classification_output)):
            names, ref = oracle_for(path, single)
            z = np.load(npz)
            assert list(z[key]) == names and z["predictions"].dtype == np.float32
            assert np.abs(z["predictions"] - ref).max() <= TOL
            assert np.array_equal(z["predictions"].argmax(1), ref.argmax(1))
            lines = tsv.read_text().splitlines()
            assert lines[0] == "seq_name\tchromosome_score\tplasmid_score\tvirus_score" and len(lines) == len(names) + 1
            for line, name, row in zip(lines[1:], names, z["predictions"]):
                assert line == f"{name}\t" + "\t".join(f"{x:.4f}" for x in row)

    def mtimes():
        return {p.name: p.stat().st_mtime_ns for p in (o.nn_classification_npz_output, o.provirus_nn_classification_npz_output,
                                                       o.seq_window_id_output, o.provirus_window_id_output)}

    nn_classification.main(fa, out, False, 128, False, 2, False, False)
    check(False)
    ids = np.load(o.provirus_window_id_output)
    assert set(ids.files) == {"provirus_names", "provirus_ids"} and ids["provirus_ids"].tolist() == [0, 0, 0, 1, 2, 2]
    m0 = mtimes()
    # 2nd run, same input and parameters: every step is skipped, nothing is rewritten
    _time.sleep(0.02)
    nn_classification.main(fa, out, False, 128, False, 2, False, False)
    log = o.nn_classification_log.read_text()
    assert "Previous execution detected" in log and "Skipping sequence classification" in log
    assert "Skipping provirus classification" in log and "Skipping provirus encoding" in log
    assert mtimes() == m0
    check(False)
    # provirus NPZ lost: only the provirus classification is redone
    o.provirus_nn_classification_npz_output.unlink()
    nn_classification.main(fa, out, False, 128, False, 2, False, False)
    log = o.nn_classification_log.read_text()
    assert "Skipping sequence classification" in log and "Skipping provirus classification" not in log
    m1 = mtimes()
    assert m1["meta_nn_classification.npz"] == m0["meta_nn_classification.npz"]
    check(False)
    # --restart: everything again
    _time.sleep(0.02)
    nn_classification.main(fa, out, False, 128, True, 2, False, False)
    assert "Previous execution detected" not in o.nn_classification_log.read_text()
    m2 = mtimes()
    assert all(m2[k] > m1[k] for k in m2)
    check(False)
    # parameter change (--single-window): previous outputs are overwritten, one window per sequence / provirus
    nn_classification.main(fa, out, True, 128, False, 2, False, True)
    assert "parameters changed" in o.nn_classification_log.read_text()
    check(True)
    assert not o.encoded_sequences_dir.exists() and not o.encoded_proviruses_dir.exists()      # --cleanup


def test_activation_range_overflow_is_reported(shipped):
    """The C ABI accepts arbitrary weights, but the split-operand recipe carries activations in fp16 + e4m3 planes scaled for
    |y| <= 3.5 (csrc/common.cuh).  Weights that exceed the range must not degrade silently: the producing kernel raises
    DeviceStatus::act_overflow and the library fails loudly (gnm_check_status / the next call / gnm_classify_host)."""
    from genomad_b200 import engine
    a = _families(8, seed=3)
    w = dict(shipped)
    w["c1w"] = (shipped["c1w"] * 12).astype(np.float32)          # |y1| reaches ~6 > 3.5: hi8 plane saturates
    c = engine.Classifier(w, device=0, max_batch=8)
    try:
        c.predict_ascii(torch.from_numpy(a).cuda())
        with pytest.raises(engine.GnmError, match="activation range exceeded in layer 1"):
            c.check_status()
        c.check_status()                                          # the flag is cleared once reported
        with pytest.raises(engine.GnmError, match="activation range"):
            c.classify_host(a)
    finally:
        c.close()
    ok = engine.Classifier(shipped, device=0, max_batch=8)        # the shipped model is far inside the range
    try:
        ok.predict_ascii(torch.from_numpy(a).cuda())
        ok.check_status()
    finally:
        ok.close()


def test_fused_wv_gather_vs_separate_kernels(shipped):
    """Round 2: the IGLOO value projection and the patch gather share one pass over the activations (csrc/wv_gather.cuh,
    band-major units of 24 positions x 8 windows; gather on warp-level mma with fp16 hi / lo operand halves).  Against the round-1
    pair (conv_t_kernel<true> + patch_stream_kernel, option fuse_gather=0): q is bitwise identical (same MMA sequence per output),
    mpi agrees to fp32 re-association level,
    probabilities to 1e-6 -- with live (synthetic) IGLOO weights, batches that are not multiples of 8 and a batch of 1."""
    from genomad_b200.engine import Classifier
    w = M.synthetic_igloo_weights(shipped)
    a = _families(45, seed=17)
    clf = Classifier(w, device=0, max_batch=45)
    try:
        for n in (45, 8, 1, 19):
            at = torch.from_numpy(a[:n]).cuda()
            res = {}
            for f in (1, 0):
                clf.set_option("fuse_gather", f)
                pr = clf.predict_ascii(at).cpu().numpy()
                res[f] = (pr, clf.debug_fetch("q0", n).cpu().numpy(), clf.debug_fetch("q1", n).cpu().numpy(),
                          clf.debug_fetch("mpi0", n).cpu().numpy(), clf.debug_fetch("mpi1", n).cpu().numpy())
            clf.check_status()
            assert np.array_equal(res[0][1], res[1][1]) and np.array_equal(res[0][2], res[1][2]), n
            for k in (3, 4):
                scale = np.abs(res[0][k]).max()
                assert np.abs(res[0][k] - res[1][k]).max() <= 2e-6 * scale, (n, k)
            assert np.abs(res[0][0] - res[1][0]).max() <= 5e-6, n
    finally:
        clf.close()


def test_tail_overlap_is_invisible(shipped):
    """Multi-step calls run each step's tail (logits / attention / dense head) on a second stream next to the following step's
    main part, alternating two buffer sets.  The result must be bitwise what the strictly ordered execution gives -- device
    entry point and host entry point, batch counts that end on either buffer set, live IGLOO weights."""
    from genomad_b200.engine import Classifier
    a = _families(7 * 16 + 5, seed=23)                                     # 8 internal steps of 16, the last one partial
    clf = Classifier(M.synthetic_igloo_weights(shipped), device=0, max_batch=16)
    try:
        at = torch.from_numpy(a).cuda()
        res = {}
        for ov in (1, 0):
            clf.set_option("tail_overlap", ov)
            p_dev = clf.predict_ascii(at).cpu().numpy()
            p_dev2 = clf.predict_ascii(at[:48]).cpu().numpy()              # 3 steps: ends on the other buffer set
            p_host = clf.classify_host(a)
            clf.check_status()
            res[ov] = (p_dev, p_dev2, p_host)
        for x, y in zip(res[0], res[1]):
            assert np.array_equal(x, y)
        assert np.array_equal(res[1][0], res[1][2]) and np.array_equal(res[1][0][:48], res[1][1])
        one = np.concatenate([clf.predict_ascii(at[i:i + 16]).cpu().numpy() for i in range(0, len(a), 16)])
        assert np.array_equal(one, res[1][0])                              # single-step calls (never overlapped) agree too
    finally:
        clf.close()


def test_adversarial_patch_sets(shipped):
    """The C ABI accepts any patch indices in [0, 5997).  Two extreme sets against the oracle: (a) every patch reads the same four
    positions at the two ends of the window (two position bands of the fused IGLOO kernel hold all 8,400 entries: its generic
    path, the cost-balanced CTA split and the finish kernel at their worst), (b) every patch reads one position four times."""
    from genomad_b200 import engine
    base = M.synthetic_igloo_weights(shipped, seed=11)
    a = _families(11, seed=41)
    tok = T.tokenize_windows(a)
    for name, rows in (("ends", [0, 1, 5995, 5996]), ("one position x4", [3001, 3001, 3001, 3001])):
        w = dict(base)
        for s in (0, 1):
            w[f"ig{s}_random_patches"] = np.tile(np.asarray(rows, np.int32).reshape(1, 4, 1), (2100, 1, 1))
        ref = _oracle_probs(tok, w)
        c = engine.Classifier(w, device=0, max_batch=16)
        try:
            p = c.predict_ascii(torch.from_numpy(a).cuda()).cpu().numpy()
            c.check_status()
        finally:
            c.close()
        assert np.abs(p - ref).max() <= TOL, (name, np.abs(p - ref).max())
        assert np.array_equal(p.argmax(1), ref.argmax(1)), name


# ------------------------------------------------------------------------------------------ vectors of the reference's own model code
def test_cuda_vs_reference_graph_golden(golden_dir, clf, clf_syn):
    """The CUDA path against vectors of the REFERENCE'S OWN model definition (genomad/neural_network/{model,igloo}.py executed on
    the NumPy stand-in tests/golden/keras_shim.py, fp64; generator tests/golden/make_reference_graph_golden.py) -- not via the
    oracle: 24 windows (N / IUPAC windows and the worst-case families included), shipped weights and synthetic O(1) IGLOO weights."""
    g = np.load(golden_dir / "reference_graph_golden.npz")
    a = torch.from_numpy(g["windows"]).cuda()
    for key, c in (("shipped", clf), ("synthetic", clf_syn)):
        p = c.predict_ascii(a).cpu().numpy()
        ref = g[key + "_fp64"]
        d = np.abs(p - ref).max()
        assert d <= TOL, (key, d)
        assert np.array_equal(p.argmax(1), ref.argmax(1)), key
        print(f"CUDA vs reference graph ({key} weights): max |dp| = {d:.2e}")
