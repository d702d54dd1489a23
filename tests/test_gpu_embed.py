"""
Encoder embeddings on the H100 (run with `-m gpu -s` for the measured precision): gnm_embed_* against fp64 (tests/encoder_ref.py and the
reference encoder's golden outputs), the bitwise identities between the entry points and with the plain forward calls, 64-bit
row offsets past 2^31 bytes, gnm_segment_sum_rows and its carry, classify_contigs(return_embeddings=True) and the module's
--write-embeddings outputs.
"""
import json
import shutil
import time
from pathlib import Path

import numpy as np
import pytest
import torch

from genomad_b200 import dist as gdist, engine, synth
from oracle import igloo_model as M
import encoder_ref as E
from oracle import tokenizer as T
from test_dist_gloo_embed import np_segment_sum_rows

pytestmark = pytest.mark.gpu

MB = 16
DEFAULTS = {"conv_impl": 0, "fuse_l1": 0, "fuse_gather": 1, "tail_overlap": 1}


@pytest.fixture(scope="module", autouse=True)
def _report_cost():
    t0 = time.time()
    yield
    print(f"\n{Path(__file__).name}: {time.time() - t0:.0f} s; peak torch allocation {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


@pytest.fixture(scope="module")
def enc_gold(golden_dir):
    return np.load(golden_dir / "reference_encoder_golden.npz")


@pytest.fixture(scope="module")
def shipped(weights_npz):
    return M.load_npz_weights(weights_npz)


@pytest.fixture(scope="module")
def weights(shipped):
    return {"shipped": shipped, "synthetic": M.synthetic_igloo_weights(shipped)}


def _cuda_tokens(tok):
    return torch.from_numpy(np.ascontiguousarray(tok, dtype=np.uint16).view(np.int16)).cuda().view(torch.uint16)


def _set(c, opts):
    for k, v in {**DEFAULTS, **opts}.items():
        c.set_option(k, v)


def _worst(e_gpu, e64):
    """max over windows of max_j |e_gpu - e64| / max(1, max_j |e64|): the bar is 1e-4."""
    err = np.abs(e_gpu.astype(np.float64) - e64).max(axis=1)
    return float((err / np.maximum(1.0, np.abs(e64).max(axis=1))).max())


# ------------------------------------------------------------------------------------------ precision
@pytest.mark.parametrize("variant", ["shipped", "synthetic"])
def test_embeddings_within_1e4_of_fp64(enc_gold, weights, golden_dir, variant):
    w = weights[variant]
    c = engine.Classifier(w, device=0, max_batch=MB)
    try:
        for inputs in ("graph", "tokens"):
            tok = enc_gold[f"{inputs}_tokens"]
            ref = enc_gold[f"{inputs}_{variant}_fp64"]
            orc = E.encoder(tok, w, torch.float64)
            for path, opts in {"default": {}, "fuse_l1": {"fuse_l1": 1}, "tail_overlap=0": {"tail_overlap": 0},
                               "fuse_gather=0": {"fuse_gather": 0}, "conv_impl=1": {"conv_impl": 1}}.items():
                _set(c, opts)
                probs, emb = c.embed_tokens(_cuda_tokens(tok))
                e = emb.cpu().numpy()
                wg, wo = _worst(e, ref), _worst(e, orc)
                print(f"\nembeddings {variant:9s} {inputs:6s} ({len(tok)} windows, {path:14s}): worst max_j|de| / max(1, max_j|e|) "
                      f"vs reference encoder fp64 {wg:.2e}, vs encoder_ref fp64 {wo:.2e}; exact zeros {np.mean(e == 0):.0%}")
                assert wg <= 1e-4 and wo <= 1e-4, (variant, inputs, path, wg, wo)
                if path == "default":
                    assert torch.equal(probs, c.predict_tokens(_cuda_tokens(tok)))
        g = np.load(golden_dir / "reference_graph_golden.npz")
        _set(c, {})
        _, emb = c.embed_ascii(torch.from_numpy(g["windows"]).cuda())
        assert _worst(emb.cpu().numpy(), enc_gold[f"graph_{variant}_fp64"]) <= 1e-4
    finally:
        c.close()


# ------------------------------------------------------------------------------------------ bitwise identities
@pytest.fixture(scope="module")
def batch():
    idx = synth.subsample_indices(2 * MB + 8, 1_000_000, seed=3)
    a = synth.windows_numpy(idx, seed=3)
    a[5, 3000:] = ord("N")                                          # a padded tail window
    return a


def test_entry_points_agree_bitwise(weights, batch):
    c = engine.Classifier(weights["synthetic"], device=0, max_batch=MB)
    try:
        n = batch.shape[0]
        a = torch.from_numpy(batch).cuda()
        launches = c.kernel_launches
        p_ref = c.predict_ascii(a[:MB])
        assert c.kernel_launches - launches == 18                   # the plain forward path is unchanged
        p_ascii, e_ascii = c.embed_ascii(a)
        torch.cuda.synchronize()
        assert torch.equal(e_ascii[n - 8:], c.debug_fetch("h1", 8))     # the last step's h1
        assert torch.equal(p_ascii, c.predict_ascii(a))
        assert torch.equal(p_ascii[:MB], p_ref)
        p_tok, e_tok = c.embed_tokens(c.encode(a))
        assert torch.equal(e_tok, e_ascii) and torch.equal(p_tok, c.predict_tokens(c.encode(a)))
        # windows straight from a sequence buffer: the batch as one contig of back-to-back windows
        seq = a.reshape(-1)
        start = torch.arange(n, dtype=torch.int64, device="cuda") * 6000
        length = torch.full((n,), 6000, dtype=torch.int32, device="cuda")
        p_win, e_win = c.embed_windows(seq, start, length)
        assert torch.equal(e_win, e_ascii) and torch.equal(p_win, c.predict_windows(seq, start, length))
        # host path: probabilities to the host, embeddings on the device
        host = np.ascontiguousarray(batch)
        h_probs = np.empty((n, 3), np.float32)
        d_emb = torch.empty((n, 512), dtype=torch.float32, device="cuda")
        c.embed_host_into(host.ctypes.data, n, h_probs.ctypes.data, d_emb.data_ptr())
        assert torch.equal(d_emb, e_ascii) and np.array_equal(h_probs, c.classify_host(host))
        d_emb2 = torch.zeros_like(d_emb)
        c.embed_host_into(host.ctypes.data, n, 0, d_emb2.data_ptr())      # probabilities not wanted
        assert torch.equal(d_emb2, e_ascii)
        # one multi-step call = one-step calls on the same rows; tail_overlap changes nothing
        steps = torch.cat([c.embed_ascii(a[i:i + MB])[1] for i in range(0, n, MB)])
        assert torch.equal(steps, e_ascii)
        _set(c, {"tail_overlap": 0})
        p, e = c.embed_ascii(a)
        assert torch.equal(e, e_ascii) and torch.equal(p, p_ascii)
        # fuse_l1 = 1 runs the IGLOO patch gather as the separate pair of kernels (mpi is summed in another order, DESIGN §4), so
        # it is bitwise the fuse_gather = 0 path, not the default one (both within 1e-4 of fp64: test above)
        for tail in (1, 0):
            _set(c, {"fuse_gather": 0, "tail_overlap": tail})
            p0, e0 = c.embed_ascii(a)
            _set(c, {"fuse_l1": 1, "tail_overlap": tail})
            p1, e1 = c.embed_ascii(a)
            assert torch.equal(e1, e0) and torch.equal(p1, p0) and torch.equal(p1, c.predict_ascii(a))
        _set(c, {})
    finally:
        c.close()


def test_batch_position_does_not_change_the_embedding(weights, batch):
    c = engine.Classifier(weights["synthetic"], device=0, max_batch=1024)
    try:
        big = np.concatenate([synth.windows_numpy(synth.subsample_indices(1023, 1_000_000, seed=4), seed=4), batch[:1]])
        _, e_big = c.embed_ascii(torch.from_numpy(big).cuda())
        _, e_one = c.embed_ascii(torch.from_numpy(batch[:1]).cuda())
        assert torch.equal(e_big[1023], e_one[0])
    finally:
        c.close()


def test_row_offsets_past_2gb(weights):
    """1,048,600 windows whose starts all point into a 1 MB sequence: the embedding rows cross 2^31 bytes at row 1,048,576."""
    n = 1_048_600
    c = engine.Classifier(weights["shipped"], device=0, max_batch=1024)
    try:
        rng = np.random.default_rng(9)
        seq = torch.from_numpy(np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 1 << 20)].copy()).cuda()
        start = torch.from_numpy(rng.integers(0, (1 << 20) - 6000, n).astype(np.int64)).cuda()
        length = torch.from_numpy(rng.integers(1, 6001, n).astype(np.int32)).cuda()
        probs, emb = c.embed_windows(seq, start, length)
        torch.cuda.synchronize()
        tail = slice(n - 40, n)                                        # rows before and after byte offset 2^31
        p_small, e_small = c.embed_windows(seq, start[tail], length[tail])
        assert torch.equal(emb[tail], e_small) and torch.equal(probs[tail], p_small)
        assert emb[tail].abs().sum() > 0
        del emb, probs
    finally:
        c.close()


# ------------------------------------------------------------------------------------------ segment sums
def _rows(n, seed=0):
    rng = np.random.default_rng(seed)
    r = (rng.standard_normal((n, 512)) * 3).astype(np.float32)
    r[r < 0] = 0
    return r


def test_segment_sum_rows_chunked_equals_one_call_and_numpy(weights):
    c = engine.Classifier(weights["shipped"], device=0, max_batch=8)
    try:
        counts = [3, 0, 250, 1, 1, 0, 700, 17, 5, 1024, 2]
        offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        rows = _rows(int(offsets[-1]))
        d_rows = torch.from_numpy(rows).cuda()
        d_off = torch.from_numpy(offsets.astype(np.int32)).cuda()
        sums, carry = c.segment_sum_rows(d_rows, d_off)
        ref, ref_carry = np_segment_sum_rows(rows, offsets)
        assert np.array_equal(sums.cpu().numpy(), ref) and np.array_equal(carry.cpu().numpy(), ref_carry)
        one_means = sums / torch.from_numpy(np.maximum(np.diff(offsets), 1).astype(np.float32)).cuda()[:, None]
        for chunk in (1, 7, 100, 999, 4096):
            sh = gdist.EmbeddingShard(offsets, 0, int(offsets[-1]), c.segment_sum_rows, device="cuda")
            for a in range(0, int(offsets[-1]), chunk):
                sh.add(d_rows[a: a + chunk])
            lo, means = sh.finish(gdist.DistInfo())
            assert lo == 0 and torch.equal(means, one_means), chunk
        # the raw carry: split inside segment 2 and chain
        s1, k1 = c.segment_sum_rows(d_rows[:100], torch.tensor([0, 3, 3, 100], dtype=torch.int32, device="cuda"))
        s2, _ = c.segment_sum_rows(d_rows[100:], (d_off[2:] - 100).clamp(min=0), k1)
        assert torch.equal(s2[0], sums[2]) and torch.equal(s2[1:], sums[3:]) and torch.equal(s1[:2], sums[:2])
        # in place: the carry buffer may be both input and output
        buf = k1.clone()
        seg = torch.tensor([0, 153], dtype=torch.int32, device="cuda")           # the rest of segment 2
        out = torch.empty(512, device="cuda")
        assert c.lib.gnm_segment_sum_rows(c._h, d_rows[100:].data_ptr(), seg.data_ptr(), 1, buf.data_ptr(), out.data_ptr(),
                                          buf.data_ptr(), c._stream()) == 0
        torch.cuda.synchronize()
        assert torch.equal(buf, sums[2])
    finally:
        c.close()


def test_classify_contigs_returns_mean_embeddings(weights):
    c = engine.Classifier(weights["shipped"], device=0, max_batch=MB)
    try:
        rng = np.random.default_rng(11)
        seqs = [np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, ln)].tobytes() for ln in (30000, 500, 14000)]
        seqs.insert(1, b"N" * 7000)                                   # empty after stripping: no windows
        means, counts = c.classify_contigs(seqs)
        m2, c2, probs, emb = c.classify_contigs(seqs, return_window_probs=True, return_embeddings=True)
        assert torch.equal(m2, means) and torch.equal(c2, counts)
        seq, offs = c.contig_buffers(seqs)
        start, length, woff = c.contig_windows(seq, offs)
        p_w, e_w = c.embed_windows(seq, start, length)
        assert torch.equal(probs, p_w)
        sums, _ = c.segment_sum_rows(e_w, woff)
        assert torch.equal(emb, sums / counts.clamp(min=1).to(torch.float32)[:, None])
        assert counts[1].item() == 0 and not emb[1].any() and emb.shape == (4, 512)
        m3, c3, e3 = c.classify_contigs(seqs, return_embeddings=True)
        assert torch.equal(e3, emb)
    finally:
        c.close()


# ------------------------------------------------------------------------------------------ module
def _working_copy(src, dst):
    shutil.copytree(src, dst)
    for p in [dst, *dst.rglob("*")]:
        p.chmod(p.stat().st_mode | 0o200)


def test_module_write_embeddings(tmp_path, golden_dir):
    from genomad_b200 import _paths, nn_classification, sequence
    inp = golden_dir / "reference_module" / "input"
    runs = {}
    for flag in (False, True):
        work = tmp_path / f"run_{int(flag)}"
        work.mkdir()
        fa = work / "toy.fna"
        shutil.copy(inp / "toy.fna", fa)
        _working_copy(inp / "toy_find_proviruses", work / "out" / "toy_find_proviruses")
        nn_classification.main(fa, work / "out", False, 128, False, 2, False, False, write_embeddings=flag)
        runs[flag] = (fa, _paths.NNOutputs("toy", work / "out"))
    (_, off), (fa, on) = runs[False], runs[True]
    for attr in ("nn_classification_output", "nn_classification_npz_output", "provirus_nn_classification_output",
                 "provirus_nn_classification_npz_output"):
        assert getattr(off, attr).read_bytes() == getattr(on, attr).read_bytes(), attr
    j_off, j_on = (json.loads(o.nn_classification_execution_info.read_text()) for o in (off, on))
    j_off.pop("start_time"), j_on.pop("start_time")
    assert j_off == j_on
    assert not off.nn_classification_embeddings_output.exists()
    # contents: the mean of the windows' encoder outputs, per contig, in the predictions' order
    clf = nn_classification._make_classifier(128, 0)
    for src, npz, emb_npz, key in ((fa, on.nn_classification_npz_output, on.nn_classification_embeddings_output, "contig_names"),
                                   (on.find_proviruses_nucleotide_output, on.provirus_nn_classification_npz_output,
                                    on.provirus_nn_classification_embeddings_output, "provirus_names")):
        z, e = np.load(npz), np.load(emb_npz)
        assert set(e.files) == {key, "embeddings"} and e["embeddings"].dtype == np.float32
        assert list(e[key]) == list(z[key]) and e["embeddings"].shape == (len(z[key]), 512)
        pf = sequence.ParsedFasta(src)
        idx = pf.index()
        win = pf.export_windows(0, pf.n_windows, np.zeros((pf.n_windows, 6000), np.uint8))
        _, d_emb = clf.embed_ascii(torch.from_numpy(np.ascontiguousarray(win)).cuda())
        sums, _ = clf.segment_sum_rows(d_emb, torch.from_numpy(idx.offsets.astype(np.int32)).cuda())
        cnt = torch.from_numpy(np.diff(idx.offsets).astype(np.float32)).cuda()
        assert np.array_equal(e["embeddings"], (sums / cnt[:, None]).cpu().numpy())
        pf.close()
    # a lost embeddings file is regenerated without --restart, the predictions bit for bit as before
    before = on.nn_classification_npz_output.read_bytes()
    ref = np.load(on.nn_classification_embeddings_output)["embeddings"]
    on.nn_classification_embeddings_output.unlink()
    nn_classification.main(fa, on.output_dir, False, 128, False, 2, False, False, write_embeddings=True)
    assert np.array_equal(np.load(on.nn_classification_embeddings_output)["embeddings"], ref)
    assert on.nn_classification_npz_output.read_bytes() == before
    log = on.nn_classification_log.read_text()
    assert "Skipping provirus classification" in log and "Skipping sequence classification" not in log
