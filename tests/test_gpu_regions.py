"""
GPU tests of the window-region decode (run with `-m gpu` on an H100): gnm_window_regions through engine.window_regions against
the fp64 oracle (tests/regions_ref.py) on seeded profiles with planted class segments and Dirichlet noise, at C = 2, 3, 5 and
32, sequences of 1, 2, ~100 and 100,000 windows, N-rule gaps, scores of exactly 0 and 1, strides 1 to 6000 and L = 12,000 and
1e9.  Checked: posteriors within 1e-6; the path equal to the oracle's wherever the max-marginal margin exceeds
1e-9 (1 + |best score|); the path's fp64 score within 1e-9 (relative) of the optimum; the region table equal to the oracle's
table built from the GPU path; bitwise independence of sequence order and chunking; and window-regions end to end on the
module's window files, the shipped classes and a seeded head, bitwise the in-memory API.
"""
from pathlib import Path

import numpy as np
import pytest

import regions_ref as R
from genomad_b200 import _paths, engine, nn_classification as nnc, sequence, weights as W
from genomad_b200 import window_regions as WR

pytestmark = pytest.mark.gpu

TOY = Path(__file__).resolve().parent / "golden" / "reference_module" / "input" / "toy.fna"


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch


def planted(rng, sizes, C, stride, extremes=True):
    """Profiles of planted class segments (mean length ~40 windows) under Dirichlet noise; some windows are dropped (N-rule
    gaps of 2..4 strides) and, with extremes, some rows are exactly one-hot (scores 0 and 1)."""
    probs, start, length, offsets = [], [], [], [0]
    for n in sizes:
        if n:
            seg = np.cumsum(rng.random(n) < 1 / 40)
            cls = rng.integers(0, C, seg[-1] + 1)[seg]
            noise = rng.dirichlet(np.full(C, 0.7), n)
            p = 0.45 * np.eye(C)[cls] + 0.55 * noise
            if extremes:
                hot = rng.random(n) < 0.05
                p[hot] = np.eye(C)[rng.integers(0, C, hot.sum())]
            step = np.where(rng.random(n - 1) < 0.05, rng.integers(2, 5, n - 1), 1)
            st = np.concatenate([[0], np.cumsum(step)]) * stride + int(rng.integers(0, 3000))
            ln = np.full(n, 6000, np.int64)
            ln[-1] = int(rng.integers(1, 6001))
            probs.append(p)
            start.append(st)
            length.append(ln)
        offsets.append(offsets[-1] + n)
    return (np.concatenate(probs).astype(np.float32), np.array(offsets, np.int64), np.concatenate(start).astype(np.int64),
            np.concatenate(length).astype(np.int32))


def to_ws(torch, probs, offsets, start, length):
    d = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()
    contig = np.repeat(np.arange(len(offsets) - 1, dtype=np.int32), np.diff(offsets))
    return engine.WindowScores(d(probs, np.float32), d(contig, np.int32), d(start, np.int64), d(length, np.int32),
                               d(offsets, np.int32))


def host(res):
    return {k: v.cpu().numpy() for k, v in res._asdict().items()}


def check_against_oracle(probs, offsets, start, length, stride, L, got):
    C = probs.shape[1]
    ref = R.decode(probs, offsets, start, length, stride, L)
    assert np.abs(got["posterior"] - ref["posterior"]).max() <= 1e-6
    for s in range(len(offsets) - 1):
        a, b = int(offsets[s]), int(offsets[s + 1])
        if a == b:
            continue
        eps, g = R.emissions(probs[a:b], stride), R.gaps(start[a:b], stride)
        best = ref["best"][s]
        score = R.path_score(got["state"][a:b], eps, g, C, stride, L)
        assert abs(score - best) <= 1e-9 * abs(best) + 1e-12, (s, score, best)
        sure = R.margins(eps, g, C, stride, L) > 1e-9 * (1 + abs(best))
        assert np.array_equal(got["state"][a:b][sure], ref["state"][a:b][sure]), s
    tab = R.decode(probs, offsets, start, length, stride, L, path_override=got["state"])
    for k in ("region_contig", "region_start", "region_end", "region_class", "region_windows", "region_scores"):
        assert np.array_equal(got[k], tab[k]), k
    assert np.abs(got["region_posterior"] - tab["region_posterior"]).max(initial=0) <= 1e-6
    return ref


SIZES = [1, 2, 97, 0, 130, 1, 33]


@pytest.mark.parametrize("C", [2, 3, 5, 32])
@pytest.mark.parametrize("stride", [1, 100, 1000, 6000])
@pytest.mark.parametrize("L", [12000.0, 1e9])
def test_against_oracle(torch, C, stride, L):
    rng = np.random.default_rng(C * 7 + stride + int(L) % 97)
    probs, offsets, start, length = planted(rng, SIZES, C, stride)
    got = host(engine.window_regions(to_ws(torch, probs, offsets, start, length), stride, L))
    check_against_oracle(probs, offsets, start, length, stride, L, got)


@pytest.mark.parametrize("C", [3, 32])
def test_long_sequence(torch, C):
    """100,000 windows in one sequence (a 10 Mbp contig at stride 100): the serial worst case of one warp."""
    rng = np.random.default_rng(C)
    probs, offsets, start, length = planted(rng, [100_000, 3], C, 100)
    got = host(engine.window_regions(to_ws(torch, probs, offsets, start, length), 100, 12000.0))
    check_against_oracle(probs, offsets, start, length, 100, 12000.0, got)


def test_all_zero_and_all_one_rows(torch):
    """Every score 0 (the 1e-30 floor in every class: a tie everywhere, so class 0 throughout) and every score 1."""
    for v in (0.0, 1.0):
        probs = np.full((50, 4), v, np.float32)
        offsets, start, length = np.array([0, 50]), np.arange(50) * 1000, np.full(50, 6000, np.int32)
        got = host(engine.window_regions(to_ws(torch, probs, offsets, start, length), 1000, 12000.0))
        assert (got["state"] == 0).all() and len(got["region_class"]) == 1
        np.testing.assert_allclose(got["posterior"], 0.25, rtol=0, atol=1e-7)
        check_against_oracle(probs, offsets, start, length, 1000, 12000.0, got)


def test_bitwise_under_order_and_chunking(torch):
    rng = np.random.default_rng(5)
    sizes = [int(x) for x in rng.integers(0, 300, 40)] + [2000]
    probs, offsets, start, length = planted(rng, sizes, 5, 100)
    base = host(engine.window_regions(to_ws(torch, probs, offsets, start, length), 100, 20000.0))
    for work in (1 << 12, 1 << 16, 1 << 20):      # 1 sequence per call (the 2000-window one alone), a few, many
        got = host(engine.window_regions(to_ws(torch, probs, offsets, start, length), 100, 20000.0, work_bytes=work))
        for k in base:
            assert np.array_equal(base[k].view(np.uint8), got[k].view(np.uint8)), (work, k)
    perm = rng.permutation(len(sizes))
    seqs = [(probs[offsets[i]:offsets[i + 1]], start[offsets[i]:offsets[i + 1]], length[offsets[i]:offsets[i + 1]])
            for i in perm]
    p2 = np.concatenate([s[0] for s in seqs])
    o2 = np.concatenate([[0], np.cumsum([len(s[0]) for s in seqs])])
    got = host(engine.window_regions(to_ws(torch, p2, o2, np.concatenate([s[1] for s in seqs]),
                                         np.concatenate([s[2] for s in seqs])), 100, 20000.0))
    for new, old in enumerate(perm):
        a, b, a2, b2 = offsets[old], offsets[old + 1], o2[new], o2[new + 1]
        assert np.array_equal(got["posterior"][a2:b2].view(np.uint32), base["posterior"][a:b].view(np.uint32))
        assert np.array_equal(got["state"][a2:b2], base["state"][a:b])
        r_old, r_new = base["region_contig"] == old, got["region_contig"] == new
        for k in ("region_start", "region_end", "region_class", "region_windows", "region_posterior", "region_scores"):
            assert np.array_equal(got[k][r_new].view(np.uint8), base[k][r_old].view(np.uint8)), k


def test_invalid_profiles_are_refused(torch):
    probs = np.full((4, 3), 0.3, np.float32)
    ok = (np.array([0, 4]), np.array([0, 1000, 2000, 4000]), np.full(4, 6000, np.int32))
    engine.window_regions(to_ws(torch, probs, *ok), 1000, 12000)
    for st in ([0, 1000, 2500, 4000], [0, 1000, 1000, 4000], [0, 2000, 1000, 4000]):
        with pytest.raises(ValueError, match="multiples of the stride"):
            engine.window_regions(to_ws(torch, probs, ok[0], np.array(st), ok[2]), 1000, 12000)
    bad = probs.copy()
    bad[2, 1] = np.inf
    with pytest.raises(ValueError, match="finite"):
        engine.window_regions(to_ws(torch, bad, *ok), 1000, 12000)
    lib = engine.load_library()
    assert lib.gnm_window_regions_workspace_bytes(10, 33) == 0 and lib.gnm_window_regions_workspace_bytes(10, 1) == 0
    assert lib.gnm_window_regions_workspace_bytes(10, 3) == 3 * 256
    for C_, s, L in ((1, 1000, 12000.0), (33, 1000, 12000.0), (3, 0, 12000.0), (3, 6001, 12000.0), (3, 1000, 11999.0)):
        assert lib.gnm_window_regions(None, 4, C_, None, 1, None, None, s, L, *([None] * 8), None, 0, None) == 1
    assert lib.gnm_window_regions(None, 4, 3, None, 1, None, None, 1000, 12000.0, *([None] * 8), None, 0, None) == 1
    assert b"null buffer" in lib.gnm_last_error()


# ------------------------------------------------------------------------------------------------- end to end
def _records(fa):
    return [s for _, s in sequence.iter_fasta(fa, strip_n=False)]


def _same(path_npz, mem, names_key="contig_names"):
    z = np.load(path_npz)
    assert np.array_equal(z["window_posteriors"].view(np.uint32), mem["posterior"].view(np.uint32))
    assert np.array_equal(z["window_state"], mem["state"])
    for k in mem:
        if k.startswith("region_"):
            assert z[k].dtype == mem[k].dtype and np.array_equal(z[k].view(np.uint8), mem[k].view(np.uint8)), k
    assert names_key in z.files


def test_module_end_to_end(torch, tmp_path):
    L = 30000.0
    w = W.load_weights()
    hp = tmp_path / "h5.npz"
    W.save_head(hp, W.initial_head(5, 7), tuple(f"c{i}" for i in range(5)), w)
    nnc.main(TOY, tmp_path / "out", False, 128, False, 4, False, False, head=hp, write_window_scores=True, window_stride=1000)
    o = _paths.NNOutputs("toy", tmp_path / "out")
    seqs = _records(TOY)
    clf = nnc._make_classifier(128, 0)
    ws = clf.window_scores(seqs, 1000)
    assert ws.probs.shape[0] > 0
    WR.main(o.nn_classification_windows_npz_output, tmp_path / "regions", L, verbose=False)
    _same(tmp_path / "regions" / "toy_nn_classification_regions.npz", host(engine.window_regions(ws, 1000, L)))
    head = engine.Head(clf, W.load_head(hp, w))
    hws = head.window_scores(seqs, 1000)
    WR.main(o.nn_classification_head_windows_npz_output, tmp_path / "regions", L, verbose=False)
    zh = np.load(tmp_path / "regions" / "toy_nn_classification_head_regions.npz")
    assert list(zh["class_names"]) == [f"c{i}" for i in range(5)] and zh["window_posteriors"].shape == (hws.probs.shape[0], 5)
    _same(tmp_path / "regions" / "toy_nn_classification_head_regions.npz", host(engine.window_regions(hws, 1000, L)))
    tsv = (tmp_path / "regions" / "toy_nn_classification_head_regions.tsv").read_text().splitlines()
    assert tsv[0].endswith("c3_score\tc4_score") and len(tsv) == 1 + len(zh["region_start"])
    head.close()
