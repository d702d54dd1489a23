"""
CPU tests of the window-region decode (no GPU).  The fp64 oracle (tests/regions_ref.py) is checked against brute force over every
path of short sequences, and the region table against its invariants.  The window-regions module and CLI run with
engine.window_regions replaced by the oracle (tests/test_gpu_regions.py holds the kernel to the oracle): file names for the four
kinds of window file, TSV and NPZ format, head class names, sequences with zero or one window, N-rule gaps, and the rejection of
malformed files and of L < 12,000 before any decode.
"""
import itertools

import numpy as np
import pytest
import torch
from click.testing import CliRunner

import regions_ref as R
from genomad_b200 import cli, engine, window_regions as WR


def brute(eps, g, C, s, L):
    """Every path's probability: (scores [C^n], paths [C^n, n])."""
    n = eps.shape[0]
    paths = np.array(list(itertools.product(range(C), repeat=n)), np.int64)
    sc = np.array([R.path_score(p, eps, g, C, s, L) for p in paths])
    return sc, paths


@pytest.mark.parametrize("C", [2, 3])
@pytest.mark.parametrize("n", [1, 2, 5, 7])
@pytest.mark.parametrize("stride,L", [(1000, 12000.0), (100, 30000.0), (6000, 1e5)])
def test_oracle_against_brute_force(C, n, stride, L):
    rng = np.random.default_rng(C * 100 + n + stride)
    p = rng.dirichlet(np.full(C, 0.5), n).astype(np.float32)
    start = np.concatenate([[0], np.cumsum(rng.integers(1, 4, n - 1))]) * stride        # gaps of 1..3 strides
    eps, g = R.emissions(p, stride), R.gaps(start, stride)
    sc, paths = brute(eps, g, C, stride, L)
    path, best = R.viterbi(eps, g, C, stride, L)
    assert np.isclose(best, sc.max(), rtol=0, atol=1e-12)
    assert np.array_equal(path, paths[np.argmax(sc)])
    prob = np.exp(sc - sc.max())
    prob /= prob.sum()
    gam = R.forward_backward(eps, g, C, stride, L)
    marg = np.stack([np.bincount(paths[:, w], weights=prob, minlength=C) for w in range(n)])
    np.testing.assert_allclose(gam, marg, rtol=0, atol=1e-12)
    assert R.path_score(path, eps, g, C, stride, L) == pytest.approx(best, abs=1e-12)


@pytest.mark.parametrize("C", [2, 3, 5, 32])
def test_gap_transition_is_the_power_of_the_one_step_matrix(C):
    s, L = 100, 12000.0
    rho = s / L
    T1, O1 = R.transition(C, s, L, 1)
    assert T1 == pytest.approx(1 - rho, abs=1e-15) and O1 == pytest.approx(rho / (C - 1), abs=1e-15)
    A = np.full((C, C), O1)
    np.fill_diagonal(A, T1)
    for g in (2, 3, 7, 60):
        Tg, Og = R.transition(C, s, L, g)
        Ag = np.linalg.matrix_power(A, g)
        assert Tg == pytest.approx(Ag[0, 0], abs=1e-12) and Og == pytest.approx(Ag[0, 1], abs=1e-12)
        assert Tg + (C - 1) * Og == pytest.approx(1.0, abs=1e-15)


def test_ties_stay_and_go_to_the_lowest_class():
    for C in (2, 3, 7):
        p = np.full((9, C), 1.0 / C, np.float32)
        eps, g = R.emissions(p, 1000), R.gaps(np.arange(9) * 1000, 1000)
        path, _ = R.viterbi(eps, g, C, 1000, 12000.0)
        assert (path == 0).all()
    # two classes exactly tied throughout, a third lower: the lowest of the tied
    p = np.tile(np.array([[0.2, 0.4, 0.4]], np.float32), (6, 1))
    path, _ = R.viterbi(R.emissions(p, 6000), R.gaps(np.arange(6) * 6000, 6000), 3, 6000, 12000.0)
    assert (path == 1).all()


def _profile(rng, sizes, C, stride, gaps=True):
    probs, start, length, offsets = [], [], [], [0]
    for n in sizes:
        if n:
            st = np.concatenate([[0], np.cumsum(rng.integers(1, 3 if gaps else 2, n - 1))]) * stride + int(rng.integers(0, 50))
            ln = np.full(n, 6000, np.int64)
            ln[-1] = int(rng.integers(1, 6001))
            start.append(st)
            length.append(ln)
            probs.append(rng.dirichlet(np.full(C, 0.3), n))
        offsets.append(offsets[-1] + n)
    cat = (lambda xs, shape: np.concatenate(xs) if xs else np.zeros(shape))
    return (cat(probs, (0, C)).astype(np.float32), np.array(offsets, np.int64), cat(start, 0).astype(np.int64),
            cat(length, 0).astype(np.int64))


@pytest.mark.parametrize("stride", [1, 100, 1000, 6000])
def test_region_invariants(stride):
    rng = np.random.default_rng(stride)
    probs, offsets, start, length = _profile(rng, [0, 1, 2, 40, 0, 13], 3, stride)
    out = R.decode(probs, offsets, start, length, stride, 12000.0)
    assert out["region_windows"].sum() == len(probs)
    for s in range(len(offsets) - 1):
        a, b = offsets[s], offsets[s + 1]
        rows = np.flatnonzero(out["region_contig"] == s)
        if a == b:
            assert rows.size == 0
            continue
        st, en = out["region_start"][rows], out["region_end"][rows]
        assert st[0] == start[a] and en[-1] == start[b - 1] + length[b - 1]
        assert (st[1:] == en[:-1]).all() and (en >= st).all()
        assert out["region_windows"][rows].sum() == b - a
        cls = np.repeat(out["region_class"][rows], out["region_windows"][rows])
        assert np.array_equal(cls, out["state"][a:b])
        assert (out["region_class"][rows][1:] != out["region_class"][rows][:-1]).all()     # maximal runs
    one = offsets[1]                                                                          # the one-window sequence
    k = int(np.flatnonzero(out["region_contig"] == 1)[0])
    assert out["region_class"][k] == np.argmax(probs[one]) and out["region_windows"][k] == 1
    np.testing.assert_array_equal(out["region_scores"][k], probs[one])


@pytest.mark.parametrize("C", [2, 3, 5])
def test_weak_evidence_gives_one_region_of_the_summed_class(C):
    """No run pays |ln M_1| twice (M_1 = rho / (C - 1), L = 1e9): one region, class argmax of sum_w eps_w."""
    rng = np.random.default_rng(C)
    stride, L, n = 1000, 1e9, 60
    p = (1.0 / C + rng.uniform(-0.01, 0.01, (n, C))).astype(np.float32)
    eps = R.emissions(p, stride)
    assert np.abs(eps - eps.mean(1, keepdims=True)).sum() < abs(np.log(stride / L / (C - 1)))
    out = R.decode(p, [0, n], np.arange(n) * stride, np.full(n, 6000), stride, L)
    assert len(out["region_class"]) == 1 and out["region_class"][0] == np.argmax(eps.sum(0))


# ---------------------------------------------------------------------------------------------------------- module and CLI

def oracle_window_regions(ws, stride, mean_region_length, **kw):
    """The oracle behind engine.window_regions' contract (CPU tensors in and out)."""
    L = engine.regions_mean_length(mean_region_length)
    o = R.decode(ws.probs.numpy(), ws.offsets.numpy(), ws.start.numpy(), ws.length.numpy(), int(stride), L)
    f = lambda k, dt: torch.from_numpy(np.ascontiguousarray(o[k]).astype(dt))
    return engine.WindowRegions(f("posterior", np.float32), f("state", np.int32), f("region_contig", np.int32),
                                f("region_start", np.int64), f("region_end", np.int64), f("region_class", np.int32),
                                f("region_windows", np.int32), f("region_posterior", np.float32),
                                f("region_scores", np.float32))


@pytest.fixture
def stub(monkeypatch):
    calls = []

    def fake(*a, **k):
        calls.append(a)
        return oracle_window_regions(*a, **k)
    monkeypatch.setattr(engine, "window_regions", fake)
    monkeypatch.setattr(WR, "_device", lambda: torch.device("cpu"))
    return calls


def write_windows(path, names_key="contig_names", sizes=(3, 0, 1, 25), C=3, stride=1000, class_names=None, head_sha=None,
                  seed=0, **override):
    rng = np.random.default_rng(seed)
    probs, offsets, start, length = _profile(rng, sizes, C, stride)
    d = {names_key: np.array([f"seq{i}" for i in range(len(sizes))]), "predictions": probs,
         "window_contig": np.repeat(np.arange(len(sizes), dtype=np.int32), np.diff(offsets)),
         "window_start": start, "window_length": length.astype(np.int32), "window_stride": np.int32(stride)}
    if class_names is not None:
        d["class_names"] = np.array(class_names)
    if head_sha is not None:
        d["head_sha256"] = np.str_(head_sha)
    d.update(override)
    np.savez(path, **d)
    return d, offsets


@pytest.mark.parametrize("name,expected", [
    ("toy_nn_classification_windows.npz", "toy_nn_classification_regions"),
    ("toy_nn_classification_head_windows.npz", "toy_nn_classification_head_regions"),
    ("toy_provirus_nn_classification_windows.npz", "toy_provirus_nn_classification_regions"),
    ("toy_provirus_nn_classification_head_windows.npz", "toy_provirus_nn_classification_head_regions"),
    ("profile.npz", "profile_regions"),
])
def test_output_names(tmp_path, stub, name, expected):
    key = "provirus_names" if "provirus" in name else "contig_names"
    head = "_head_" in name
    write_windows(tmp_path / name, key, C=4 if head else 3, class_names=list("wxyz") if head else None,
                  head_sha="ab" * 32 if head else None)
    WR.main(tmp_path / name, tmp_path / "out", 12000, verbose=False)
    assert sorted(p.name for p in (tmp_path / "out").iterdir()) == [expected + ".npz", expected + ".tsv"]
    z = np.load(tmp_path / "out" / (expected + ".npz"))
    assert key in z.files and ("head_sha256" in z.files) == head


def test_tsv_and_npz_format(tmp_path, stub):
    d, offsets = write_windows(tmp_path / "a_nn_classification_head_windows.npz", C=4, class_names=["p", "q", "r", "s"],
                               head_sha="cd" * 32, stride=100, sizes=(0, 1, 2, 70, 5))
    WR.main(tmp_path / "a_nn_classification_head_windows.npz", tmp_path, 25000.5, verbose=False)
    z = np.load(tmp_path / "a_nn_classification_head_regions.npz")
    o = R.decode(d["predictions"], offsets, d["window_start"], d["window_length"], 100, 25000.5)
    assert sorted(z.files) == sorted(["contig_names", "region_contig", "region_start", "region_end", "region_class",
                                      "region_windows", "region_posterior", "region_scores", "window_posteriors",
                                      "window_state", "class_names", "window_stride", "mean_region_length", "head_sha256"])
    for k, dt in (("region_contig", np.int32), ("region_start", np.int64), ("region_end", np.int64),
                  ("region_class", np.int32), ("region_windows", np.int32), ("region_posterior", np.float32),
                  ("region_scores", np.float32)):
        assert z[k].dtype == dt
        np.testing.assert_array_equal(z[k], o[k])
    assert z["window_posteriors"].dtype == np.float32 and z["window_state"].dtype == np.int32
    np.testing.assert_array_equal(z["window_posteriors"], o["posterior"].astype(np.float32))
    assert list(z["class_names"]) == ["p", "q", "r", "s"] and str(z["head_sha256"]) == "cd" * 32
    assert int(z["window_stride"]) == 100 and float(z["mean_region_length"]) == 25000.5
    lines = (tmp_path / "a_nn_classification_head_regions.tsv").read_text().splitlines()
    assert lines[0] == "seq_name\tstart\tend\tlength\tclass\tn_windows\tposterior\tp_score\tq_score\tr_score\ts_score"
    assert len(lines) == 1 + len(o["region_start"])
    for line, r in zip(lines[1:], range(len(o["region_start"]))):
        f = line.split("\t")
        s, e = int(o["region_start"][r]), int(o["region_end"][r])
        assert f[0] == f"seq{o['region_contig'][r]}" and f[1:4] == [str(s + 1), str(e), str(e - s)]
        assert f[4] == "pqrs"[o["region_class"][r]] and f[5] == str(o["region_windows"][r])
        assert f[6] == f"{o['region_posterior'][r]:.4f}"
        assert f[7:] == [f"{x:.4f}" for x in o["region_scores"][r]]
    # zero-window sequences have no rows, a one-window sequence one
    assert "seq0\t" not in "".join(lines) and sum(ln.startswith("seq1\t") for ln in lines) == 1


def test_default_class_names_and_no_head_sha(tmp_path, stub):
    write_windows(tmp_path / "x_nn_classification_windows.npz")
    WR.main(tmp_path / "x_nn_classification_windows.npz", tmp_path, 12000, verbose=False)
    z = np.load(tmp_path / "x_nn_classification_regions.npz")
    assert list(z["class_names"]) == ["chromosome", "plasmid", "virus"] and "head_sha256" not in z.files
    head = (tmp_path / "x_nn_classification_regions.tsv").read_text().splitlines()[0]
    assert head.endswith("chromosome_score\tplasmid_score\tvirus_score")


def test_empty_file(tmp_path, stub):
    write_windows(tmp_path / "e_nn_classification_windows.npz", sizes=(0, 0))
    WR.main(tmp_path / "e_nn_classification_windows.npz", tmp_path, 12000, verbose=False)
    z = np.load(tmp_path / "e_nn_classification_regions.npz")
    assert z["region_start"].shape == (0,) and z["window_posteriors"].shape == (0, 3)
    assert len((tmp_path / "e_nn_classification_regions.tsv").read_text().splitlines()) == 1


BAD = {
    "no names": dict(contig_names=None),
    "both names": dict(provirus_names=np.array(["a", "b", "c", "d"])),
    "no stride": dict(window_stride=None),
    "1-d predictions": dict(predictions=np.zeros(29, np.float32)),
    "C = 1": dict(predictions=np.zeros((29, 1), np.float32)),
    "C = 33": dict(predictions=np.zeros((29, 33), np.float32)),
    "integer predictions": dict(predictions=np.zeros((29, 3), np.int32)),
    "NaN score": dict(predictions=np.where(np.arange(87).reshape(29, 3) == 40, np.nan, 0.5).astype(np.float32)),
    "class names": dict(class_names=np.array(["a", "b"])),
    "short contig": dict(window_contig=np.zeros(28, np.int32)),
    "contig out of range": dict(window_contig=np.full(29, 7, np.int32)),
    "contig order": dict(window_contig=np.array([3] * 25 + [0] * 3 + [2], np.int32)),
    "stride 0": dict(window_stride=np.int32(0)),
    "stride 6001": dict(window_stride=np.int32(6001)),
    "length 0": dict(window_length=np.zeros(29, np.int32)),
    "float starts": dict(window_start=np.zeros(29, np.float64)),
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_malformed_files_are_refused_before_any_decode(tmp_path, stub, case):
    path = tmp_path / "bad_nn_classification_windows.npz"
    d, _ = write_windows(path)
    for k, v in BAD[case].items():
        if v is None:
            d.pop(k)
        else:
            d[k] = v
    np.savez(path, **d)
    with pytest.raises(WR.WindowsFileError):
        WR.main(path, tmp_path / "out", 12000, verbose=False)
    assert not stub and not (tmp_path / "out").exists()


@pytest.mark.parametrize("how", ["not a multiple", "repeated", "decreasing"])
def test_starts_off_the_stride_grid_are_refused(tmp_path, stub, how):
    path = tmp_path / "g_nn_classification_windows.npz"
    d, _ = write_windows(path, sizes=(30,))
    st = d["window_start"].copy()
    st[10] = {"not a multiple": st[10] + 1, "repeated": st[9], "decreasing": st[9] - 1000}[how]
    d["window_start"] = st
    np.savez(path, **d)
    with pytest.raises(WR.WindowsFileError, match="window 10"):
        WR.main(path, tmp_path, 12000, verbose=False)
    assert not stub


def test_not_an_npz(tmp_path, stub):
    (tmp_path / "x.npz").write_bytes(b"not a zip")
    with pytest.raises(WR.WindowsFileError):
        WR.main(tmp_path / "x.npz", tmp_path, 12000, verbose=False)


def test_short_mean_region_length_is_refused(tmp_path, stub):
    write_windows(tmp_path / "w_nn_classification_windows.npz")
    for L in (11999.9, 0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            WR.main(tmp_path / "w_nn_classification_windows.npz", tmp_path / "o", L, verbose=False)
    res = CliRunner().invoke(cli.cli, ["window-regions", str(tmp_path / "w_nn_classification_windows.npz"), str(tmp_path / "o"),
                                       "--mean-region-length", "11999"])
    assert res.exit_code != 0 and "12000" in res.output
    res = CliRunner().invoke(cli.cli, ["window-regions", str(tmp_path / "w_nn_classification_windows.npz"), str(tmp_path / "o")])
    assert res.exit_code != 0 and "--mean-region-length" in res.output
    assert not stub and not (tmp_path / "o").exists()


def test_cli(tmp_path, stub):
    write_windows(tmp_path / "c_provirus_nn_classification_windows.npz", "provirus_names")
    res = CliRunner().invoke(cli.cli, ["window-regions", str(tmp_path / "c_provirus_nn_classification_windows.npz"),
                                       str(tmp_path / "out"), "--mean-region-length", "50000", "-q"])
    assert res.exit_code == 0, res.output
    z = np.load(tmp_path / "out" / "c_provirus_nn_classification_regions.npz")
    assert float(z["mean_region_length"]) == 50000.0 and "provirus_names" in z.files
    assert "one process on one GPU" in " ".join(CliRunner().invoke(cli.cli, ["window-regions", "--help"]).output.split())


def test_engine_argument_checks():
    ws = engine.WindowScores(torch.zeros((2, 3)), torch.zeros(2, dtype=torch.int32), torch.tensor([0, 1000]),
                             torch.full((2,), 6000, dtype=torch.int32), torch.tensor([0, 2], dtype=torch.int32))
    with pytest.raises(ValueError, match="mean_region_length"):
        engine.window_regions(ws, 1000, 11000)
    with pytest.raises(ValueError, match="stride"):
        engine.window_regions(ws, 0, 12000)
    with pytest.raises(ValueError, match="C <= 32"):
        engine.window_regions(ws._replace(probs=torch.zeros((2, 1))), 1000, 12000)
