"""
CPU tests of head novelty around the kernels: the head file's four novelty keys (round trip, byte-identical files, partial or
malformed sets refused naming the key), the p-value rule of engine.novelty_scores, the nn-classification --head novelty files
(layout, values, provirus twin, written exactly when the head has a model, restart and head_sha256 rules, other files
unchanged) with stub classifiers (tests/window_stub.py, tests/head_stub.py), and train-head --novelty's argument checks and
CLI wiring.
"""
import shutil
import zipfile

import numpy as np
import pytest

import head_stub as HS
import novelty_ref as R
import window_stub as WS
from genomad_b200 import _paths, engine, nn_classification, sequence, train_head, weights as W
from test_strands_cpu import EmbedStub, _all_files, stub_emb
from test_window_scores_cpu import _module_fasta, _run

CLASSES = ("alpha", "beta", "gamma.1")


def stub_novelty(emb: np.ndarray, C: int) -> np.ndarray:
    """float32 [n, 512] -> float32 [n, C]: a distance-like function of the row, positive and class dependent."""
    proj = np.sin(np.arange(512 * C, dtype=np.float64).reshape(512, C) * 0.11)
    return ((emb.astype(np.float64) @ proj * 0.01) ** 2 + 0.5 + np.arange(C) * 0.1).astype(np.float32)


class StubNoveltyHead(HS.StubHead):
    def __init__(self, clf, head_file):
        super().__init__(clf, head_file)
        self.has_novelty = head_file.novelty is not None

    def novelty(self, embeddings, out=None):
        assert self.has_novelty
        d = __import__("torch").from_numpy(stub_novelty(embeddings.numpy(), self.n_classes))
        if out is None:
            return d
        out.copy_(d)
        return out


def model(C, seed=0, n_cal=9):
    rng = np.random.default_rng(seed)
    P = np.tril(rng.normal(0, 0.1, (512, 512)))
    np.fill_diagonal(P, rng.uniform(0.5, 2, 512))
    return {"novelty_center": rng.normal(0, 1, 512), "novelty_whitening": P, "novelty_means": rng.normal(0, 1, (C, 512)),
            "novelty_calibration": np.sort(rng.uniform(0.5, 3, n_cal)).astype(np.float32)}


def write_novelty_head(path, C=len(CLASSES), seed=1, names=CLASSES, nov_seed=0):
    w = W.load_weights()
    W.save_head(path, W.initial_head(C, seed), names, w, novelty=model(C, nov_seed))
    return path


# ---------------------------------------------------------------------------------------------------------------- head files
def test_round_trip_and_bytes(tmp_path):
    w = W.load_weights()
    a = write_novelty_head(tmp_path / "a.npz")
    b = write_novelty_head(tmp_path / "b.npz")
    assert a.read_bytes() == b.read_bytes()
    h = W.load_head(a, w)
    for k, v in model(len(CLASSES)).items():
        assert h.novelty[k].dtype == v.dtype and np.array_equal(h.novelty[k], v), k
    # without the model: exactly the members and bytes of a plain head file
    W.save_head(tmp_path / "p.npz", W.initial_head(3, 1), CLASSES, w)
    W.save_head(tmp_path / "q.npz", W.initial_head(3, 1), CLASSES, w, novelty=None)
    assert (tmp_path / "p.npz").read_bytes() == (tmp_path / "q.npz").read_bytes()
    assert W.load_head(tmp_path / "p.npz", w).novelty is None
    plain = zipfile.ZipFile(tmp_path / "p.npz").namelist()
    assert not any(n.startswith("novelty") for n in plain)
    assert zipfile.ZipFile(a).namelist() == plain + [k + ".npy" for k in W.NOVELTY_KEYS]


def _rewrite(src, dst, drop=(), replace=None):
    with zipfile.ZipFile(src) as zin, zipfile.ZipFile(dst, "w") as zout:
        for name in zin.namelist():
            key = name[:-4]
            if key in drop:
                continue
            if replace and key in replace:
                with zout.open(name, "w") as f:
                    np.lib.format.write_array(f, replace[key], allow_pickle=False)
            else:
                zout.writestr(name, zin.read(name))


@pytest.mark.parametrize("key", W.NOVELTY_KEYS)
def test_partial_set_is_refused(tmp_path, key):
    src = write_novelty_head(tmp_path / "a.npz")
    _rewrite(src, tmp_path / "b.npz", drop=(key,))
    with pytest.raises(ValueError, match=f"{key} missing"):
        W.load_head(tmp_path / "b.npz", W.load_weights())


def _bad_cases():
    m = model(3)
    P_up = m["novelty_whitening"].copy()
    P_up[3, 7] = 1e-3
    P_diag = m["novelty_whitening"].copy()
    P_diag[5, 5] = 0.0
    nan_c = m["novelty_center"].copy()
    nan_c[2] = np.nan
    return [("novelty_center", m["novelty_center"].astype(np.float32), "dtype"),
            ("novelty_center", nan_c, "not all finite"),
            ("novelty_whitening", P_up, "not lower triangular"),
            ("novelty_whitening", P_diag, "diagonal not positive at 5"),
            ("novelty_means", m["novelty_means"][:2], "shape"),
            ("novelty_calibration", m["novelty_calibration"][::-1].copy(), "not sorted"),
            ("novelty_calibration", np.zeros(0, np.float32), "n >= 1"),
            ("novelty_calibration", m["novelty_calibration"].astype(np.float64), "dtype")]


@pytest.mark.parametrize("key,value,msg", _bad_cases())
def test_malformed_key_is_refused(tmp_path, key, value, msg):
    src = write_novelty_head(tmp_path / "a.npz")
    _rewrite(src, tmp_path / "b.npz", replace={key: value})
    with pytest.raises(ValueError, match=f"{key}.*{msg}"):
        W.load_head(tmp_path / "b.npz", W.load_weights())
    with pytest.raises(ValueError, match=key):
        W.save_head(tmp_path / "c.npz", W.initial_head(3, 1), CLASSES, W.load_weights(), novelty={**model(3), key: value})


# ----------------------------------------------------------------------------------------------------------------- p-values
def test_p_value_rule():
    cal = np.array([0.5, 1.0, 1.0, 2.0, 4.0], np.float32)
    dist = np.array([[1.0, 3.0], [5.0, 4.5], [0.1, 0.2], [2.0, 2.0], [9.0, 9.0], [0.7, 1.5]], np.float32)
    counts = np.array([3, 1, 2, 5, 0, 1])
    nov, nearest, p = engine.novelty_scores(dist, counts, cal)
    assert nov.dtype == np.float32 and nearest.dtype == np.int32 and p.dtype == np.float64
    assert nearest.tolist() == [0, 1, 0, 0, -1, 0]                      # ties: the lowest index
    assert p[0] == 5 / 6                                                # ties with calibration values count as >=
    assert p[1] == 1 / 6                                                # beyond the largest value: 1 / (1 + |cal|)
    assert p[2] == 1.0 and p[3] == 3 / 6
    assert np.isnan(nov[4]) and np.isnan(p[4])                          # no window: never 0, never "typical"
    for i in range(len(counts)):
        r = R.p_value(nov[i], cal)
        assert (np.isnan(r) and np.isnan(p[i])) or r == p[i]


# ----------------------------------------------------------------------------------------------------- nn-classification
@pytest.fixture
def stub(monkeypatch):
    clf = EmbedStub()
    WS.install(monkeypatch.setattr, nn_classification, clf)
    monkeypatch.setattr(nn_classification, "_make_head", StubNoveltyHead)
    for k in ("GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS", "GENOMAD_B200_ATTRIBUTIONS",
              "GENOMAD_B200_BOTH_STRANDS", "GENOMAD_B200_HEAD_ATTRIBUTIONS", "RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    return clf


def _expected(fa, single_window=False):
    pf = sequence.ParsedFasta(fa, single_window)
    try:
        win = pf.export_windows(0, pf.n_windows, np.empty((pf.n_windows, 6000), np.uint8))
        offsets = np.asarray(pf.index().offsets)
    finally:
        pf.close()
    return WS.running_mean(stub_novelty(stub_emb(win), len(CLASSES)), offsets), np.diff(offsets)


def _check_files(npz, tsv, names_key, cal, dist=None, counts=None):
    z = np.load(npz)
    assert set(z.files) == {names_key, "distances", "novelty", "nearest_class", "p_value", "class_names", "head_sha256"}
    n = len(z[names_key])
    assert z["distances"].dtype == np.float32 and z["distances"].shape == (n, len(CLASSES))
    assert z["novelty"].dtype == np.float32 and z["nearest_class"].dtype == np.int32 and z["p_value"].dtype == np.float64
    assert list(z["class_names"]) == list(CLASSES)
    if dist is not None:
        assert z["distances"].tobytes() == dist.astype(np.float32).tobytes()
        nov, near, p = engine.novelty_scores(dist, counts, cal)
        assert np.array_equal(z["novelty"], nov, equal_nan=True) and np.array_equal(z["nearest_class"], near)
        assert np.array_equal(z["p_value"], p, equal_nan=True)
    lines = tsv.read_text().split("\n")
    assert lines[0] == "seq_name\tnearest_class\tnovelty\tp_value" and lines[-1] == "" and len(lines) == n + 2
    for i in range(n):
        c = int(z["nearest_class"][i])
        want = (f"{z[names_key][i]}\tNA\tNA\tNA" if c < 0 else
                f"{z[names_key][i]}\t{CLASSES[c]}\t{float(z['novelty'][i]):.6g}\t{float(z['p_value'][i]):.6g}")
        assert lines[1 + i] == want
    return z


@pytest.mark.parametrize("single_window", [False, True])
def test_novelty_file(tmp_path, stub, single_window):
    hp = write_novelty_head(tmp_path / "h.npz")
    fa = _module_fasta(tmp_path / "sample.fna")
    o = _run(fa, tmp_path / "out", head=hp, single_window=single_window)
    dist, counts = _expected(fa, single_window)
    z = _check_files(o.nn_classification_head_novelty_npz_output, o.nn_classification_head_novelty_output, "contig_names",
                     model(3)["novelty_calibration"], dist, counts)
    assert list(z["contig_names"]) == list(np.load(o.nn_classification_head_npz_output)["contig_names"])


@pytest.mark.parametrize("extra", [{"both_strands": True}, {"write_window_scores": True, "window_stride": 1000},
                                   {"write_embeddings": True}])
def test_novelty_file_with_other_outputs_is_forward_only(tmp_path, stub, extra):
    hp = write_novelty_head(tmp_path / "h.npz")
    fa = _module_fasta(tmp_path / "sample.fna")
    o = _run(fa, tmp_path / "out", head=hp, **extra)
    dist, counts = _expected(fa)
    _check_files(o.nn_classification_head_novelty_npz_output, o.nn_classification_head_novelty_output, "contig_names",
                 model(3)["novelty_calibration"], dist, counts)


def test_written_exactly_with_a_model_and_nothing_else_changes(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    hp = HS.write_head(tmp_path / "plain.npz", 3, 1, names=CLASSES)
    hn = write_novelty_head(tmp_path / "nov.npz")
    o1 = _run(fa, tmp_path / "a", head=hp)
    o2 = _run(fa, tmp_path / "b", head=hn)
    assert not o1.nn_classification_head_novelty_npz_output.exists() and not o1.nn_classification_head_novelty_output.exists()
    assert o2.nn_classification_head_novelty_npz_output.exists()
    f1, f2 = _all_files(tmp_path / "a"), _all_files(tmp_path / "b")
    f2 = {k: v for k, v in f2.items() if "novelty" not in k}
    assert f1 == f2
    for p in (o1.nn_classification_head_npz_output, o1.nn_classification_npz_output):
        q = tmp_path / "b" / p.relative_to(tmp_path / "a")
        za, zb = np.load(p), np.load(q)
        for k in za.files:
            if k != "head_sha256":
                assert za[k].tobytes() == zb[k].tobytes(), k


def test_provirus_twin(tmp_path, stub, golden_dir):
    inp = golden_dir / "reference_module" / "input"
    out = tmp_path / "out"
    shutil.copytree(inp / "toy_find_proviruses", out / "toy_find_proviruses")
    hp = write_novelty_head(tmp_path / "h.npz")
    nn_classification.main(inp / "toy.fna", out, False, 128, False, 2, False, False, head=hp)
    o = _paths.NNOutputs("toy", out)
    zp = _check_files(o.provirus_nn_classification_head_novelty_npz_output, o.provirus_nn_classification_head_novelty_output,
                      "provirus_names", model(3)["novelty_calibration"])
    assert len(zp["provirus_names"]) > 0 and o.nn_classification_head_novelty_npz_output.exists()


def test_empty_input_writes_zero_rows(tmp_path, stub, golden_dir):
    inp = golden_dir / "reference_module" / "input"
    out = tmp_path / "out"
    shutil.copytree(inp / "toy_find_proviruses", out / "toy_find_proviruses")
    (out / "toy_find_proviruses" / "toy_provirus.fna").write_text(">p1|provirus_1_500\n" + "N" * 500 + "\n")
    nn_classification.main(inp / "toy.fna", out, False, 128, False, 2, False, False, head=write_novelty_head(tmp_path / "h.npz"))
    o = _paths.NNOutputs("toy", out)
    z = np.load(o.provirus_nn_classification_head_novelty_npz_output)
    assert z["distances"].shape == (len(z["provirus_names"]), len(CLASSES)) and z["novelty"].shape == (len(z["provirus_names"]),)
    assert np.isnan(z["novelty"]).all() and np.isnan(z["p_value"]).all() and (z["nearest_class"] == -1).all()
    lines = o.provirus_nn_classification_head_novelty_output.read_text().split("\n")
    assert lines[0] == "seq_name\tnearest_class\tnovelty\tp_value" and all(x.endswith("\tNA\tNA\tNA") for x in lines[1:-1])


def test_restart_rules(tmp_path, stub):
    fa = _module_fasta(tmp_path / "sample.fna")
    h1 = write_novelty_head(tmp_path / "h1.npz")
    h2 = write_novelty_head(tmp_path / "h2.npz", nov_seed=5)             # same layers, another model: another sha256
    o = _run(fa, tmp_path / "out", head=h1)
    p = o.nn_classification_head_novelty_npz_output
    t0 = p.stat().st_mtime_ns
    n0 = len(stub.seen)
    _run(fa, tmp_path / "out", head=h1)
    assert len(stub.seen) == n0 and p.stat().st_mtime_ns == t0, "a current novelty file was recomputed"
    _run(fa, tmp_path / "out", head=h2)
    assert len(stub.seen) > n0
    assert str(np.load(p)["head_sha256"]) == nn_classification._load_head_file(h2)[1]
    o.nn_classification_head_novelty_output.unlink()                    # a missing file triggers a rerun
    n1 = len(stub.seen)
    _run(fa, tmp_path / "out", head=h2)
    assert len(stub.seen) > n1 and o.nn_classification_head_novelty_output.exists()


# ------------------------------------------------------------------------------------------------------------- train-head
def test_novelty_without_validation_is_refused_before_any_work(tmp_path, monkeypatch):
    def boom(*a, **k):
        raise AssertionError("work started")
    monkeypatch.setattr(train_head, "_make_classifier", boom)
    monkeypatch.setattr(train_head.sequence, "ParsedFasta", boom)
    with pytest.raises(ValueError, match="validation fraction > 0"):
        train_head.main(tmp_path / "x.fna", tmp_path / "l.tsv", tmp_path / "out", validation_fraction=0.0, novelty=True)


def test_cli_flag_is_wired(tmp_path, monkeypatch):
    from click.testing import CliRunner
    from genomad_b200 import cli
    fa, lab = tmp_path / "x.fna", tmp_path / "l.tsv"
    fa.write_text(">a\nACGT\n")
    lab.write_text("seq_name\tclass\n")
    seen = []
    monkeypatch.setattr(train_head, "main", lambda *a, **k: seen.append(k))
    for args, want in ((["--novelty"], True), ([], None)):
        r = CliRunner().invoke(cli.cli, ["train-head", str(fa), str(lab), str(tmp_path / "o"), *args])
        assert r.exit_code == 0, r.output
        assert seen[-1].get("novelty") == want
