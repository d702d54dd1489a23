"""
Gloo tests (CPU, world sizes 2 and 3) of the per-window score export under torchrun: every rank classifies its contiguous shard
of the window list through the module's real chunk loop (with a stub classifier that is a deterministic function of the window
bytes), rank 0 collects the shards in rank order, and the windows NPZ and TSV it writes must be bitwise those of one process,
at stride 6000 (the contig pass's own windows) and at stride 1000 (a second pass over overlapping windows).
"""
import os
import shutil
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import window_stub as WS
from genomad_b200 import _paths, nn_classification


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _fasta(path):
    rng = np.random.default_rng(12)
    lengths = [20000, 3000, 47000, 6100, 1200, 31000, 9000]
    with open(path, "w") as fh:
        for i, ln in enumerate(lengths):
            s = bytearray(np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, ln)].tobytes())
            if i == 2:
                s[12000:16800] = b"N" * 4800                         # windows dropped by the N rule
            fh.write(f">c{i}\n" + "\n".join(s[k:k + 70].decode() for k in range(0, ln, 70)) + "\n")
    return path


def _worker(rank, world, port, tmp, stride):
    from pathlib import Path
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    os.environ.pop("GENOMAD_B200_WINDOW_SCORES", None)
    clf = WS.StubClassifier()
    WS.install(setattr, nn_classification, clf)
    tmp = Path(tmp)
    out = tmp / f"out_{world}"
    nn_classification.main(tmp / "sample.fna", out, False, 128, False, 2, False, False, write_window_scores=True,
                           window_stride=stride)
    n_seen = np.array([len(clf.windows_seen())])
    np.save(tmp / f"seen_{world}_{rank}.npy", n_seen)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("stride", [6000, 1000])
@pytest.mark.parametrize("world", [2, 3])
def test_windows_npz_matches_one_process(tmp_path, monkeypatch, world, stride):
    fa = _fasta(tmp_path / "sample.fna")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "GENOMAD_B200_WINDOW_SCORES"):
        monkeypatch.delenv(k, raising=False)
    one = WS.StubClassifier()
    WS.install(monkeypatch.setattr, nn_classification, one)
    nn_classification.main(fa, tmp_path / "one", False, 128, False, 2, False, False, write_window_scores=True,
                           window_stride=stride)
    o1 = _paths.NNOutputs("sample", tmp_path / "one")
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path), stride), nprocs=world, join=True)
    ow = _paths.NNOutputs("sample", tmp_path / f"out_{world}")
    z1, zw = np.load(o1.nn_classification_windows_npz_output), np.load(ow.nn_classification_windows_npz_output)
    assert set(z1.files) == set(zw.files)
    for k in z1.files:
        assert z1[k].dtype == zw[k].dtype and np.array_equal(z1[k], zw[k]), k
    assert o1.nn_classification_windows_output.read_bytes() == ow.nn_classification_windows_output.read_bytes()
    p1, pw = np.load(o1.nn_classification_npz_output), np.load(ow.nn_classification_npz_output)
    assert np.array_equal(p1["predictions"], pw["predictions"])
    # every window was classified exactly once across the ranks (the contig pass, plus the profile pass at stride 1000)
    seen = sum(int(np.load(tmp_path / f"seen_{world}_{r}.npy")[0]) for r in range(world))
    assert seen == len(one.windows_seen())
    if stride == 1000:
        assert len(z1["predictions"]) > len(np.load(o1.nn_classification_npz_output)["contig_names"]) * 3
    shutil.rmtree(tmp_path / f"out_{world}")
