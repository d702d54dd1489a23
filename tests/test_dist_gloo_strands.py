"""
Gloo tests (CPU, world sizes 2 and 3) of `nn-classification --both-strands --write-embeddings` under torchrun: the reverse pass
shards its window list like the forward pass, reduces the scores by the gather route and the embeddings by the carry chain, and
the strand files and the embeddings file rank 0 writes must be bitwise those of one process.  The classifier is a stub that is a
deterministic function of the window bytes (tests/test_strands_cpu.py).
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
from test_strands_cpu import EmbedStub


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _fasta(path):
    rng = np.random.default_rng(13)
    lengths = [20000, 3000, 47000, 6100, 1200, 31000, 9000, 12500]
    with open(path, "w") as fh:
        for i, ln in enumerate(lengths):
            s = bytearray(np.frombuffer(b"ACGTacgt", np.uint8)[rng.integers(0, 8, ln)].tobytes())
            if i == 2:
                s[12000:16800] = b"N" * 4800                         # windows the N rule drops
            if i == 7:
                s[1000:5600] = b"N" * 4600                           # dropped on the reverse strand only
            fh.write(f">c{i}\n" + "\n".join(s[k:k + 70].decode() for k in range(0, ln, 70)) + "\n")
    return path


def _run(fa, out, single_window):
    nn_classification.main(fa, out, single_window, 128, False, 2, False, False, write_embeddings=True, both_strands=True)


def _worker(rank, world, port, tmp, single_window):
    from pathlib import Path
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    for k in ("GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS", "GENOMAD_B200_BOTH_STRANDS"):
        os.environ.pop(k, None)
    clf = EmbedStub()
    WS.install(setattr, nn_classification, clf)
    tmp = Path(tmp)
    _run(tmp / "sample.fna", tmp / f"out_{world}", single_window)
    np.save(tmp / f"seen_{world}_{rank}.npy", np.array([len(clf.windows_seen())]))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("single_window", [False, True])
@pytest.mark.parametrize("world", [2, 3])
def test_strand_files_match_one_process(tmp_path, monkeypatch, world, single_window):
    fa = _fasta(tmp_path / "sample.fna")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS",
              "GENOMAD_B200_BOTH_STRANDS"):
        monkeypatch.delenv(k, raising=False)
    one = EmbedStub()
    WS.install(monkeypatch.setattr, nn_classification, one)
    _run(fa, tmp_path / "one", single_window)
    o1 = _paths.NNOutputs("sample", tmp_path / "one")
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path), single_window), nprocs=world, join=True)
    ow = _paths.NNOutputs("sample", tmp_path / f"out_{world}")
    for path in ("nn_classification_strands_npz_output", "nn_classification_embeddings_output", "nn_classification_npz_output"):
        z1, zw = np.load(getattr(o1, path)), np.load(getattr(ow, path))
        assert set(z1.files) == set(zw.files)
        for k in z1.files:
            assert z1[k].dtype == zw[k].dtype and np.array_equal(z1[k], zw[k]), (path, k)
    assert o1.nn_classification_strands_output.read_bytes() == ow.nn_classification_strands_output.read_bytes()
    assert "embeddings_both_strands" in np.load(ow.nn_classification_embeddings_output).files
    seen = sum(int(np.load(tmp_path / f"seen_{world}_{r}.npy")[0]) for r in range(world))
    assert seen == len(one.windows_seen())                  # every window of both strands classified exactly once
    shutil.rmtree(tmp_path / f"out_{world}")
