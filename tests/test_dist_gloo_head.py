"""
Gloo tests (CPU, world sizes 2 and 3) of `nn-classification --head` under torchrun: the head scores of each rank's shard are
reduced per contig by the gather route (bitwise those of one process) or the allreduce route (fp32 re-association only), for a
width other than 3; and train-head refuses to run with more than one process.  Stub classifier and head: tests/head_stub.py.
"""
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import head_stub as HS
import window_stub as WS
from genomad_b200 import _paths, nn_classification, train_head
from test_dist_gloo_strands import _fasta
from test_strands_cpu import EmbedStub

C = 5


class SumStub(EmbedStub):
    def segment_sum(self, probs, offsets):
        import torch
        return torch.from_numpy(HS.running_sum(probs.numpy(), offsets.numpy()))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _install(setattr_, clf):
    WS.install(setattr_, nn_classification, clf)
    setattr_(nn_classification, "_make_head", HS.StubHead)


def _run(fa, out, head, reduce):
    nn_classification.main(fa, out, False, 128, False, 2, False, False, contig_reduce=reduce, head=head)


def _worker(rank, world, port, tmp, reduce):
    from pathlib import Path
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    for k in ("GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS", "GENOMAD_B200_BOTH_STRANDS", "GENOMAD_B200_CONTIG_REDUCE"):
        os.environ.pop(k, None)
    _install(setattr, SumStub())
    tmp = Path(tmp)
    _run(tmp / "sample.fna", tmp / f"out_{world}_{reduce}", tmp / "h.npz", reduce)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("reduce", ["gather", "allreduce"])
@pytest.mark.parametrize("world", [2, 3])
def test_head_files_match_one_process(tmp_path, monkeypatch, world, reduce):
    fa = _fasta(tmp_path / "sample.fna")
    HS.write_head(tmp_path / "h.npz", C, 4)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS",
              "GENOMAD_B200_BOTH_STRANDS", "GENOMAD_B200_CONTIG_REDUCE"):
        monkeypatch.delenv(k, raising=False)
    _install(monkeypatch.setattr, SumStub())
    _run(fa, tmp_path / "one", tmp_path / "h.npz", "gather")
    o1 = _paths.NNOutputs("sample", tmp_path / "one")
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path), reduce), nprocs=world, join=True)
    ow = _paths.NNOutputs("sample", tmp_path / f"out_{world}_{reduce}")
    z1, zw = np.load(o1.nn_classification_head_npz_output), np.load(ow.nn_classification_head_npz_output)
    assert set(z1.files) == set(zw.files)
    for k in z1.files:
        if k == "predictions" and reduce == "allreduce":
            assert zw[k].dtype == np.float32 and zw[k].shape == z1[k].shape
            assert np.abs(zw[k] - z1[k]).max() <= 4 * np.finfo(np.float32).eps
        else:
            assert z1[k].dtype == zw[k].dtype and np.array_equal(z1[k], zw[k]), k
    if reduce == "gather":
        assert o1.nn_classification_head_output.read_bytes() == ow.nn_classification_head_output.read_bytes()
    assert o1.nn_classification_output.read_bytes() == ow.nn_classification_output.read_bytes() or reduce == "allreduce"


@pytest.mark.parametrize("world", [2, 3])
def test_train_head_refuses_more_than_one_process(tmp_path, monkeypatch, world):
    fa = _fasta(tmp_path / "sample.fna")
    lab = tmp_path / "l.tsv"
    lab.write_text("seq_name\tclass\nc0\ta\nc1\tb\n")
    monkeypatch.setenv("WORLD_SIZE", str(world))
    monkeypatch.setenv("RANK", "0")
    monkeypatch.setattr(train_head, "_make_classifier", lambda device: pytest.fail("no classifier may be built"))
    with pytest.raises(SystemExit) as e:
        train_head.main(fa, lab, tmp_path / "out", verbose=False)
    assert e.value.code == 1
    assert not (tmp_path / "out").exists()
