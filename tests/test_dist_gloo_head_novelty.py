"""
Gloo tests (CPU, world sizes 2 and 3) of the head's novelty file under torchrun: the window distances are reduced per contig by
the gather route (the file bitwise that of one process) or the allreduce route (fp32 re-association only).  One input has fewer
windows than ranks, so a rank classifies an empty shard.  Stub classifier and head: tests/head_stub.py, tests/test_novelty_cpu.py.
"""
import os
from pathlib import Path

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from genomad_b200 import _paths, nn_classification
from test_dist_gloo_head import SumStub, _free_port
from test_dist_gloo_head_outputs import _tiny
from test_dist_gloo_strands import _fasta
from test_novelty_cpu import StubNoveltyHead, write_novelty_head
import window_stub as WS

RUNS = {"sample": {}, "tiny": {"both_strands": True}}


def _install(setattr_):
    WS.install(setattr_, nn_classification, SumStub())
    setattr_(nn_classification, "_make_head", StubNoveltyHead)


def _run_all(tmp: Path, tag: str, reduce: str):
    for name, kw in RUNS.items():
        nn_classification.main(tmp / name / "sample.fna", tmp / f"{tag}_{name}", False, 128, False, 2, False, False,
                               contig_reduce=reduce, head=tmp / "h.npz", **kw)


def _worker(rank, world, port, tmp, reduce):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    for k in ("GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS", "GENOMAD_B200_BOTH_STRANDS",
              "GENOMAD_B200_CONTIG_REDUCE"):
        os.environ.pop(k, None)
    _install(setattr)
    _run_all(Path(tmp), f"w{world}", reduce)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("reduce", ["gather", "allreduce"])
@pytest.mark.parametrize("world", [2, 3])
def test_novelty_file_matches_one_process(tmp_path, monkeypatch, world, reduce):
    for d in RUNS:
        (tmp_path / d).mkdir()
    _fasta(tmp_path / "sample" / "sample.fna")
    _tiny(tmp_path / "tiny" / "sample.fna")
    write_novelty_head(tmp_path / "h.npz")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS",
              "GENOMAD_B200_BOTH_STRANDS", "GENOMAD_B200_CONTIG_REDUCE"):
        monkeypatch.delenv(k, raising=False)
    _install(monkeypatch.setattr)
    _run_all(tmp_path, "one", "gather")
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path), reduce), nprocs=world, join=True)
    for name in RUNS:
        o1 = _paths.NNOutputs("sample", tmp_path / f"one_{name}")
        ow = _paths.NNOutputs("sample", tmp_path / f"w{world}_{name}")
        z1, zw = np.load(o1.nn_classification_head_novelty_npz_output), np.load(ow.nn_classification_head_novelty_npz_output)
        assert set(z1.files) == set(zw.files)
        if reduce == "gather":
            for k in z1.files:
                assert z1[k].dtype == zw[k].dtype and np.array_equal(z1[k], zw[k]), (name, k)
            assert o1.nn_classification_head_novelty_output.read_bytes() == \
                ow.nn_classification_head_novelty_output.read_bytes()
        else:
            d1, dw = z1["distances"], zw["distances"]
            assert dw.dtype == np.float32 and dw.shape == d1.shape
            assert (np.abs(dw - d1) <= 4 * np.finfo(np.float32).eps * np.abs(d1)).all(), name
            assert np.array_equal(z1["contig_names"], zw["contig_names"])
        if name == "tiny":
            assert len(z1["contig_names"]) == 2
