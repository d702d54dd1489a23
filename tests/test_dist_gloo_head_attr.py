"""
Gloo test (CPU, world sizes 2 and 3) of `nn-classification --head --write-head-attributions` under torchrun: each rank's
attribution rows travel to rank 0 in window order, so the head attributions file (and the head and main outputs) are
bitwise those of one process.  Stub classifier and head: tests/test_head_attr_module_cpu.py.
"""
import os

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import window_stub as WS
from genomad_b200 import _paths, nn_classification
from test_dist_gloo_head import SumStub, _free_port
from test_dist_gloo_strands import _fasta
from test_head_attr_module_cpu import AttrHead

ENV = ("RANK", "WORLD_SIZE", "LOCAL_RANK", "GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS", "GENOMAD_B200_BOTH_STRANDS",
       "GENOMAD_B200_CONTIG_REDUCE", "GENOMAD_B200_ATTRIBUTIONS", "GENOMAD_B200_HEAD_ATTRIBUTIONS",
       "GENOMAD_B200_ATTRIBUTION_STEPS", "GENOMAD_B200_ATTRIBUTION_BASELINE")


def _install(setattr_, clf):
    WS.install(setattr_, nn_classification, clf)
    setattr_(nn_classification, "_make_head", AttrHead)


def _run(fa, out, head):
    nn_classification.main(fa, out, False, 128, False, 2, False, False, head=head, write_head_attributions="k1",
                           attribution_steps=4)


def _worker(rank, world, port, tmp):
    from pathlib import Path
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    for k in ENV[3:]:
        os.environ.pop(k, None)
    _install(setattr, SumStub())
    tmp = Path(tmp)
    _run(tmp / "sample.fna", tmp / f"out_{world}", tmp / "h.npz")
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_head_attributions_match_one_process(tmp_path, monkeypatch, world):
    import head_stub as HS
    fa = _fasta(tmp_path / "sample.fna")
    HS.write_head(tmp_path / "h.npz", 4, 6)
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    _install(monkeypatch.setattr, SumStub())
    _run(fa, tmp_path / "one", tmp_path / "h.npz")
    o1 = _paths.NNOutputs("sample", tmp_path / "one")
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    ow = _paths.NNOutputs("sample", tmp_path / f"out_{world}")
    for path in ("nn_classification_head_attributions_output", "nn_classification_head_npz_output"):
        z1, zw = np.load(getattr(o1, path)), np.load(getattr(ow, path))
        assert z1.files == zw.files
        for k in z1.files:
            assert z1[k].dtype == zw[k].dtype and np.array_equal(z1[k], zw[k]), (path, k)
    assert len(np.load(o1.nn_classification_head_attributions_output)["attributions"]) > world
    assert o1.nn_classification_output.read_bytes() == ow.nn_classification_output.read_bytes()
    assert o1.nn_classification_head_output.read_bytes() == ow.nn_classification_head_output.read_bytes()
