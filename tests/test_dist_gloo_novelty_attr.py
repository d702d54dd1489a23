"""
Gloo tests (CPU, world sizes 2 and 3) of --write-novelty-attributions and --write-window-novelty under torchrun: the
attribution rows, distances and targets and the window novelty rows reach rank 0 by the attribution route
(gdist.collect_window_probs), so both files are bitwise those of one process.  One input has fewer windows than ranks, so a
rank has an empty shard.  Stubs: tests/test_novelty_attr_module_cpu.py.
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
from test_novelty_attr_module_cpu import NovAttrHead
from test_novelty_cpu import write_novelty_head
import window_stub as WS

RUNS = {"sample": {}, "tiny": {"attribution_steps": 2}, "stride": {"window_stride": 1000}}
ENV = ("GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS", "GENOMAD_B200_BOTH_STRANDS", "GENOMAD_B200_CONTIG_REDUCE",
       "GENOMAD_B200_NOVELTY_ATTRIBUTIONS", "GENOMAD_B200_WINDOW_NOVELTY", "GENOMAD_B200_ATTRIBUTION_STEPS")


def _install(setattr_):
    WS.install(setattr_, nn_classification, SumStub())
    setattr_(nn_classification, "_make_head", NovAttrHead)


def _run_all(tmp: Path, tag: str):
    for name, kw in RUNS.items():
        src = "tiny" if name == "tiny" else "sample"
        nn_classification.main(tmp / src / "sample.fna", tmp / f"{tag}_{name}", False, 128, False, 2, False, False,
                               head=tmp / "h.npz", write_novelty_attributions=True, write_window_novelty=True, **kw)


def _worker(rank, world, port, tmp):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    for k in ENV:
        os.environ.pop(k, None)
    _install(setattr)
    _run_all(Path(tmp), f"w{world}")
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_novelty_attr_files_match_one_process(tmp_path, monkeypatch, world):
    for d in ("sample", "tiny"):
        (tmp_path / d).mkdir()
    _fasta(tmp_path / "sample" / "sample.fna")
    _tiny(tmp_path / "tiny" / "sample.fna")
    write_novelty_head(tmp_path / "h.npz")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK") + ENV:
        monkeypatch.delenv(k, raising=False)
    _install(monkeypatch.setattr)
    _run_all(tmp_path, "one")
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    for name in RUNS:
        o1 = _paths.NNOutputs("sample", tmp_path / f"one_{name}")
        ow = _paths.NNOutputs("sample", tmp_path / f"w{world}_{name}")
        for p1, pw in ((o1.nn_classification_head_novelty_attributions_output,
                        ow.nn_classification_head_novelty_attributions_output),
                       (o1.nn_classification_head_novelty_windows_npz_output,
                        ow.nn_classification_head_novelty_windows_npz_output)):
            z1, zw = np.load(p1), np.load(pw)
            assert set(z1.files) == set(zw.files)
            for k in z1.files:
                assert z1[k].dtype == zw[k].dtype and np.array_equal(z1[k], zw[k], equal_nan=z1[k].dtype.kind == "f"), (name, k)
        assert o1.nn_classification_head_novelty_windows_output.read_bytes() == \
            ow.nn_classification_head_novelty_windows_output.read_bytes()
        if name == "tiny":
            assert len(np.load(o1.nn_classification_head_novelty_attributions_output)["contig_names"]) == 2
