"""
Gloo tests (CPU, world sizes 2 and 3) of the head's strand and window files under torchrun: the reverse pass reduces the head's
scores per contig by the gather route (bitwise one process) or the allreduce route (fp32 re-association only), and the head's
window rows, from the contig pass at stride 6000 and from the profile pass at another stride, are collected on rank 0 in window
order (bitwise one process on both routes).  One input has fewer windows than ranks, so a rank classifies an empty shard.
Stub classifier and head: tests/head_stub.py.
"""
import os
from pathlib import Path

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import head_stub as HS
from genomad_b200 import _paths, nn_classification
from test_dist_gloo_head import SumStub, _free_port, _install
from test_dist_gloo_strands import _fasta

C = 5
RUNS = {"strands_windows": dict(both_strands=True, write_window_scores=True),
        "profile": dict(window_stride=1000),
        "tiny": dict(both_strands=True, write_window_scores=True)}


def _tiny(path):
    """Two contigs of one window each: with three ranks, one shard is empty."""
    rng = np.random.default_rng(2)
    with open(path, "w") as fh:
        for i, n in enumerate((7000, 3000)):
            fh.write(f">t{i}\n" + np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)].tobytes().decode() + "\n")
    return path


def _run_all(tmp: Path, tag: str, reduce: str):
    for name, kw in RUNS.items():
        fa = tmp / ("tiny" if name == "tiny" else "sample") / "sample.fna"
        nn_classification.main(fa, tmp / f"{tag}_{name}", False, 128, False, 2, False, False, contig_reduce=reduce,
                               head=tmp / "h.npz", **kw)


def _worker(rank, world, port, tmp, reduce):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    for k in ("GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS", "GENOMAD_B200_BOTH_STRANDS",
              "GENOMAD_B200_CONTIG_REDUCE"):
        os.environ.pop(k, None)
    _install(setattr, SumStub())
    _run_all(Path(tmp), f"w{world}", reduce)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("reduce", ["gather", "allreduce"])
@pytest.mark.parametrize("world", [2, 3])
def test_head_strands_and_windows_match_one_process(tmp_path, monkeypatch, world, reduce):
    for d in ("sample", "tiny"):
        (tmp_path / d).mkdir()
    _fasta(tmp_path / "sample" / "sample.fna")
    _tiny(tmp_path / "tiny" / "sample.fna")
    HS.write_head(tmp_path / "h.npz", C, 4)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "GENOMAD_B200_WINDOW_SCORES", "GENOMAD_B200_EMBEDDINGS",
              "GENOMAD_B200_BOTH_STRANDS", "GENOMAD_B200_CONTIG_REDUCE"):
        monkeypatch.delenv(k, raising=False)
    _install(monkeypatch.setattr, SumStub())
    _run_all(tmp_path, "one", "gather")
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path), reduce), nprocs=world, join=True)
    for name, kw in RUNS.items():
        o1 = _paths.NNOutputs("sample", tmp_path / f"one_{name}")
        ow = _paths.NNOutputs("sample", tmp_path / f"w{world}_{name}")
        pairs = []
        if kw.get("both_strands"):
            pairs.append((o1.nn_classification_head_strands_npz_output, ow.nn_classification_head_strands_npz_output,
                          o1.nn_classification_head_strands_output, ow.nn_classification_head_strands_output, True))
        pairs.append((o1.nn_classification_head_windows_npz_output, ow.nn_classification_head_windows_npz_output,
                      o1.nn_classification_head_windows_output, ow.nn_classification_head_windows_output, False))
        for n1, nw, t1, tw, per_contig in pairs:
            z1, zw = np.load(n1), np.load(nw)
            assert set(z1.files) == set(zw.files)
            for k in z1.files:
                if per_contig and reduce == "allreduce" and k in nn_classification.STRANDS:
                    assert zw[k].dtype == np.float32 and zw[k].shape == z1[k].shape
                    assert np.abs(zw[k] - z1[k]).max() <= 4 * np.finfo(np.float32).eps, (name, k)
                else:
                    assert z1[k].dtype == zw[k].dtype and np.array_equal(z1[k], zw[k]), (name, k)
            if not per_contig or reduce == "gather":
                assert t1.read_bytes() == tw.read_bytes(), (name, t1.name)
        if name == "tiny":
            assert len(np.load(o1.nn_classification_head_windows_npz_output)["predictions"]) == 2
