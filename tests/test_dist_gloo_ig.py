"""
Gloo tests (CPU, world sizes 2 and 3) of `--write-attributions --attribution-steps` under torchrun: every rank runs its
contiguous shard of the contig pass through the integrated-gradients calls (stub classifier, tests/test_ig_module_cpu.py),
rank 0 collects the attribution rows and the log_p_target rows in rank order (dist.collect_window_probs), and the NPZ it
writes must be bitwise that of one process.
"""
import os

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import window_stub as WS
from genomad_b200 import _paths, nn_classification
from test_dist_gloo_window_scores import _fasta, _free_port
from test_ig_module_cpu import IGStub


def _worker(rank, world, port, tmp):
    from pathlib import Path
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    for k in ("GENOMAD_B200_ATTRIBUTIONS", "GENOMAD_B200_ATTRIBUTION_STEPS", "GENOMAD_B200_ATTRIBUTION_BASELINE"):
        os.environ.pop(k, None)
    clf = IGStub()
    WS.install(setattr, nn_classification, clf)
    tmp = Path(tmp)
    nn_classification.main(tmp / "sample.fna", tmp / f"out_{world}", False, 128, False, 2, False, False,
                           write_attributions="virus", attribution_steps=8, attribution_baseline="N")
    np.save(tmp / f"seen_{world}_{rank}.npy", np.array([len(clf.windows_seen())]))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_ig_npz_matches_one_process(tmp_path, monkeypatch, world):
    fa = _fasta(tmp_path / "sample.fna")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "GENOMAD_B200_ATTRIBUTIONS", "GENOMAD_B200_ATTRIBUTION_STEPS",
              "GENOMAD_B200_ATTRIBUTION_BASELINE"):
        monkeypatch.delenv(k, raising=False)
    one = IGStub()
    WS.install(monkeypatch.setattr, nn_classification, one)
    nn_classification.main(fa, tmp_path / "one", False, 128, False, 2, False, False, write_attributions="virus",
                           attribution_steps=8, attribution_baseline="N")
    o1 = _paths.NNOutputs("sample", tmp_path / "one")
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    ow = _paths.NNOutputs("sample", tmp_path / f"out_{world}")
    z1, zw = np.load(o1.nn_classification_attributions_output), np.load(ow.nn_classification_attributions_output)
    assert set(z1.files) == set(zw.files) and "log_p_target" in z1.files
    for k in z1.files:
        assert z1[k].dtype == zw[k].dtype and np.array_equal(z1[k], zw[k]), k
    p1, pw = np.load(o1.nn_classification_npz_output), np.load(ow.nn_classification_npz_output)
    assert np.array_equal(p1["predictions"], pw["predictions"])
    seen = sum(int(np.load(tmp_path / f"seen_{world}_{r}.npy")[0]) for r in range(world))
    assert seen == len(one.windows_seen()) == len(z1["attributions"])
