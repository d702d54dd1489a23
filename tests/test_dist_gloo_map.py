"""
Gloo tests (CPU, world sizes 2 and 3) of the embedding-map module under torchrun, with the stand-ins of tests/test_map_cpu.py:
every rank searches its shard of the rows for the all-vs-all lists, rank 0 merges them and lays out the map.  The files rank 0
writes must be bitwise those of one process.
"""
import os

import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from genomad_b200 import embedding_map as EM
from test_dist_gloo_window_scores import _free_port
from test_map_cpu import install
from test_neighbours_cpu import rows, write_npz


def _worker(rank, world, port, tmp, p):
    from pathlib import Path
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    install(setattr)
    EM.main(p, Path(tmp) / f"out_{world}", 6, 40, 5, False)
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_matches_one_process(tmp_path, monkeypatch, world):
    for key in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(key, raising=False)
    install(monkeypatch.setattr)
    p = write_npz(tmp_path / "s_nn_classification_embeddings.npz", 0, emb=rows(23, 4))
    EM.main(p, tmp_path / "one", 6, 40, 5, False)
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path), str(p)), nprocs=world, join=True)
    for ext in ("tsv", "npz"):
        a = (tmp_path / "one" / f"s_embedding_map.{ext}").read_bytes()
        b = (tmp_path / f"out_{world}" / f"s_embedding_map.{ext}").read_bytes()
        assert a == b, ext
