"""
Gloo tests (CPU, world sizes 2 and 3) of embedding-clusters --index under torchrun, with the stand-ins of
tests/test_clusters_index_cpu.py: each rank holds the slots of its contiguous range of lists, rank 0 ORs the covering flags,
decides the block and sends the new representatives, every rank appends those of its lists, and rank 0 merges the final lists in
rank order.  The files rank 0 writes must be bitwise those of one process, also while some ranks' lists hold no representative.
"""
import os

import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from genomad_b200 import embedding_clusters as EC
from test_clusters_cpu import families
from test_clusters_index_cpu import install, setup
from test_dist_gloo_window_scores import _free_port


def _worker(rank, world, port, tmp, p, ix, block, nprobe):
    from pathlib import Path
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    install(setattr)
    EC.main(p, Path(tmp) / f"out_{world}", 0.9, False, block=block, index=ix, nprobe=nprobe)
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("block,nprobe", [(3, 2), (64, 1), (5, 6)])
def test_matches_one_process(tmp_path, monkeypatch, world, block, nprobe):
    for key in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(key, raising=False)
    install(monkeypatch.setattr)
    p, ix, _ = setup(tmp_path, families(8, 4, 0.25, 12), lists=6)
    EC.main(p, tmp_path / "one", 0.9, False, block=block, index=ix, nprobe=nprobe)
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path), str(p), str(ix), block, nprobe), nprocs=world, join=True)
    for ext in ("tsv", "npz"):
        a = (tmp_path / "one" / f"s_embedding_clusters.{ext}").read_bytes()
        b = (tmp_path / f"out_{world}" / f"s_embedding_clusters.{ext}").read_bytes()
        assert a == b, ext
