"""
Gloo tests (CPU, world sizes 2 and 3) of the embedding-clusters module under torchrun, with the fp64 stand-ins of
tests/test_clusters_cpu.py: every rank holds all rows and covers each block against its shard of the representatives, rank 0
ORs the flags, runs the block step and sends the new representatives to every rank, and the final assignment is the neighbour
search's sharded route.  The files rank 0 writes must be bitwise those of one process, also while the early blocks have fewer
representatives than ranks (empty shards).
"""
import os

import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from genomad_b200 import embedding_clusters as EC
from test_clusters_cpu import families, install
from test_dist_gloo_window_scores import _free_port
from test_neighbours_cpu import write_npz


def _worker(rank, world, port, tmp, p, t, block):
    from pathlib import Path
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    install(setattr)
    EC.main(p, Path(tmp) / f"out_{world}", t, False, block=block, rep_chunk=2)
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("block", [3, 64])
def test_matches_one_process(tmp_path, monkeypatch, world, block):
    for key in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(key, raising=False)
    install(monkeypatch.setattr)
    p = write_npz(tmp_path / "s_nn_classification_embeddings.npz", 0, emb=families(8, 4, 0.25, 12))
    EC.main(p, tmp_path / "one", 0.9, False, block=block, rep_chunk=5)
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path), str(p), 0.9, block), nprocs=world, join=True)
    for ext in ("tsv", "npz"):
        a = (tmp_path / "one" / f"s_embedding_clusters.{ext}").read_bytes()
        b = (tmp_path / f"out_{world}" / f"s_embedding_clusters.{ext}").read_bytes()
        assert a == b, ext
