"""
Gloo tests (CPU, world sizes 2 and 3) of the embedding-neighbours module under torchrun: every rank searches its contiguous
reference shard with the fp64 stand-in (tests/test_neighbours_cpu.py), rank 0 receives the lists point to point and merges
them in rank order, and the files it writes must be bitwise those of one process -- also with a rank whose shard is empty.
"""
import os

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from genomad_b200 import embedding_neighbours as EN
from test_dist_gloo_window_scores import _free_port
from test_neighbours_cpu import install, rows, write_npz


def _worker(rank, world, port, tmp, q, r, k):
    from pathlib import Path
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    install(setattr)
    EN.main(q, r if r else None, Path(tmp) / f"out_{world}", k, False)
    dist.destroy_process_group()


def _run(tmp_path, monkeypatch, world, q, r, k):
    for key in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(key, raising=False)
    install(monkeypatch.setattr)
    EN.main(q, r, tmp_path / "one", k, False)
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path), str(q), str(r) if r else "", k), nprocs=world, join=True)
    prefix = EN.output_prefix(q)
    for ext in ("tsv", "npz"):
        a = (tmp_path / "one" / f"{prefix}_embedding_neighbours.{ext}").read_bytes()
        b = (tmp_path / f"out_{world}" / f"{prefix}_embedding_neighbours.{ext}").read_bytes()
        assert a == b, ext


@pytest.mark.parametrize("world", [2, 3])
def test_all_vs_all_matches_one_process(tmp_path, monkeypatch, world):
    e = rows(11, 5)
    e[9] = e[2]                                     # a tie across shards
    q = write_npz(tmp_path / "s_nn_classification_embeddings.npz", 0, emb=e)
    _run(tmp_path, monkeypatch, world, q, None, 4)


@pytest.mark.parametrize("world", [2, 3])
def test_reference_with_an_empty_shard_matches_one_process(tmp_path, monkeypatch, world):
    q = write_npz(tmp_path / "q_nn_classification_embeddings.npz", 6, 1)
    r = write_npz(tmp_path / "r.npz", world - 1, 2)         # fewer reference rows than ranks: the last shard is empty
    _run(tmp_path, monkeypatch, world, q, r, 3)
    z = np.load(tmp_path / f"out_{world}" / "q_embedding_neighbours.npz")
    assert np.all(z["neighbour_index"][:, world - 1:] == -1)
