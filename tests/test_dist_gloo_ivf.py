"""
Gloo tests (CPU, world sizes 2 and 3) of embedding-neighbours (all-vs-all and against a reference) and embedding-map
--index under torchrun, with the stand-ins of
tests/test_ivf_cpu.py: every rank searches a contiguous range of the index's lists, balanced by rows, and rank 0 merges in rank
order.  The files rank 0 writes must be bitwise those of one process.
"""
import os

import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from genomad_b200 import embedding_index as EI, embedding_map as EM, embedding_neighbours as EN
from test_dist_gloo_window_scores import _free_port
from test_ivf_cpu import install as install_ivf
from test_map_cpu import install as install_map
from test_neighbours_cpu import write_npz


def install(setattr_):
    install_map(setattr_)
    install_ivf(setattr_)


def _worker(rank, world, port, tmp, p, ix, q):
    from pathlib import Path
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    install(setattr)
    EN.main(p, None, Path(tmp) / f"n_{world}", 4, False, index=ix, nprobe=3)
    EM.main(p, Path(tmp) / f"m_{world}", 5, 30, 2, False, index=ix, nprobe=3)
    EN.main(q, p, Path(tmp) / f"r_{world}", 4, False, index=ix, nprobe=2)
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_matches_one_process(tmp_path, monkeypatch, world):
    for key in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(key, raising=False)
    install(monkeypatch.setattr)
    p = write_npz(tmp_path / "s_nn_classification_embeddings.npz", 37, 4)
    EI.main(p, tmp_path / "ix", 7, 3, 0, False)
    ix = tmp_path / "ix" / "s_embedding_index.npz"
    EN.main(p, None, tmp_path / "n_one", 4, False, index=ix, nprobe=3)
    EM.main(p, tmp_path / "m_one", 5, 30, 2, False, index=ix, nprobe=3)
    q = write_npz(tmp_path / "q_nn_classification_embeddings.npz", 9, 8)
    EN.main(q, p, tmp_path / "r_one", 4, False, index=ix, nprobe=2)
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path), str(p), str(ix), str(q)), nprocs=world, join=True)
    for d, stem in (("n", "s_embedding_neighbours"), ("m", "s_embedding_map"), ("r", "q_embedding_neighbours")):
        for ext in ("tsv", "npz"):
            a = (tmp_path / f"{d}_one" / f"{stem}.{ext}").read_bytes()
            b = (tmp_path / f"{d}_{world}" / f"{stem}.{ext}").read_bytes()
            assert a == b, (stem, ext)
