"""
Gloo tests (CPU, world sizes 2 and 3) of the per-contig embedding carry chain in genomad_b200.dist: every rank streams its shard
in chunks through EmbeddingShard with a NumPy sequential fp32 reducer, the carry runs from rank 0 upward, and the gathered
per-contig means must be bitwise the one-process result.
"""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from genomad_b200 import dist as gdist

WIDTH = 512


def np_segment_sum_rows(rows: np.ndarray, offsets: np.ndarray, carry=None):
    """NumPy statement of gnm_segment_sum_rows: per column, one fp32 running sum in row order; segment 0 starts from `carry`;
    returns (sums [k, 512], running sum of the last segment)."""
    k = len(offsets) - 1
    sums = np.zeros((k, rows.shape[1]), np.float32)
    for c in range(k):
        s = np.array(carry, np.float32).copy() if (c == 0 and carry is not None) else np.zeros(rows.shape[1], np.float32)
        for i in range(offsets[c], offsets[c + 1]):
            s = (s + rows[i]).astype(np.float32)
        sums[c] = s
    return sums, (sums[k - 1].copy() if k else np.zeros(rows.shape[1], np.float32))


def torch_reducer(rows, offsets, carry):
    s, c = np_segment_sum_rows(rows.numpy(), offsets.numpy(), None if carry is None else carry.numpy())
    return torch.from_numpy(s), torch.from_numpy(c)


def one_process_means(rows: np.ndarray, offsets: np.ndarray) -> np.ndarray:
    sums, _ = np_segment_sum_rows(rows, offsets)
    cnt = np.maximum(np.diff(offsets), 1).astype(np.float32)
    return sums / cnt[:, None]


def _rows(n: int) -> np.ndarray:
    rng = np.random.default_rng(5)
    r = rng.standard_normal((n, WIDTH)).astype(np.float32) * 3
    r[r < 0] = 0                                                          # post-ReLU-like: many exact zeros
    return r


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def run_shard(rows, offsets, start, end, chunk, info):
    sh = gdist.EmbeddingShard(offsets, start, end, torch_reducer)
    for a in range(start, end, chunk):
        sh.add(torch.from_numpy(rows[a: min(end, a + chunk)].copy()))
    lo, means = sh.finish(info)
    return gdist.gather_contig_means(lo, means, len(offsets) - 1, info)


def _worker(rank, world, port, tmp, counts, chunk):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    info = gdist.init_process_group_if_needed("gloo")
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    n = int(offsets[-1])
    rows = _rows(n)
    s, e = gdist.shard_bounds(n, world, rank)
    out = run_shard(rows, offsets, s, e, chunk, info)
    if rank == 0:
        np.save(os.path.join(tmp, "means.npy"), out.numpy())
    else:
        assert out is None
    dist.destroy_process_group()


CASES = {
    "contig_spans_whole_shard": ([2, 20, 1, 3], 3),              # the 20-window contig covers all of rank 1's shard (and more)
    "fewer_windows_than_ranks": ([1, 0, 1], 1),                   # n < world: a shard with no windows, and an empty contig
    "one_window_contigs_on_edges": ([3, 1, 1, 4, 1, 1, 2], 2),   # one-window contigs where the shards meet
    "single_window": ([1, 1, 0, 1, 1, 1, 1, 1], 2),               # --single-window: every contig has at most one window
    "chunk_inside_contig": ([1, 17, 2, 0, 5], 4),
}


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("case", sorted(CASES))
def test_carry_chain_matches_one_process(tmp_path, world, case):
    counts, chunk = CASES[case]
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path), counts, chunk), nprocs=world, join=True)
    got = np.load(tmp_path / "means.npy")
    ref = one_process_means(_rows(int(offsets[-1])), offsets)
    assert got.dtype == np.float32 and got.shape == (len(counts), WIDTH)
    assert np.array_equal(got, ref)
    assert not got[np.asarray(counts) == 0].any()


@pytest.mark.parametrize("counts", [[5, 1, 7, 2, 0, 9], [30], [1] * 12, [0, 4, 0, 0, 3]])
@pytest.mark.parametrize("chunk", [1, 2, 3, 5, 64])
def test_segment_sum_rows_statement_is_chunking_invariant(counts, chunk):
    """Chained calls over consecutive row blocks (segments spanning several blocks, blocks inside one segment) give the bits of
    one call: what the module relies on when it reduces chunk by chunk."""
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    rows = _rows(int(offsets[-1]))
    sh = gdist.EmbeddingShard(offsets, 0, int(offsets[-1]), torch_reducer)
    for a in range(0, int(offsets[-1]), chunk):
        sh.add(torch.from_numpy(rows[a: a + chunk].copy()))
    lo, means = sh.finish(gdist.DistInfo())
    got = gdist.gather_contig_means(lo, means, len(counts), gdist.DistInfo()).numpy()
    assert np.array_equal(got, one_process_means(rows, offsets))


def test_float_order_matters():
    """The bar is bitwise for a reason: summing the same rows in another order changes the bits, so a tree or a re-ordered
    chain would be caught."""
    rows = np.array([[1e8], [1.0], [-1e8], [1.0]], np.float32)
    s, _ = np_segment_sum_rows(rows, np.array([0, 4]))
    assert s[0, 0] == np.float32(1.0)                        # ((1e8 + 1) - 1e8) + 1 in fp32
    assert np.float32(rows.sum(dtype=np.float64)) == np.float32(2.0)
