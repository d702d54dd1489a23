"""
Multi-GPU plumbing for nn-classification: one process per GPU (torchrun), windows sharded in
contiguous blocks, one exchange step at the end over NCCL (NVLink/NVSwitch).

The reference has no distributed code at all (single process, GPUs hidden --
reference genomad/modules/nn_classification.py:8); what has to be preserved is its result:
``tf.math.segment_mean`` over ALL windows of a contig in FASTA order (nn_classification.py:319-320).
Windows are independent until that mean, so the only collective is on per-window probabilities
(12 B/window) or per-contig partial sums (16 B/contig):

  * gather_window_probs : all_gather of the [W_local, 3] shards -> every rank holds [W, 3] in window
                          order; the segment mean is then computed exactly as on one GPU (bitwise
                          identical outputs for any world size).  Default.
  * allreduce_partials  : each rank reduces its own shard to [n_contigs, 4] = (sum p, count) with
                          gnm_segment_sum, then one all_reduce(SUM); used when contigs are long and
                          n_contigs << W (BASELINE config 4).  Order-free: differs from the gather
                          variant by fp32 re-association only (~1e-7).

Everything here is backend-agnostic (tensors in, tensors out) so the logic is covered on CPU with
gloo at world_size 2 (tests/test_dist_gloo.py); in production the backend is NCCL.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np


@dataclass
class DistInfo:
    rank: int = 0
    world_size: int = 1
    local_rank: int = 0

    @property
    def is_main(self) -> bool:
        return self.rank == 0


def dist_info_from_env() -> DistInfo:
    return DistInfo(int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)),
                    int(os.environ.get("LOCAL_RANK", 0)))


def init_process_group_if_needed(backend: Optional[str] = None) -> DistInfo:
    """Initialise torch.distributed from the torchrun environment (no-op for a single process)."""
    info = dist_info_from_env()
    if info.world_size > 1:
        import torch
        import torch.distributed as dist
        if not dist.is_initialized():
            if backend is None:
                backend = "nccl" if torch.cuda.is_available() else "gloo"
            if backend == "nccl":
                torch.cuda.set_device(info.local_rank)
                dist.init_process_group(backend=backend, device_id=torch.device("cuda", info.local_rank))
            else:
                dist.init_process_group(backend=backend)
    return info


def broadcast_object(obj, info: DistInfo, src: int = 0):
    """Rank `src`'s Python object on every rank (no-op for a single process).  Used for control-flow decisions that
    depend on the file system: only rank 0 looks, everybody follows."""
    if info.world_size == 1:
        return obj
    import torch.distributed as dist
    box = [obj if info.rank == src else None]
    dist.broadcast_object_list(box, src=src)
    return box[0]


def barrier(info: DistInfo) -> None:
    if info.world_size > 1:
        import torch.distributed as dist
        dist.barrier()


def shard_bounds(n_items: int, world_size: int, rank: int) -> Tuple[int, int]:
    """Contiguous, balanced block of [0, n_items) owned by `rank` (first n % world ranks get one extra)."""
    base, extra = divmod(n_items, world_size)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def local_offsets(offsets: np.ndarray, start: int, end: int) -> np.ndarray:
    """Contig window offsets [n_contigs+1] (global) -> offsets into the local shard [start, end)."""
    return (np.clip(offsets.astype(np.int64), start, end) - start).astype(np.int32)


def gather_window_probs(local_probs, n_total: int, world_size: int, group=None):
    """all_gather of contiguous shards of unequal length [W_local, width] -> [n_total, width] in global window order."""
    import torch
    import torch.distributed as dist
    if world_size == 1:
        return local_probs
    max_len = -(-n_total // world_size)
    width = local_probs.shape[1]
    buf = torch.zeros((max_len, width), dtype=local_probs.dtype, device=local_probs.device)
    buf[: local_probs.shape[0]] = local_probs
    out = torch.empty((world_size * max_len, width), dtype=local_probs.dtype, device=local_probs.device)
    dist.all_gather_into_tensor(out, buf, group=group)
    parts = []
    for r in range(world_size):
        s, e = shard_bounds(n_total, world_size, r)
        parts.append(out[r * max_len: r * max_len + (e - s)])
    return torch.cat(parts, dim=0)


def collect_window_probs(local_probs, n_total: int, info: "DistInfo", send=None, recv=None):
    """Contiguous shards of per-window rows [W_local, width] -> [n_total, width] in global window order on rank 0 (None on the
    other ranks): each rank sends its shard to rank 0, which receives them in rank order.  Only rank 0 ever holds every window
    (a score profile can have far more windows than the contig pass).  Any row width: the class scores (3) or the
    attributions (5,997); a rank without windows passes a [0, width] tensor."""
    import torch
    if info.world_size == 1:
        return local_probs
    send = send or (lambda t, dst: _p2p_send(t, dst))
    recv = recv or (lambda t, src: _p2p_recv(t, src))
    if not info.is_main:
        if local_probs.shape[0]:
            send(local_probs.contiguous(), 0)
        return None
    parts = [local_probs]
    for r in range(1, info.world_size):
        s, e = shard_bounds(n_total, info.world_size, r)
        if e > s:
            buf = torch.empty((e - s, local_probs.shape[1]), dtype=local_probs.dtype, device=local_probs.device)
            recv(buf, r)
            parts.append(buf)
    return torch.cat(parts, dim=0)


def allreduce_partials(partials, world_size: int, group=None):
    """[n_contigs, C + 1] per-rank (sum p0, ..., sum p_{C-1}, count) -> global; then mean = sums / count."""
    import torch.distributed as dist
    if world_size > 1:
        dist.all_reduce(partials, op=dist.ReduceOp.SUM, group=group)
    return partials


def finish_mean(partials):
    """[n_contigs, C + 1] (sums, count) -> [n_contigs, C] means."""
    cnt = partials[:, -1:].clamp(min=1)
    return partials[:, :-1] / cnt


# ------------------------------------------------------------------------------------------------ per-contig embeddings
# Per-contig mean embeddings must not depend on the number of GPUs either, but an all-gather of the [W, 512] window embeddings
# is out of the question (100 GB at 50 M windows).  Instead every rank sums its rows per contig with a carry chain:
#   * interior contigs (those that begin on the rank) are reduced from zero as the rank's chunks arrive;
#   * the HEAD FRAGMENT -- the rows of a contig that began on an earlier rank -- is kept unreduced (bounded by the longest
#     contig: 167 k windows, 333 MB for a 1 Gbp chromosome);
#   * at the end a carry runs from rank 0 upward (point-to-point): rank r receives the running sum of its head contig, reduces the
#     head fragment seeded with it, and passes on that running sum if the contig continues past its shard, else the running sum
#     of its own last contig;
#   * the rank that holds a contig's last window completes it; the means (sum / count, fp32) are gathered to rank 0.
# Every column is one fp32 running sum in window order however the rows are split, so the result is bitwise the one-process
# result.  `reducer(rows [R, 512], offsets int32 [k + 1], carry [512] or None) -> (sums [k, 512], carry [512])` is the segment sum
# (Classifier.segment_sum_rows on the GPU; a NumPy statement in the CPU tests).

def _contig_of(offsets: np.ndarray, w: int) -> int:
    """Index of the (non-empty) contig that holds window w."""
    return int(np.searchsorted(offsets, w, side="right")) - 1


class EmbeddingShard:
    """Streams one rank's rows [start, end) of the global window list and reduces them per contig (see above)."""

    def __init__(self, offsets: np.ndarray, start: int, end: int, reducer, device="cpu", width: int = 512):
        import torch
        self.offsets = np.asarray(offsets, dtype=np.int64)
        self.start, self.end, self.reducer, self.width = start, end, reducer, width
        self.device = torch.device(device)
        self.pos = start
        self.head = -1                                   # contig of the head fragment, -1 = none
        self.head_end = start                            # rows [start, head_end) are the head fragment
        if start < end:
            c = _contig_of(self.offsets, start)
            if self.offsets[c] < start:
                self.head, self.head_end = c, min(end, int(self.offsets[c + 1]))
        self.head_rows = []
        # contigs completed on this rank: those whose last window lies in [start, end) -- a contiguous index range
        self.lo = int(np.searchsorted(self.offsets[1:], start, side="right"))
        self.hi = int(np.searchsorted(self.offsets[1:], end, side="right"))
        self.sums = torch.zeros((self.hi - self.lo, width), dtype=torch.float32, device=self.device)
        self.carry = None                                # running sum of the interior contig that holds row pos - 1
        self._torch = torch

    def add(self, rows) -> None:
        """The next rows of the shard, in order (any split into calls gives the same result)."""
        a, b = self.pos, self.pos + rows.shape[0]
        assert b <= self.end
        self.pos = b
        sums = self.sums
        if a < self.head_end:                            # head fragment: kept as is (a copy: the caller reuses its buffer)
            k = min(b, self.head_end) - a
            self.head_rows.append(rows[:k].clone())
            rows, a = rows[k:], a + k
        if a >= b:
            return
        off = self.offsets
        ca, cb = _contig_of(off, a), _contig_of(off, b - 1)
        seg = (np.clip(off[ca: cb + 2], a, b) - a).astype(np.int32)
        carry = self.carry if off[ca] < a else None      # segment 0 continues the previous rows' contig
        s, self.carry = self.reducer(rows, self._torch.from_numpy(seg).to(self.device), carry)
        done = cb + 1 if off[cb + 1] <= b else cb         # contigs ca .. done-1 end inside these rows
        if done > ca:
            sums[ca - self.lo: done - self.lo] = s[: done - ca]

    def finish(self, info: "DistInfo", send=None, recv=None):
        """Run the carry chain; returns (first completed contig, means [hi - lo, width]) of this rank."""
        import torch
        assert self.pos == self.end, "EmbeddingShard.finish before all rows were added"
        dev = self.device
        send = send or (lambda t, dst: _p2p_send(t, dst))
        recv = recv or (lambda t, src: _p2p_recv(t, src))
        carry_in = torch.zeros(self.width, dtype=torch.float32, device=dev)
        if info.rank > 0:
            recv(carry_in, info.rank - 1)
        out = self.carry if self.carry is not None else torch.zeros_like(carry_in)
        if self.start == self.end:
            out = carry_in                               # no rows: pass the running sum on unchanged
        elif self.head >= 0:
            rows = torch.cat(self.head_rows) if self.head_rows else torch.zeros((0, self.width), dtype=torch.float32, device=dev)
            seg = torch.tensor([0, rows.shape[0]], dtype=torch.int32, device=dev)
            s, run = self.reducer(rows, seg, carry_in)
            if int(self.offsets[self.head + 1]) > self.end:
                out = run                                # the head contig also covers the whole shard: forward its carry
            else:
                self.sums[self.head - self.lo] = s[0]
        if info.rank + 1 < info.world_size:
            send(out.contiguous(), info.rank + 1)
        cnt = np.diff(self.offsets)[self.lo: self.hi].astype(np.float32)
        cnt_t = torch.from_numpy(np.maximum(cnt, 1.0)).to(dev)
        return self.lo, self.sums / cnt_t[:, None]


def _p2p_send(t, dst):
    import torch.distributed as dist
    dist.send(t, dst)


def _p2p_recv(t, src):
    import torch.distributed as dist
    dist.recv(t, src)


def gather_contig_means(lo: int, means, n_contigs: int, info: DistInfo, group=None):
    """Each rank's completed contigs [lo, lo + len) -> [n_contigs, width] on rank 0 (None on the others).  Contigs no rank
    completed (no windows) stay zero."""
    import torch
    import torch.distributed as dist
    width = means.shape[1]
    if info.world_size == 1:
        out = torch.zeros((n_contigs, width), dtype=torch.float32, device=means.device)
        out[lo: lo + means.shape[0]] = means
        return out
    meta = torch.tensor([lo, means.shape[0]], dtype=torch.int64, device=means.device)
    metas = [torch.empty_like(meta) for _ in range(info.world_size)]
    dist.all_gather(metas, meta, group=group)
    cap = max(1, max(int(m[1]) for m in metas))
    buf = torch.zeros((cap, width), dtype=torch.float32, device=means.device)
    buf[: means.shape[0]] = means
    parts = [torch.empty_like(buf) for _ in range(info.world_size)]
    dist.all_gather(parts, buf, group=group)
    if not info.is_main:
        return None
    out = torch.zeros((n_contigs, width), dtype=torch.float32, device=means.device)
    for m, p in zip(metas, parts):
        a, k = int(m[0]), int(m[1])
        out[a: a + k] = p[:k]
    return out
