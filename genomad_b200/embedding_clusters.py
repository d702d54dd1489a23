"""
``embedding-clusters`` module: greedy clustering of the sequences of an embeddings file written by ``nn-classification
--write-embeddings`` at a cosine-similarity threshold t, the dereplication of CD-HIT, MMseqs2 or vOTU pipelines carried out in
the encoder's embedding space.  Sequences are taken in file order; a sequence is a representative iff its similarity to every
earlier representative is below t (the first sequence always is), and every other sequence joins the representative it is most
similar to (ties to the earlier one), which scores >= t by construction.  The representative of a group is therefore its first
member in file order: sort the FASTA by length first to make the longest sequence the representative, as CD-HIT does.

s(j, i) is the similarity gnm_embedding_neighbours returns with the sequence being placed, j, as the query and the candidate
representative, i, as the reference (include/gnm.h; it is not bitwise symmetric).  Rows stay on the device for the whole run
and are processed in blocks of ``block`` rows:
  * covering: a row is covered when its best representative of the earlier blocks scores >= t -- engine.embedding_neighbours
    at k = 1 against the representatives, ``rep_chunk`` rows per call, the flags ORed;
  * the block step (engine.cluster_block, gnm_cluster_block): the uncovered rows decided against the block itself, in order,
    from a tensor-core threshold mask computed by the search's own mainloop;
  * final assignment: every non-representative searched at k = 1 against all representatives (embedding_neighbours.search).
The result depends only on the rows, their order and t (rounded once to fp32): not on the block size, the chunk size or the
GPU count.  Under torchrun every rank holds all rows; each rank searches the block against its contiguous shard of the
representatives and sends its flags to rank 0, which ORs them, runs the block step and sends the new representatives to every
rank; the final assignment is embedding_neighbours.search's sharding and rank-order merge.  DESIGN.md, "Embedding clusters".

Outputs in OUTPUT, <prefix> = the input file's stem without ``_nn_classification_embeddings``:
    <prefix>_embedding_clusters.tsv   seq_name, representative, cosine_similarity (6 decimals), one line per sequence in input
                                      order; a representative names itself with 1.000000
    <prefix>_embedding_clusters.npz   seq_names, representative_index int64 [n], similarity float32 [n] (1 for a
                                      representative), representatives int64 [R] ascending, cluster_size int64 [R],
                                      min_similarity float64 (the fp32 threshold applied)
"""
from __future__ import annotations

from pathlib import Path
from typing import Optional, Tuple

import numpy as np

from . import dist, engine, utils
from . import embedding_neighbours as EN

_HEADER = "seq_name\trepresentative\tcosine_similarity\n"


def output_paths(input_npz, output_dir) -> Tuple[Path, Path]:
    prefix = EN.output_prefix(input_npz)
    out = Path(output_dir)
    return out / f"{prefix}_embedding_clusters.tsv", out / f"{prefix}_embedding_clusters.npz"


def _covered(blk, rep_rows, thr: float, rep_chunk: int):
    """uint8 [b]: 1 where some row of rep_rows has similarity >= thr with the block row (the row as the query)."""
    import torch
    cov = torch.zeros(blk.shape[0], dtype=torch.uint8, device=blk.device)
    for a in range(0, rep_rows.shape[0], rep_chunk):
        sim, _ = engine.embedding_neighbours(blk, rep_rows[a:a + rep_chunk], 1)
        cov |= (sim[:, 0] >= thr).to(torch.uint8)
    return cov


def _block_step(blk, rep_rows, thr: float, rep_chunk: int, info):
    """The block's new representatives (block-local int64 on the device, ascending), the same on every rank."""
    import torch
    s, e = dist.shard_bounds(rep_rows.shape[0], info.world_size, info.rank)
    cov = _covered(blk, rep_rows[s:e], thr, rep_chunk)
    if info.world_size == 1:
        return engine.cluster_block(blk, cov, thr)
    count = torch.zeros(1, dtype=torch.int64, device=blk.device)
    if not info.is_main:
        dist._p2p_send(cov, 0)
        dist._p2p_recv(count, 0)
        new = torch.empty(int(count.item()), dtype=torch.int64, device=blk.device)
        if new.numel():
            dist._p2p_recv(new, 0)
        return new
    part = torch.empty_like(cov)
    for src in range(1, info.world_size):
        dist._p2p_recv(part, src)
        cov |= part
    new = engine.cluster_block(blk, cov, thr)
    count[0] = new.numel()
    for dst in range(1, info.world_size):
        dist._p2p_send(count, dst)
        if new.numel():
            dist._p2p_send(new.contiguous(), dst)
    return new


def cluster(emb: np.ndarray, min_similarity: float, info, block: int = engine.CLUSTER_MAX_BLOCK,
            rep_chunk: int = engine.NEIGHBOURS_CHUNK) -> Optional[Tuple[np.ndarray, np.ndarray, np.ndarray]]:
    """Greedy clustering of the rows of emb (float32 [n, 512]) at min_similarity.  Returns, on rank 0, (representative_index
    int64 [n], similarity float32 [n], representatives int64 [R]); None on the other ranks."""
    import torch
    thr = engine.cluster_threshold(min_similarity)
    if not 1 <= block <= engine.CLUSTER_MAX_BLOCK:
        raise ValueError(f"block must be in [1, {engine.CLUSTER_MAX_BLOCK}], not {block}")
    if rep_chunk < 1:
        raise ValueError(f"rep_chunk must be >= 1, not {rep_chunk}")
    dev = EN._device(info)
    n = emb.shape[0]
    x = torch.from_numpy(emb).to(dev)
    rep_rows = torch.empty_like(x)                 # the representatives' rows, in order: appended once, never re-uploaded
    reps = torch.empty(n, dtype=torch.int64, device=dev)
    n_rep = 0
    for a in range(0, n, block):
        blk = x[a: min(n, a + block)]
        new = _block_step(blk, rep_rows[:n_rep], thr, rep_chunk, info)
        m = new.numel()
        rep_rows[n_rep: n_rep + m] = blk[new]
        reps[n_rep: n_rep + m] = new + a
        n_rep += m
    reps = reps[:n_rep]
    is_rep = torch.zeros(n, dtype=torch.bool, device=dev)
    is_rep[reps] = True
    members = torch.nonzero(~is_rep).flatten()
    res = EN.search(x[members], rep_rows[:n_rep], 1, info) if members.numel() else (np.empty((0, 1), np.float32),
                                                                                   np.empty((0, 1), np.int64))
    if not info.is_main:
        return None
    reps_np, members_np = reps.cpu().numpy(), members.cpu().numpy()
    sim, idx = res
    rep_index = np.empty(n, np.int64)
    similarity = np.ones(n, np.float32)
    rep_index[reps_np] = reps_np
    rep_index[members_np] = reps_np[idx[:, 0]]
    similarity[members_np] = sim[:, 0]
    return rep_index, similarity, reps_np


def write_tsv(path, names, rep_index, similarity) -> None:
    with open(path, "w") as fout:
        fout.write(_HEADER)
        for name, r, s in zip(names, rep_index, similarity):
            fout.write(f"{name}\t{names[r]}\t{float(s):.6f}\n")


def main(input_npz, output_dir, min_similarity: float, verbose: bool = True, *, block: int = engine.CLUSTER_MAX_BLOCK,
         rep_chunk: int = engine.NEIGHBOURS_CHUNK, both_strands: bool = False):
    """both_strands: cluster the strand-averaged embeddings (EN.BOTH_STRANDS_KEY), so that a sequence and its reverse
    complement have bitwise the same row."""
    console = utils.HybridConsole(None, verbose)
    thr = engine.cluster_threshold(min_similarity)
    names, emb = EN.read_embeddings(input_npz, EN.BOTH_STRANDS_KEY if both_strands else "embeddings")
    info = dist.init_process_group_if_needed()
    tsv_path, npz_path = output_paths(input_npz, output_dir)
    console.log(f"Clustering {len(names):,} sequences at cosine similarity >= {thr:.6g}.")
    res = cluster(emb, thr, info, block, rep_chunk)
    if info.is_main:
        rep_index, similarity, reps = res
        sizes = np.bincount(np.searchsorted(reps, rep_index), minlength=len(reps)).astype(np.int64)
        Path(output_dir).mkdir(parents=True, exist_ok=True)
        write_tsv(tsv_path, names, rep_index, similarity)
        np.savez(npz_path, seq_names=names, representative_index=rep_index, similarity=similarity,
                 representatives=reps.astype(np.int64), cluster_size=sizes, min_similarity=np.float64(thr))
        console.log(f"{len(reps):,} clusters written to {tsv_path.name} and {npz_path.name}.")
    dist.barrier(info)
