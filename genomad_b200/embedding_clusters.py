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

With --index (an embedding-index file built on the input with the same strand key) and --nprobe, a row is compared only with the
representatives whose home list (the list the index places them in) is one of its nprobe probed lists: row j is a representative
iff s(j, i) < t for every representative i < j with home(i) in P(j), and every other row joins its first representative under
(s descending, index ascending) among those.  At nprobe = L this is the exact clustering, bitwise.  The representatives live in
slots laid out like the index (engine.ClusterSlots): covering and the final assignment are engine.cluster_slots_search at k = 1
over the row's probed lists, the block step engine.cluster_block_probed.  Under torchrun each rank holds the slots of its
contiguous range of lists (EN.list_shard), rank 0 ORs the covering flags and decides the block as above, every rank appends
the new representatives of its lists, and rank 0 merges the final lists in rank order.  DESIGN.md, "Embedding clusters through
the index".

Outputs in OUTPUT, <prefix> = the input file's stem without ``_nn_classification_embeddings``:
    <prefix>_embedding_clusters.tsv   seq_name, representative, cosine_similarity (6 decimals), one line per sequence in input
                                      order; a representative names itself with 1.000000
    <prefix>_embedding_clusters.npz   seq_names, representative_index int64 [n], similarity float32 [n] (1 for a
                                      representative), representatives int64 [R] ascending, cluster_size int64 [R],
                                      min_similarity float64 (the fp32 threshold applied); with --index also nprobe
                                      and index_sha256 (of the index file)
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
    s, e = dist.shard_bounds(rep_rows.shape[0], info.world_size, info.rank)
    return _decide(_covered(blk, rep_rows[s:e], thr, rep_chunk), lambda cov: engine.cluster_block(blk, cov, thr), info)


def _decide(cov, decide, info):
    """Rank 0 ORs every rank's covering flags and runs decide(cov), the block step; its new representatives are returned on every
    rank."""
    import torch
    if info.world_size == 1:
        return decide(cov)
    count = torch.zeros(1, dtype=torch.int64, device=cov.device)
    if not info.is_main:
        dist._p2p_send(cov, 0)
        dist._p2p_recv(count, 0)
        new = torch.empty(int(count.item()), dtype=torch.int64, device=cov.device)
        if new.numel():
            dist._p2p_recv(new, 0)
        return new
    part = torch.empty_like(cov)
    for src in range(1, info.world_size):
        dist._p2p_recv(part, src)
        cov |= part
    new = decide(cov)
    count[0] = new.numel()
    for dst in range(1, info.world_size):
        dist._p2p_send(count, dst)
        if new.numel():
            dist._p2p_send(new.contiguous(), dst)
    return new


def _gather_merged(sim, idx, info):
    """Rank 0: every rank's k = 1 lists merged in rank order (numpy); None on the other ranks."""
    import torch
    if info.world_size > 1:
        if not info.is_main:
            dist._p2p_send(sim.contiguous(), 0)
            dist._p2p_send(idx.contiguous(), 0)
            return None
        for src in range(1, info.world_size):
            sb, ib = torch.empty_like(sim), torch.empty_like(idx)
            dist._p2p_recv(sb, src)
            dist._p2p_recv(ib, src)
            engine.neighbours_merge(sim, idx, sb, ib)
    return sim.cpu().numpy(), idx.cpu().numpy()


def index_bytes_per_row(nprobe: int) -> int:
    """Device bytes per row of a clustering through the index on one GPU: the row, its probes and home list, and its slot
    (every row has one: the capacities are the index's list sizes)."""
    return engine.EMBED * 4 + 4 * nprobe + 4 + 8 + engine.CLUSTER_SLOT_BYTES


def _free_bytes(dev) -> float:
    """The device's free memory plus what PyTorch's allocator holds unused."""
    import torch
    if dev.type != "cuda":
        return float("inf")
    return float(torch.cuda.mem_get_info(dev)[0] + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev))


def home_lists(index) -> np.ndarray:
    """int32 [n]: the list the index places each row in."""
    home = np.empty(len(index["rows"]), np.int32)
    home[index["rows"]] = np.repeat(np.arange(index["lists"], dtype=np.int32), np.diff(index["offsets"]))
    return home


def _check_memory(n: int, index, nprobe: int, info, dev) -> None:
    """MemoryError unless this rank's share of a clustering through the index fits in 90 % of the device's free memory."""
    off = index["offsets"]
    l0, l1 = EN.list_shard(off, info.world_size, info.rank)
    need = n * index_bytes_per_row(nprobe) - (n - int(off[l1] - off[l0])) * engine.CLUSTER_SLOT_BYTES + engine.IVF_QUERY_BYTES
    free = _free_bytes(dev)
    if need > 0.9 * free:
        raise MemoryError(f"clustering {n:,} rows through the index needs about {need / 2**30:.1f} GiB of GPU memory "
                          f"({index_bytes_per_row(nprobe):,} bytes per row and a {engine.IVF_QUERY_BYTES / 2**30:.0f} GiB search "
                          f"workspace); {free / 2**30:.1f} GiB are free")


def _cluster_index(x, thr: float, info, block: int, index, nprobe: int):
    """The block loop through the index: (representatives int64 [R] ascending, members int64, sim, idx) on rank 0."""
    import torch
    from . import embedding_index as EI
    dev, n = x.device, x.shape[0]
    off = index["offsets"]
    l0, l1 = EN.list_shard(off, info.world_size, info.rank)
    home = torch.from_numpy(home_lists(index)).to(dev)
    probes = engine.ivf_probes(x, torch.from_numpy(index["centroids"]).to(dev), nprobe)
    bad = torch.nonzero(probes[:, 0] != home).flatten()
    if bad.numel():
        raise EI.IndexFileError(f"row {int(bad[0])}: the index places it in list {int(home[bad[0]])}, but its nearest centroid is "
                                f"list {int(probes[bad[0], 0])}: the index's centroids and lists disagree")
    slots = engine.cluster_slots(off, l0, l1, dev)
    reps = torch.empty(n, dtype=torch.int64, device=dev)
    n_rep = 0
    for a in range(0, n, block):
        b = min(n, a + block)
        blk, pr, hm = x[a:b], probes[a:b], home[a:b]
        sim, _ = engine.cluster_slots_search(slots, blk, pr)
        cov = (sim[:, 0] >= thr).to(torch.uint8)
        new = _decide(cov, lambda c: engine.cluster_block_probed(blk, c, thr, pr, hm), info)
        engine.cluster_slots_append(slots, blk[new], new + a, hm[new])
        reps[n_rep: n_rep + new.numel()] = new + a
        n_rep += new.numel()
    reps = reps[:n_rep]
    is_rep = torch.zeros(n, dtype=torch.bool, device=dev)
    is_rep[reps] = True
    members = torch.nonzero(~is_rep).flatten()
    parts = [engine.cluster_slots_search(slots, x[mc], probes[mc]) for mc in members.split(engine.NEIGHBOURS_CHUNK)]
    sim = torch.cat([p[0] for p in parts]) if parts else torch.empty((0, 1), dtype=torch.float32, device=dev)
    idx = torch.cat([p[1] for p in parts]) if parts else torch.empty((0, 1), dtype=torch.int64, device=dev)
    res = _gather_merged(sim, idx, info)
    if res is None:
        return None
    return reps.cpu().numpy(), members.cpu().numpy(), res[0][:, 0], res[1][:, 0]


def cluster(emb: np.ndarray, min_similarity: float, info, block: int = engine.CLUSTER_MAX_BLOCK,
            rep_chunk: int = engine.NEIGHBOURS_CHUNK, index=None,
            nprobe: Optional[int] = None) -> Optional[Tuple[np.ndarray, np.ndarray, np.ndarray]]:
    """Greedy clustering of the rows of emb (float32 [n, 512]) at min_similarity.  Returns, on rank 0, (representative_index
    int64 [n], similarity float32 [n], representatives int64 [R]); None on the other ranks.  index (embedding_index.read_index
    of emb) and nprobe: cluster through the index (rep_chunk then does not apply); at nprobe = lists the result is bitwise the
    exact one."""
    import torch
    thr = engine.cluster_threshold(min_similarity)
    if not 1 <= block <= engine.CLUSTER_MAX_BLOCK:
        raise ValueError(f"block must be in [1, {engine.CLUSTER_MAX_BLOCK}], not {block}")
    if rep_chunk < 1:
        raise ValueError(f"rep_chunk must be >= 1, not {rep_chunk}")
    if index is not None:
        nprobe = engine.ivf_nprobe(nprobe, index["lists"])
        if len(index["rows"]) != emb.shape[0]:
            raise ValueError(f"the index holds {len(index['rows']):,} rows, emb {emb.shape[0]:,}")
    dev = EN._device(info)
    n = emb.shape[0]
    if index is not None:
        _check_memory(n, index, nprobe, info, dev)
    x = torch.from_numpy(emb).to(dev)
    if index is not None:
        res = _cluster_index(x, thr, info, block, index, nprobe)
        return None if res is None else _assemble(n, *res)
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
    return _assemble(n, reps_np, members_np, sim[:, 0], reps_np[idx[:, 0]])


def _assemble(n: int, reps, members, sim, rep_of):
    """(representative_index int64 [n], similarity float32 [n], representatives) from the members' representatives and
    similarities."""
    rep_index = np.empty(n, np.int64)
    similarity = np.ones(n, np.float32)
    rep_index[reps] = reps
    rep_index[members] = rep_of
    similarity[members] = sim
    return rep_index, similarity, reps


def write_tsv(path, names, rep_index, similarity) -> None:
    with open(path, "w") as fout:
        fout.write(_HEADER)
        for name, r, s in zip(names, rep_index, similarity):
            fout.write(f"{name}\t{names[r]}\t{float(s):.6f}\n")


def main(input_npz, output_dir, min_similarity: float, verbose: bool = True, *, block: int = engine.CLUSTER_MAX_BLOCK,
         rep_chunk: int = engine.NEIGHBOURS_CHUNK, both_strands: bool = False, index=None, nprobe: Optional[int] = None):
    """both_strands: cluster the strand-averaged embeddings (EN.BOTH_STRANDS_KEY), so that a sequence and its reverse
    complement have bitwise the same row.  index: an embedding-index file built on the input file with the same strand key,
    probed at nprobe lists per sequence (required with it)."""
    console = utils.HybridConsole(None, verbose)
    thr = engine.cluster_threshold(min_similarity)
    key = EN.BOTH_STRANDS_KEY if both_strands else "embeddings"
    names, emb = EN.read_embeddings(input_npz, key)
    ix = None
    if index is not None:
        from . import embedding_index as EI
        ix = EI.read_index(index, names, emb, key)
        nprobe = EI.check_nprobe(nprobe, ix)
    elif nprobe is not None:
        raise ValueError("--nprobe applies only with --index")
    info = dist.init_process_group_if_needed()
    tsv_path, npz_path = output_paths(input_npz, output_dir)
    via = "" if ix is None else f" through an index of {ix['lists']:,} lists ({nprobe} probed per sequence)"
    console.log(f"Clustering {len(names):,} sequences at cosine similarity >= {thr:.6g}{via}.")
    res = cluster(emb, thr, info, block, rep_chunk, ix, nprobe)
    if info.is_main:
        rep_index, similarity, reps = res
        sizes = np.bincount(np.searchsorted(reps, rep_index), minlength=len(reps)).astype(np.int64)
        Path(output_dir).mkdir(parents=True, exist_ok=True)
        write_tsv(tsv_path, names, rep_index, similarity)
        np.savez(npz_path, seq_names=names, representative_index=rep_index, similarity=similarity,
                 representatives=reps.astype(np.int64), cluster_size=sizes, min_similarity=np.float64(thr),
                 **({} if ix is None else {"nprobe": np.int64(nprobe), "index_sha256": np.str_(ix["sha256"])}))
        console.log(f"{len(reps):,} clusters written to {tsv_path.name} and {npz_path.name}.")
    dist.barrier(info)
