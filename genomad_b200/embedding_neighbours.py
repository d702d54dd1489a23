"""
``embedding-neighbours`` module: for every sequence of an embeddings file written by ``nn-classification
--write-embeddings``, its k nearest sequences in the encoder's embedding space (cosine similarity), either among the
sequences of a reference embeddings file or, without one, among the query sequences themselves (all-vs-all, a sequence
never being its own neighbour).  Sequences of the same class have more similar representations than sequences of
different classes (reference docs/_source/nn_classification.md), so the neighbours answer "which known plasmids or viruses
does this contig resemble" or "which contigs of this assembly are near-duplicates".

The search is gnm_embedding_neighbours (include/gnm.h) through ``engine.embedding_neighbours``.  Under torchrun every rank
searches a contiguous shard of the reference rows (``dist.shard_bounds``) for all queries and sends its [n, k] lists to rank 0
point to point; rank 0 merges them in rank order (gnm_neighbours_merge) and writes the files.  The lists do not depend on how
the reference is split, so the files are bitwise those of one process.

Outputs in OUTPUT, <prefix> = the query file's stem without ``_nn_classification_embeddings``:
    <prefix>_embedding_neighbours.tsv   seq_name, rank (1-based), neighbour_name, cosine_similarity (6 decimals); padded
                                        entries (fewer than k references) are left out
    <prefix>_embedding_neighbours.npz   query_names, reference_names, neighbour_index int64 [n, k] (-1 = none),
                                        similarity float32 [n, k] (-inf = none), k; with --index also nprobe and
                                        index_sha256 (of the index file)

With --index (an embedding-index file) each query scans only the rows of its nprobe nearest lists (engine.ivf_search); under
torchrun each rank then takes a contiguous range of the lists, balanced by rows, and rank 0 merges in rank order as above.
"""
from __future__ import annotations

from pathlib import Path
from typing import Optional, Tuple

import numpy as np

from . import dist, engine, utils

_HEADER = "seq_name\trank\tneighbour_name\tcosine_similarity\n"
NAME_KEYS = ("contig_names", "provirus_names")
_SUFFIX = "_nn_classification_embeddings"


class EmbeddingsFileError(ValueError):
    pass


def output_prefix(query_npz) -> str:
    stem = Path(query_npz).name
    if stem.endswith(".npz"):
        stem = stem[:-4]
    return stem[: -len(_SUFFIX)] if stem.endswith(_SUFFIX) and len(stem) > len(_SUFFIX) else stem


def output_paths(query_npz, output_dir) -> Tuple[Path, Path]:
    prefix = output_prefix(query_npz)
    out = Path(output_dir)
    return out / f"{prefix}_embedding_neighbours.tsv", out / f"{prefix}_embedding_neighbours.npz"


BOTH_STRANDS_KEY = "embeddings_both_strands"


def read_embeddings(path, key: str = "embeddings") -> Tuple[np.ndarray, np.ndarray]:
    """An embeddings NPZ of nn-classification -> (names [n] str, embeddings float32 [n, 512]); every check before any GPU work.
    key: the array to read, "embeddings" (the forward strand) or BOTH_STRANDS_KEY (the mean of both strands' embeddings,
    which nn-classification --write-embeddings --both-strands adds)."""
    path = Path(path)
    try:
        z = np.load(path, allow_pickle=False)
        files = set(z.files)
    except Exception as e:
        raise EmbeddingsFileError(f"{path}: not a readable NPZ file ({e})") from None
    keys = [k for k in NAME_KEYS if k in files]
    if key != "embeddings" and key not in files and len(keys) == 1 and "embeddings" in files:
        raise EmbeddingsFileError(f"{path}: no '{key}' array: nn-classification writes it with --write-embeddings "
                                  f"--both-strands")
    if len(keys) != 1 or key not in files:
        raise EmbeddingsFileError(f"{path}: expected 'embeddings' and one of {NAME_KEYS} (nn-classification "
                                  f"--write-embeddings output), found {sorted(files)}")
    try:
        names, emb = z[keys[0]], z[key]
    except Exception as e:
        raise EmbeddingsFileError(f"{path}: cannot read its arrays ({e})") from None
    if emb.ndim != 2 or emb.shape[1] != engine.EMBED:
        raise EmbeddingsFileError(f"{path}: '{key}' must be [n, {engine.EMBED}], not {list(emb.shape)}")
    if not np.issubdtype(emb.dtype, np.floating):
        raise EmbeddingsFileError(f"{path}: '{key}' must be floating point, not {emb.dtype}")
    emb = np.ascontiguousarray(emb, dtype=np.float32)
    if not np.isfinite(emb).all():
        bad = int(np.flatnonzero(~np.isfinite(emb).all(axis=1))[0])
        raise EmbeddingsFileError(f"{path}: '{key}' has non-finite values (first in row {bad})")
    if names.ndim != 1 or names.shape[0] != emb.shape[0]:
        raise EmbeddingsFileError(f"{path}: {names.shape[0] if names.ndim == 1 else list(names.shape)} names in "
                                  f"'{keys[0]}' for {emb.shape[0]} embedding rows")
    return names.astype(str), emb


def _device(info):
    import torch
    return torch.device("cuda", info.local_rank) if torch.cuda.is_available() else torch.device("cpu")


def list_shard(offsets, world_size: int, rank: int) -> Tuple[int, int]:
    """The contiguous range of an index's lists rank `rank` searches: the lists are split where the rows are, so every rank
    gets about n / world_size rows."""
    off = np.asarray(offsets, np.int64)
    n, L = int(off[-1]), len(off) - 1
    cut = lambda r: 0 if r == 0 else L if r == world_size else int(np.searchsorted(off, r * n // world_size, side="left"))
    return cut(rank), max(cut(rank), cut(rank + 1))


def search(query, reference, k: int, info, index=None, nprobe: Optional[int] = None) -> Optional[Tuple[np.ndarray, np.ndarray]]:
    """This rank's reference shard searched on the device, the lists gathered on rank 0 and merged there in rank order.
    Returns (sim float32 [n, k], idx int64 [n, k]) on rank 0, None on the others.  reference None: all-vs-all.  query and
    reference are NumPy arrays, or tensors already on this rank's device (embedding_clusters keeps its rows there).
    index (embedding_index.read_index of the reference) and nprobe: search through the index instead; a rank's shard is then a
    contiguous range of its lists (list_shard)."""
    import torch
    dev = _device(info)
    ref = query if reference is None else reference
    q = torch.as_tensor(query).to(dev)
    if index is None:
        s, e = dist.shard_bounds(ref.shape[0], info.world_size, info.rank)
        r = torch.as_tensor(ref[s:e]).to(dev)
        sim, idx = engine.embedding_neighbours(q, r, k, ref_index0=s, self_index0=0 if reference is None else -1)
    else:
        from . import embedding_index as EI
        l0, l1 = list_shard(index["offsets"], info.world_size, info.rank)
        if reference is None:                                  # the queries are the reference, already on the device
            sim, idx = engine.ivf_search(q, None, EI.to_device(index, dev), k, nprobe, lists=(l0, l1))
        else:                                                  # only the rows of this rank's lists, in list order
            own = index["rows"][index["offsets"][l0]:index["offsets"][l1]]
            r = torch.as_tensor(ref[torch.as_tensor(own)] if torch.is_tensor(ref) else ref[own]).to(dev)
            sim, idx = engine.ivf_search(q, r, EI.to_device(index, dev), k, nprobe, self_index0=-1, lists=(l0, l1),
                                         reference_shard=True)
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


def write_tsv(path, query_names, reference_names, sim, idx) -> None:
    with open(path, "w") as fout:
        fout.write(_HEADER)
        for qn, srow, irow in zip(query_names, sim, idx):
            for rank, (s, i) in enumerate(zip(srow, irow), 1):
                if i >= 0:
                    fout.write(f"{qn}\t{rank}\t{reference_names[i]}\t{float(s):.6f}\n")


def main(query_npz, reference_npz, output_dir, k: int = 10, verbose: bool = True, *, both_strands: bool = False,
         index=None, nprobe: Optional[int] = None):
    """both_strands: search the strand-averaged embeddings (BOTH_STRANDS_KEY) of every input file, so that a sequence and its
    reverse complement have bitwise the same row.  index: an embedding-index file built on the reference file (the query file
    for all-vs-all) with the same strand key, searched at nprobe lists per query (required with it)."""
    console = utils.HybridConsole(None, verbose)
    k = int(k)
    if not 1 <= k <= engine.NEIGHBOURS_MAX_K:
        raise ValueError(f"k must be in [1, {engine.NEIGHBOURS_MAX_K}], not {k}")
    key = BOTH_STRANDS_KEY if both_strands else "embeddings"
    qnames, qemb = read_embeddings(query_npz, key)
    if reference_npz is not None:
        rnames, remb = read_embeddings(reference_npz, key)
    else:
        rnames, remb = qnames, None
    ix = None
    if index is not None:
        from . import embedding_index as EI
        ix = EI.read_index(index, rnames, qemb if remb is None else remb, key)
        nprobe = EI.check_nprobe(nprobe, ix)
    elif nprobe is not None:
        raise ValueError("--nprobe applies only with --index")
    info = dist.init_process_group_if_needed()
    tsv_path, npz_path = output_paths(query_npz, output_dir)
    mode = f"against {len(rnames):,} reference sequences" if remb is not None else "all-vs-all"
    via = "" if ix is None else f" through an index of {ix['lists']:,} lists ({nprobe} probed per query)"
    console.log(f"Searching the {k} nearest neighbours of {len(qnames):,} sequences {mode}{via}.")
    res = search(qemb, remb, k, info, ix, nprobe)
    if info.is_main:
        sim, idx = res
        Path(output_dir).mkdir(parents=True, exist_ok=True)
        write_tsv(tsv_path, qnames, rnames, sim, idx)
        extra = {} if ix is None else {"nprobe": np.int64(nprobe), "index_sha256": np.str_(ix["sha256"])}
        np.savez(npz_path, query_names=qnames, reference_names=rnames, neighbour_index=idx.astype(np.int64),
                 similarity=sim.astype(np.float32), k=np.int64(k), **extra)
        console.log(f"Neighbours written to {tsv_path.name} and {npz_path.name}.")
    dist.barrier(info)
