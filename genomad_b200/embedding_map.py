"""
``embedding-map`` module: a two-dimensional map of the sequences of an embeddings file written by ``nn-classification
--write-embeddings``, so that one can look at the encoder's embedding space: whether chromosomes, plasmids and viruses form
separate groups, and where a head's classes, the novel sequences or the clusters of ``embedding-clusters`` sit.  Sequences of
the same class have more similar representations (reference docs/_source/nn_classification.md), and the map keeps each
sequence near its nearest neighbours.

The map is UMAP (McInnes, Healy & Melville 2018) as umap-learn computes it at n_neighbors = k + 1, min_dist = 0.1 and spread = 1,
with a PCA initialisation, exactly five negatives per sample and synchronous, gather-only epochs (DESIGN.md, "Embedding map"):
  * the all-vs-all k-nearest-neighbour lists: embedding_neighbours.search, sharded under torchrun like embedding-neighbours;
    with --index, the lists of an embedding-index search instead (EN.search through engine.ivf_search);
  * on rank 0, the memberships, the graph, the initialisation and the layout epochs: engine.map_layout.
The map depends only on the rows, their order, k, the epoch count and the seed: not on the GPU count.

Outputs in OUTPUT, <prefix> = the input file's stem without ``_nn_classification_embeddings``:
    <prefix>_embedding_map.tsv   seq_name, x, y (6 decimals), one line per sequence in input order
    <prefix>_embedding_map.npz   seq_names, coordinates float32 [n, 2], k, epochs, seed, both_strands
"""
from __future__ import annotations

from pathlib import Path
from typing import Optional, Tuple

import numpy as np

from . import dist, engine, utils
from . import embedding_neighbours as EN

_HEADER = "seq_name\tx\ty\n"


def output_paths(input_npz, output_dir) -> Tuple[Path, Path]:
    prefix = EN.output_prefix(input_npz)
    out = Path(output_dir)
    return out / f"{prefix}_embedding_map.tsv", out / f"{prefix}_embedding_map.npz"


def layout(emb: np.ndarray, k: int, epochs: int, seed: int, info, index=None, nprobe: Optional[int] = None) -> Optional[np.ndarray]:
    """The map of the rows of emb (float32 [n, 512]): float32 [n, 2] on rank 0, None on the other ranks.  index, nprobe: the
    neighbour lists come from the index search (EN.search)."""
    import torch
    res = EN.search(emb, None, k, info, index, nprobe)
    if not info.is_main:
        return None
    if index is not None and (res[1] < 0).any():
        # a row whose probed lists hold k or fewer other rows: the memberships need k real neighbours per row
        bad = int(np.flatnonzero((res[1] < 0).any(axis=1))[0])
        raise ValueError(f"sequence {bad} has fewer than {k} neighbours in its {nprobe} probed lists: raise --nprobe (or lower "
                         f"-k) so every sequence's lists hold more than k sequences")
    dev = EN._device(info)
    sim, idx = (torch.from_numpy(a).to(dev) for a in res)
    return engine.map_layout(torch.from_numpy(emb).to(dev), sim, idx, epochs, seed).cpu().numpy()


def write_tsv(path, names, coords) -> None:
    with open(path, "w") as fout:
        fout.write(_HEADER)
        for name, (x, y) in zip(names, coords):
            fout.write(f"{name}\t{float(x):.6f}\t{float(y):.6f}\n")


def main(input_npz, output_dir, k: int = 15, epochs: Optional[int] = None, seed: int = 0, verbose: bool = True, *,
         both_strands: bool = False, index=None, nprobe: Optional[int] = None):
    """k: neighbours per sequence, other sequences only (umap-learn's n_neighbors = k + 1); epochs: None for umap-learn's
    default (engine.map_default_epochs); both_strands: map the strand-averaged embeddings (EN.BOTH_STRANDS_KEY); index, nprobe:
    find the neighbours through an embedding-index file built on the input (nprobe required with it)."""
    console = utils.HybridConsole(None, verbose)
    key = EN.BOTH_STRANDS_KEY if both_strands else "embeddings"
    names, emb = EN.read_embeddings(input_npz, key)
    k, epochs, seed = engine.map_check(len(names), k, epochs, seed)
    ix = None
    if index is not None:
        from . import embedding_index as EI
        ix = EI.read_index(index, names, emb, key)
        nprobe = EI.check_nprobe(nprobe, ix)
    elif nprobe is not None:
        raise ValueError("--nprobe applies only with --index")
    info = dist.init_process_group_if_needed()
    tsv_path, npz_path = output_paths(input_npz, output_dir)
    console.log(f"Mapping {len(names):,} sequences with {k} neighbours each and {epochs} epochs (seed {seed}).")
    coords = layout(emb, k, epochs, seed, info, ix, nprobe)
    if info.is_main:
        Path(output_dir).mkdir(parents=True, exist_ok=True)
        write_tsv(tsv_path, names, coords)
        np.savez(npz_path, seq_names=names, coordinates=coords.astype(np.float32), k=np.int64(k), epochs=np.int64(epochs),
                 seed=np.uint64(seed), both_strands=np.bool_(both_strands))
        console.log(f"Map written to {tsv_path.name} and {npz_path.name}.")
    dist.barrier(info)
