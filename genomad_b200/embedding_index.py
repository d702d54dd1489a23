"""
``embedding-index`` module: an inverted-file (IVF) index of the sequences of an embeddings file written by ``nn-classification
--write-embeddings``, so that ``embedding-neighbours --index`` and ``embedding-map --index`` search millions of sequences
without comparing every pair.  Spherical k-means (Dhillon & Modha 2001) splits the rows into L lists; a query then scans only
the rows of its nprobe nearest lists (Jegou, Douze & Schmid 2011).  Every similarity the index returns is bitwise the one the
exact search computes for that pair: the index only chooses which pairs to compute.  At nprobe = L the result is the exact
search.  DESIGN.md, "Embedding index".

The build runs in one process on one GPU (engine.ivf_build); under torchrun with more than one process it is refused before any
work.

Output in OUTPUT, <prefix> = the input file's stem without ``_nn_classification_embeddings``:
    <prefix>_embedding_index.npz   centroids float32 [L, 512], rows int64 [n] (the rows in list order), offsets int64 [L + 1],
                                   lists, iterations, seed, training_rows, embeddings_key ("embeddings" or
                                   "embeddings_both_strands") and embeddings_sha256 (of the embedding array's bytes and the
                                   names).  It holds no embedding rows.
"""
from __future__ import annotations

import hashlib
import os
from pathlib import Path
from typing import Dict

import numpy as np

from . import engine, utils
from . import embedding_neighbours as EN

_KEYS = ("centroids", "rows", "offsets", "lists", "iterations", "seed", "training_rows", "embeddings_key", "embeddings_sha256")


class IndexFileError(ValueError):
    pass


def output_path(input_npz, output_dir) -> Path:
    return Path(output_dir) / f"{EN.output_prefix(input_npz)}_embedding_index.npz"


def embeddings_sha256(names, emb) -> str:
    """sha256 of the float32 embedding array's bytes, then the names (UTF-8, each followed by a newline)."""
    h = hashlib.sha256(np.ascontiguousarray(emb, dtype=np.float32).tobytes())
    for nm in names:
        h.update(str(nm).encode() + b"\n")
    return h.hexdigest()


def file_sha256(path) -> str:
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for block in iter(lambda: f.read(1 << 20), b""):
            h.update(block)
    return h.hexdigest()


def _world_size() -> int:
    return int(os.environ.get("WORLD_SIZE", "1") or 1)


def read_index(path, names, emb, key: str) -> Dict[str, object]:
    """An index NPZ checked against the embeddings it must have been built on (names, emb of the file under `key`): the key,
    the row count and the hash, and the layout's shape.  Returns dict(centroids, rows, offsets, lists, sha256).  Every check
    runs here, before any GPU work."""
    path = Path(path)
    try:
        z = np.load(path, allow_pickle=False)
        files = set(z.files)
        missing = [k for k in _KEYS if k not in files]
        if missing:
            raise IndexFileError(f"{path}: not an embedding-index file: missing {missing}")
        a = {k: z[k] for k in _KEYS}
    except IndexFileError:
        raise
    except Exception as e:
        raise IndexFileError(f"{path}: not a readable NPZ file ({e})") from None
    n = emb.shape[0]
    if str(a["embeddings_key"]) != key:
        raise IndexFileError(f"{path}: built on '{a['embeddings_key']}', but this search reads '{key}' (--both-strands must "
                             f"match)")
    rows, off, cent = a["rows"], a["offsets"], a["centroids"]
    if rows.ndim != 1 or rows.shape[0] != n:
        raise IndexFileError(f"{path}: indexes {rows.shape[0] if rows.ndim == 1 else list(rows.shape)} rows, the embeddings "
                             f"file has {n:,}")
    if str(a["embeddings_sha256"]) != embeddings_sha256(names, emb):
        raise IndexFileError(f"{path}: built on other embeddings (embeddings_sha256 differs)")
    L = int(a["lists"])
    if cent.ndim != 2 or cent.shape != (L, engine.EMBED) or not np.issubdtype(cent.dtype, np.floating) \
            or not np.isfinite(cent).all():
        raise IndexFileError(f"{path}: 'centroids' must be finite [{L}, {engine.EMBED}], not {cent.dtype} {list(cent.shape)}")
    if not 1 <= L <= n:
        raise IndexFileError(f"{path}: {L} lists for {n:,} rows")
    if off.shape != (L + 1,) or not np.issubdtype(off.dtype, np.integer) or off[0] != 0 or off[-1] != n \
            or (np.diff(off) < 0).any():
        raise IndexFileError(f"{path}: 'offsets' must be non-decreasing integers [{L + 1}] from 0 to {n:,}")
    if not np.issubdtype(rows.dtype, np.integer) or not np.array_equal(np.sort(rows), np.arange(n)):
        raise IndexFileError(f"{path}: 'rows' must be a permutation of the {n:,} rows")
    down = np.diff(rows) <= 0
    inner = off[1:-1][(off[1:-1] > 0) & (off[1:-1] < n)]
    down[inner - 1] = False                                  # a new list may start lower
    if down.any():
        raise IndexFileError(f"{path}: the rows of each list must ascend (row position {int(np.flatnonzero(down)[0]) + 1})")
    return {"centroids": np.ascontiguousarray(cent, np.float32), "rows": rows.astype(np.int64), "offsets": off.astype(np.int64),
            "lists": L, "sha256": file_sha256(path)}


def to_device(idx: Dict[str, object], device) -> "engine.IvfIndex":
    import torch
    return engine.IvfIndex(torch.from_numpy(idx["centroids"]).to(device), torch.from_numpy(idx["rows"]).to(device),
                           torch.from_numpy(idx["offsets"]).to(device))


def check_nprobe(nprobe, idx) -> int:
    if nprobe is None:
        raise ValueError("--nprobe is required with --index: how many lists a query scans (1 to min(64, lists)); recall "
                         "against the exact search depends on it")
    return engine.ivf_nprobe(nprobe, idx["lists"])


def build(emb: np.ndarray, lists: int, iterations: int, seed: int) -> Dict[str, np.ndarray]:
    import torch
    dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
    ix = engine.ivf_build(torch.from_numpy(emb).to(dev), lists, iterations, seed)
    return {"centroids": ix.centroids.cpu().numpy(), "rows": ix.rows.cpu().numpy(), "offsets": ix.offsets.cpu().numpy()}


def main(input_npz, output_dir, lists=None, iterations: int = 20, seed: int = 0, verbose: bool = True, *,
         both_strands: bool = False):
    """lists: None for ceil(4 sqrt(n)) (engine.ivf_default_lists)."""
    console = utils.HybridConsole(None, verbose)
    if _world_size() > 1:
        raise RuntimeError("embedding-index builds on one GPU in one process: run it without torchrun (or with one process)")
    key = EN.BOTH_STRANDS_KEY if both_strands else "embeddings"
    names, emb = EN.read_embeddings(input_npz, key)
    n = len(names)
    L, iterations, seed = engine.ivf_check(n, engine.ivf_default_lists(n) if lists is None else lists, iterations, seed)
    path = output_path(input_npz, output_dir)
    console.log(f"Building an index of {n:,} sequences: {L:,} lists, {iterations} k-means iterations (seed {seed}).")
    ix = build(emb, L, iterations, seed)
    Path(output_dir).mkdir(parents=True, exist_ok=True)
    np.savez(path, centroids=ix["centroids"].astype(np.float32), rows=ix["rows"].astype(np.int64),
             offsets=ix["offsets"].astype(np.int64), lists=np.int64(L), iterations=np.int64(iterations), seed=np.uint64(seed),
             training_rows=np.int64(min(n, engine.IVF_TRAIN_PER_LIST * L)), embeddings_key=np.str_(key),
             embeddings_sha256=np.str_(embeddings_sha256(names, emb)))
    console.log(f"Index written to {path.name}.")
