"""
``window-regions`` module: class regions along each sequence of a window-score file written by ``nn-classification
--write-window-scores`` (the three shipped classes, ``<prefix>_nn_classification_windows.npz``) or, with ``--head``, by a head
(its C classes, ``<prefix>_nn_classification_head_windows.npz``), and the ``provirus_`` twins of both.  Where along a contig the
virus or plasmid signal lies, as coordinates with a confidence, instead of a per-window argmax that flickers on noisy windows.

Each sequence's windows are decoded by an HMM with one state per class (engine.window_regions, gnm_window_regions): the
Viterbi path gives the regions, the forward-backward posteriors their confidence.  The only parameter is the mean region
length L (bases, >= 12,000), which sets the switch rate per stride s / L; the emissions are the window scores tempered by
s / 6000 so that each base counts about once at any stride.  DESIGN.md, "Window regions", states the model.  The result of a
sequence depends only on its own windows.  One process on one GPU; not a torchrun job.

Outputs in OUTPUT, <stem> = the input file's stem with its trailing ``_windows`` replaced by ``_regions`` (otherwise
``<stem>_regions``), so the classifier's and a head's files never collide:
    <stem>.tsv   seq_name, start (1-based), end (inclusive), length, class, n_windows, posterior, then <class>_score per class
                 (4 decimals), one row per region in sequence and window order
    <stem>.npz   the input's names key (contig_names or provirus_names), region_contig int32 [R], region_start int64 [R]
                 (0-based), region_end int64 [R] (exclusive), region_class int32 [R], region_windows int32 [R],
                 region_posterior float32 [R], region_scores float32 [R, C], window_posteriors float32 [W, C], window_state
                 int32 [W], class_names, window_stride int32, mean_region_length float64, and head_sha256 if the input had one
"""
from __future__ import annotations

from pathlib import Path
from typing import Dict, Tuple

import numpy as np

from . import engine, utils

NAME_KEYS = ("contig_names", "provirus_names")
DEFAULT_CLASSES = ("chromosome", "plasmid", "virus")
_WINDOW_KEYS = ("predictions", "window_contig", "window_start", "window_length", "window_stride")


class WindowsFileError(ValueError):
    pass


def output_stem(input_npz) -> str:
    stem = Path(input_npz).name
    if stem.endswith(".npz"):
        stem = stem[:-4]
    return stem[: -len("_windows")] + "_regions" if stem.endswith("_windows") and len(stem) > len("_windows") else stem + "_regions"


def output_paths(input_npz, output_dir) -> Tuple[Path, Path]:
    stem = output_stem(input_npz)
    out = Path(output_dir)
    return out / f"{stem}.tsv", out / f"{stem}.npz"


def read_windows(path) -> Dict[str, object]:
    """A window-score NPZ of nn-classification -> dict(names_key, names [n] str, predictions float32 [W, C], window_contig int32,
    window_start int64, window_length int32, offsets int64 [n + 1], window_stride int, class_names [C] str, head_sha256 or
    None).  Every check runs here, before any GPU work."""
    path = Path(path)
    try:
        z = np.load(path, allow_pickle=False)
        files = set(z.files)
    except Exception as e:
        raise WindowsFileError(f"{path}: not a readable NPZ file ({e})") from None
    keys = [k for k in NAME_KEYS if k in files]
    missing = [k for k in _WINDOW_KEYS if k not in files]
    if len(keys) != 1 or missing:
        raise WindowsFileError(f"{path}: expected one of {NAME_KEYS} and {list(_WINDOW_KEYS)} (nn-classification "
                               f"--write-window-scores output), found {sorted(files)}")
    try:
        arr = {k: z[k] for k in (keys[0], *_WINDOW_KEYS)}
        class_names = z["class_names"] if "class_names" in files else np.array(DEFAULT_CLASSES)
        head_sha = str(z["head_sha256"]) if "head_sha256" in files else None
    except Exception as e:
        raise WindowsFileError(f"{path}: cannot read its arrays ({e})") from None
    names, pred = arr[keys[0]], arr["predictions"]
    if names.ndim != 1:
        raise WindowsFileError(f"{path}: '{keys[0]}' must be one-dimensional, not {list(names.shape)}")
    if pred.ndim != 2 or not 2 <= pred.shape[1] <= 32:
        raise WindowsFileError(f"{path}: 'predictions' must be [W, C] with 2 <= C <= 32, not {list(pred.shape)}")
    if not np.issubdtype(pred.dtype, np.floating):
        raise WindowsFileError(f"{path}: 'predictions' must be floating point, not {pred.dtype}")
    W, C = pred.shape
    if class_names.ndim != 1 or class_names.shape[0] != C:
        raise WindowsFileError(f"{path}: {class_names.size} class names for {C} score columns")
    for k in ("window_contig", "window_start", "window_length"):
        if arr[k].shape != (W,) or not np.issubdtype(arr[k].dtype, np.integer):
            raise WindowsFileError(f"{path}: '{k}' must be integers [{W}], not {arr[k].dtype} {list(arr[k].shape)}")
    st = arr["window_stride"]
    if st.shape != () or not np.issubdtype(st.dtype, np.integer) or not 1 <= int(st) <= engine.WINDOW:
        raise WindowsFileError(f"{path}: 'window_stride' must be an integer in [1, {engine.WINDOW}], not {st}")
    stride = int(st)
    pred = np.ascontiguousarray(pred, dtype=np.float32)
    if not np.isfinite(pred).all():
        bad = int(np.flatnonzero(~np.isfinite(pred).all(axis=1))[0])
        raise WindowsFileError(f"{path}: 'predictions' has non-finite values (first in window {bad})")
    contig = arr["window_contig"].astype(np.int64)
    start = arr["window_start"].astype(np.int64)
    length = arr["window_length"].astype(np.int64)
    n = names.shape[0]
    if W and (contig.min() < 0 or contig.max() >= n or (np.diff(contig) < 0).any()):
        raise WindowsFileError(f"{path}: 'window_contig' must be non-decreasing indices into the {n} names")
    if W and (start.min() < 0 or length.min() < 1 or length.max() > engine.WINDOW):
        raise WindowsFileError(f"{path}: window starts must be >= 0 and lengths in [1, {engine.WINDOW}]")
    same = contig[1:] == contig[:-1]
    d = start[1:] - start[:-1]
    bad = np.flatnonzero(same & ((d <= 0) | (d % stride != 0)))
    if bad.size:
        raise WindowsFileError(f"{path}: window {int(bad[0]) + 1} does not start a positive multiple of the stride {stride} "
                               f"after the window before it in its sequence")
    offsets = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(contig, minlength=n), out=offsets[1:])
    return {"names_key": keys[0], "names": names.astype(str), "predictions": pred, "window_contig": contig.astype(np.int32),
            "window_start": start, "window_length": length.astype(np.int32), "offsets": offsets, "window_stride": stride,
            "class_names": class_names.astype(str), "head_sha256": head_sha}


def _device():
    import torch
    return torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")


def decode(win: Dict[str, object], mean_region_length: float) -> Dict[str, np.ndarray]:
    """engine.window_regions on the windows of read_windows -> the WindowRegions fields as numpy arrays."""
    import torch
    dev = _device()
    ws = engine.WindowScores(*(torch.from_numpy(np.ascontiguousarray(win[k])).to(dev) for k in (
        "predictions", "window_contig", "window_start", "window_length")),
        torch.from_numpy(win["offsets"].astype(np.int32)).to(dev))
    res = engine.window_regions(ws, win["window_stride"], mean_region_length)
    return {k: v.cpu().numpy() for k, v in res._asdict().items()}


def write_tsv(path, names, class_names, reg) -> None:
    with open(path, "w") as fout:
        fout.write("seq_name\tstart\tend\tlength\tclass\tn_windows\tposterior\t"
                   + "\t".join(f"{c}_score" for c in class_names) + "\n")
        for r in range(len(reg["region_start"])):
            s, e = int(reg["region_start"][r]), int(reg["region_end"][r])
            scores = "\t".join(f"{float(x):.4f}" for x in reg["region_scores"][r])
            fout.write(f"{names[reg['region_contig'][r]]}\t{s + 1}\t{e}\t{e - s}\t{class_names[reg['region_class'][r]]}\t"
                       f"{int(reg['region_windows'][r])}\t{float(reg['region_posterior'][r]):.4f}\t{scores}\n")


def main(input_npz, output_dir, mean_region_length: float, verbose: bool = True):
    console = utils.HybridConsole(None, verbose)
    L = engine.regions_mean_length(mean_region_length)
    win = read_windows(input_npz)
    tsv_path, npz_path = output_paths(input_npz, output_dir)
    console.log(f"Decoding {len(win['predictions']):,} windows of {len(win['names']):,} sequences into "
                f"{', '.join(win['class_names'])} regions (stride {win['window_stride']}, mean region length {L:,.0f}).")
    reg = decode(win, L)
    Path(output_dir).mkdir(parents=True, exist_ok=True)
    write_tsv(tsv_path, win["names"], win["class_names"], reg)
    out = {win["names_key"]: win["names"], **{k: reg[k] for k in reg if k.startswith("region_")},
           "window_posteriors": reg["posterior"], "window_state": reg["state"], "class_names": win["class_names"],
           "window_stride": np.int32(win["window_stride"]), "mean_region_length": np.float64(L)}
    if win["head_sha256"] is not None:
        out["head_sha256"] = np.str_(win["head_sha256"])
    np.savez(npz_path, **out)
    console.log(f"{len(reg['region_start']):,} regions written to {tsv_path.name} and {npz_path.name}.")
