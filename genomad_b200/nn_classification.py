"""
``nn-classification`` module driver -- drop-in for ``genomad.nn_classification.main``
(reference genomad/modules/nn_classification.py:21-427): same signature, same files on disk
(<prefix>_nn_classification.{log,json,tsv,npz}, <prefix>_encoded_sequences/, the provirus twins), same
skip/restart/cleanup semantics, same error behaviour (message + sys.exit(1)).

What changed underneath: the FASTA is indexed once by the native reader (csrc/fasta.cpp: mmap, no copy); its 6 kb
windows are streamed through pinned chunks to the GPU (the host fills chunk i+1 while the GPU classifies chunk i),
tokenised and classified by libgnm.so (hand-written sm_90a kernels) and reduced per contig on the device.
``--batch-size`` keeps the reference's meaning -- an upper bound on the memory one prediction step may use -- but no
longer sets the device step: the library steps through >= 1024 windows at a time whatever the option says (the
reference's default of 128 would pay the fixed per-step cost 8x as often for no benefit on an 80 GB part).  TensorFlow, TFRecords and the per-batch ``predict`` call are gone; the
"encoded sequences" directory only records which window belongs to which sequence.  With torchrun (WORLD_SIZE > 1)
windows are sharded across GPUs and combined over NCCL (genomad_b200.dist); rank 0 writes the outputs.
"""
from __future__ import annotations

import os
import shutil
import sys
from pathlib import Path

import numpy as np

from . import __version__, dist as gdist, sequence, utils
from ._paths import NNOutputs

_HEADER = "seq_name\tchromosome_score\tplasmid_score\tvirus_score\n"

# wall-clock breakdown of the most recent main() call on this rank (seconds): read by bench.py's module_e2e report
last_timings: dict = {}


DEVICE_STEP_MIN, DEVICE_STEP_MAX = 1024, 4096
_WORKSPACE_BYTES_PER_WINDOW = 7.0e6          # libgnm workspace per window of max_batch (DESIGN.md section 4)


def device_step(batch_size: int, free_bytes: int) -> int:
    """Windows per internal GPU step.  `--batch-size` (reference cli.py:757-764: "smaller value to reduce memory") only
    bounds memory in the reference; here the step is max(batch_size, 1024) capped at 4096, and halved until its workspace fits
    in half of the free HBM."""
    step = min(DEVICE_STEP_MAX, max(DEVICE_STEP_MIN, int(batch_size)))
    while step > 64 and step * _WORKSPACE_BYTES_PER_WINDOW > 0.5 * free_bytes:
        step //= 2
    return step


_CLASSIFIERS: dict = {}          # (device, windows per step) -> engine.Classifier, kept for the life of the process


def release_classifiers() -> None:
    """Destroy the cached classifiers (frees ~7 GB of HBM per device; the next main() call rebuilds them)."""
    for c in list(_CLASSIFIERS.values()):
        c.close()
    _CLASSIFIERS.clear()


def _make_classifier(batch_size: int, device: int):
    """Factory (patched in CPU tests): the real one needs an H100 and libgnm.so -- no fallback.
    The classifier (weights re-packed on the device + workspace, ~0.3 s to build and ~0.4 s to free) stays resident between
    main() calls of one process -- `genomad end-to-end`, a service, the provirus twin -- unless GENOMAD_B200_KEEP_MODEL=0."""
    import torch
    from .engine import Classifier
    free, _total = torch.cuda.mem_get_info(device)
    keep = os.environ.get("GENOMAD_B200_KEEP_MODEL", "1") not in ("", "0")
    for (dev, step), c in _CLASSIFIERS.items():
        if dev == device and keep:
            return c                                          # its step already fitted this device
    clf = Classifier(None, device=device, max_batch=device_step(batch_size, free))
    if keep:
        _CLASSIFIERS[(device, clf.max_batch)] = clf
    return clf


def _pinned_chunk(n: int):
    """uint8 [n, 6000] in page-locked host memory (H2D copies then run at full PCIe speed and overlap compute)."""
    import torch
    t = torch.empty((n, sequence.WINDOW), dtype=torch.uint8).pin_memory()
    return t, t.numpy()


def _pinned_probs(n: int):
    """float32 [n, 3] in page-locked host memory: where gnm_classify_host writes a rank's per-window probabilities."""
    import torch
    return torch.empty((n, 3), dtype=torch.float32).pin_memory()


def _device(clf):
    import torch
    return torch.device("cuda", clf.device)


def _classify_parsed(clf, parsed, offsets, info: gdist.DistInfo, contig_reduce: str = "gather",
                     embeddings: bool = False, window_probs: bool = False, attributions: "dict | None" = None,
                     head: "dict | None" = None, window_embeddings=None):
    """
    Indexed FASTA -> float32 [n_contigs, 3] per-contig mean (identical on all ranks).

    `parsed` is the window source: a ParsedFasta (the reference's windows) or a sequence.WindowList (windows at another
    stride); all the loop needs is n_windows, export_windows and release_before.

    This rank's contiguous block of the global window list is streamed in chunks: the native reader fills one pinned
    chunk straight from the mmap'ed file (upper-case + pad, multi-threaded) while the GPU classifies the previous one
    (gnm_classify_host on a worker thread; the C call releases the GIL) into a pinned result buffer, so neither copy
    direction blocks the host.  Windows never exist on disk, and file pages behind the cursor are released.

    With `embeddings`, every chunk goes through gnm_embed_host instead (same probabilities, plus the encoder output of each
    window in a device chunk buffer), is summed per contig right away (segment_sum_rows, carried from chunk to chunk) and
    the per-contig means are combined over the ranks by the carry chain of genomad_b200.dist; returns (means, embeddings),
    the embeddings float32 [n_contigs, 512] on rank 0 and None on the other ranks.

    With `window_probs`, the per-window probabilities float32 [n_windows, 3] are collected on rank 0 (None on the other
    ranks) and returned last.  With offsets None there is no per-contig reduction: only those are returned.

    With `attributions` ({"target": class name}), every chunk goes through the attribution calls instead
    (Classifier.attribute_ascii: the same forward step, so bitwise the same probabilities, plus each window's 5,997
    attributions in a device buffer of this rank's shard); they are collected on rank 0 in window order and stored as
    attributions["attr"] (float32 [n_windows, 5997] on rank 0, None on the other ranks).  With attributions["steps"] >= 1 the
    calls are the integrated-gradients ones (Classifier.integrated_gradients_ascii, same probabilities), and the rows of
    log p_target at the window and at the baseline travel to rank 0 the same way, as attributions["logp"] (float32 [n_windows, 2]).
    With attributions["head"] true, the target is a class of the `head` and the calls are the head's (Head.attribute_ascii /
    integrated_gradients_ascii): one call gives the probabilities, the head's scores of the windows (bitwise Head.predict of
    their embeddings) and the attributions of the head's log p_target, so the chunk takes no other route.

    With `head` ({"head": engine.Head}), every chunk takes the embedding route and the head scores each window's embedding on
    the device into a buffer of this rank's shard; they are reduced per contig by the routes of the class scores (gather or
    allreduce, any width) and stored as head["preds"] (float32 [n_contigs, C], identical on all ranks).  With head["windows"]
    true, those rows are also collected on rank 0 in window order, as the class scores are with `window_probs`, and stored as
    head["window_preds"] (float32 [n_windows, C] on rank 0, None on the other ranks); with offsets None only that is done.
    With head["novelty"] true (the head carries a novelty model), the head also scores each window's embedding by
    Head.novelty into a second buffer of this rank's shard, reduced per contig the same way and stored as head["novelty_dist"]
    (float32 [n_contigs, C], identical on all ranks).
    With attributions["novelty"] (int32 [n_windows], each window's target class, in global window order), the calls are the
    head's novelty ones (Head.attribute_novelty_ascii / integrated_gradients_novelty_ascii) and each window's distance to its
    target travels to rank 0 as attributions["distance"] (float32 [n_windows]), with IG's (D_c(x), D_c(x')) rows as
    attributions["logp"].  With head["windows"] and head["novelty"] true, and head["window_novelty_wanted"] or no offsets, the
    windows' novelty rows are collected on rank 0 too, as head["window_novelty"] (float32 [n_windows, C]).
    With `window_embeddings` (float32 cuda [shard windows, 512]), each window's embedding is kept in its row of that matrix.
    """
    import torch
    from concurrent.futures import ThreadPoolExecutor
    n = parsed.n_windows
    start, end = gdist.shard_bounds(n, info.world_size, info.rank)
    chunk = max(4 * clf.max_batch, 4096)
    keep, bufs = zip(*(_pinned_chunk(min(chunk, max(1, end - start))) for _ in range(2)))
    out_t = _pinned_probs(max(1, end - start))
    dev = _device(clf)

    def sync():
        if dev.type == "cuda":
            torch.cuda.current_stream(dev).synchronize()

    def run(win, m, row):                                    # one chunk: windows win[:m] are rows [row, row + m) of the shard
        clf.classify_host_into(win.ctypes.data, m, out_t.data_ptr() + row * 12)
    scorer = head["head"] if head is not None else None
    nov = scorer is not None and bool(head.get("novelty"))
    if scorer is not None:
        d_head = torch.empty((end - start, scorer.n_classes), dtype=torch.float32, device=dev)
    if nov:
        d_nov = torch.empty((end - start, scorer.n_classes), dtype=torch.float32, device=dev)
    if embeddings:
        shard = gdist.EmbeddingShard(offsets, start, end, clf.segment_sum_rows, device=dev)
    if embeddings or scorer is not None or window_embeddings is not None:
        d_emb = torch.empty((min(chunk, max(1, end - start)), 512), dtype=torch.float32, device=dev)
        if attributions is None and (scorer is not None or window_embeddings is not None):
            def run(win, m, row):                            # the worker owns d_emb: one chunk at a time
                e = window_embeddings[row: row + m] if window_embeddings is not None else d_emb[:m]
                clf.embed_host_into(win.ctypes.data, m, out_t.data_ptr() + row * 12, e.data_ptr())
                if scorer is not None:
                    scorer.predict(e, out=d_head[row: row + m])
                if nov:
                    scorer.novelty(e, out=d_nov[row: row + m])
                if embeddings:
                    shard.add(e)
                sync()
        elif attributions is None:
            def run(win, m, row):                            # the worker owns d_emb: one chunk at a time
                clf.embed_host_into(win.ctypes.data, m, out_t.data_ptr() + row * 12, d_emb.data_ptr())
                shard.add(d_emb[:m])
                sync()
    if attributions is not None:
        d_attr = torch.empty((end - start, ATTR_TOKENS), dtype=torch.float32, device=dev)
        ig_steps = attributions.get("steps") or 0
        if ig_steps:
            d_logp = torch.empty((end - start, 2), dtype=torch.float32, device=dev)

        head_route = bool(attributions.get("head"))
        nov_targets = attributions.get("novelty")            # the novelty route: each window's target class, global order
        assert not (head_route or nov_targets is not None) or scorer is not None
        if nov_targets is not None:
            d_distance = torch.empty((end - start, 1), dtype=torch.float32, device=dev)

        def run(win, m, row):                                # probabilities and attributions from the attribution calls
            d_win = torch.from_numpy(win[:m]).to(dev)
            if nov_targets is not None:                      # the head's novelty distance to each window's target
                tg = np.ascontiguousarray(nov_targets[start + row: start + row + m], dtype=np.int32)
                if ig_steps:
                    probs, dist, dt, attr = scorer.integrated_gradients_novelty_ascii(d_win, tg, ig_steps,
                                                                                      attributions["baseline"])
                    d_logp[row: row + m].copy_(dt)
                else:
                    probs, dist, attr = scorer.attribute_novelty_ascii(d_win, tg)
                d_distance[row: row + m].copy_(dist.gather(1, torch.from_numpy(tg).to(dist.device, torch.int64)[:, None]))
            elif head_route:                                 # the head's scores come out of the same call
                if ig_steps:
                    probs, head_probs, logp, attr = scorer.integrated_gradients_ascii(d_win, attributions["target"], ig_steps,
                                                                                      attributions["baseline"])
                    d_logp[row: row + m].copy_(logp)
                else:
                    probs, head_probs, attr = scorer.attribute_ascii(d_win, attributions["target"])
                d_head[row: row + m].copy_(head_probs)
            elif ig_steps:
                probs, logp, attr = clf.integrated_gradients_ascii(d_win, attributions["target"], ig_steps,
                                                                   attributions["baseline"])
                d_logp[row: row + m].copy_(logp)
            else:
                probs, attr = clf.attribute_ascii(d_win, attributions["target"])
            out_t[row: row + m].copy_(probs)
            d_attr[row: row + m].copy_(attr)
            if embeddings or nov or (scorer is not None and not head_route and nov_targets is None):
                e = clf.embed_ascii(d_win)[1]
                if embeddings:
                    shard.add(e)
                if scorer is not None and not head_route and nov_targets is None:
                    scorer.predict(e, out=d_head[row: row + m])
                if nov:
                    scorer.novelty(e, out=d_nov[row: row + m])
            sync()
    futures = []
    with ThreadPoolExecutor(max_workers=1) as gpu:
        for i, a in enumerate(range(start, end, chunk)):
            b = min(end, a + chunk)
            if i >= 2:
                futures[i - 2].result()                          # buffer i%2 is free again
                parsed.release_before(a - chunk)
            win = parsed.export_windows(a, b - a, bufs[i % 2])
            futures.append(gpu.submit(run, win, b - a, a - start))
        for f in futures:
            f.result()
    del keep
    local_t = out_t[: end - start].to(dev, non_blocking=True)
    out = []
    if offsets is not None:
        out.append(_reduce_probs(clf, local_t, offsets, start, end, n, info, contig_reduce))
        if embeddings:
            lo, means = shard.finish(info)
            emb = gdist.gather_contig_means(lo, means, len(offsets) - 1, info)
            out.append(emb.cpu().numpy() if emb is not None else None)
        if scorer is not None:
            head["preds"] = _reduce_rows(scorer.segment_mean, scorer.segment_sum, d_head, offsets, start, end, n, info,
                                         contig_reduce)
            if nov:
                head["novelty_dist"] = _reduce_rows(scorer.segment_mean, scorer.segment_sum, d_nov, offsets, start, end, n,
                                                    info, contig_reduce)
    if window_probs:
        full = gdist.collect_window_probs(local_t, n, info)
        out.append(full.cpu().numpy() if full is not None else None)
    if scorer is not None and head.get("windows"):
        full = gdist.collect_window_probs(d_head, n, info)
        head["window_preds"] = full.cpu().numpy() if full is not None else None
        if nov and (offsets is None or head.get("window_novelty_wanted")):
            full = gdist.collect_window_probs(d_nov, n, info)
            head["window_novelty"] = full.cpu().numpy() if full is not None else None
    if attributions is not None:
        full = gdist.collect_window_probs(d_attr, n, info)
        attributions["attr"] = full.cpu().numpy() if full is not None else None
        if ig_steps:
            full = gdist.collect_window_probs(d_logp, n, info)
            attributions["logp"] = full.cpu().numpy() if full is not None else None
        if nov_targets is not None:
            full = gdist.collect_window_probs(d_distance, n, info)
            attributions["distance"] = full.reshape(-1).cpu().numpy() if full is not None else None
    if not out:
        return None
    return out[0] if len(out) == 1 else tuple(out)


def _reduce_probs(clf, local_t, offsets, start, end, n, info, contig_reduce) -> np.ndarray:
    """This rank's per-window probabilities (device) -> float32 [n_contigs, 3] per-contig means, identical on all ranks."""
    return _reduce_rows(lambda p, o: clf.segment_mean(p, o), lambda p, o: clf.segment_sum(p, o), local_t, offsets, start, end,
                        n, info, contig_reduce)


def _reduce_rows(segment_mean, segment_sum, local_t, offsets, start, end, n, info, contig_reduce) -> np.ndarray:
    """_reduce_probs for rows of any width C, given the segment mean ([W, C] -> [k, C]) and sum ([W, C] -> [k, C + 1])."""
    import torch
    dev = local_t.device
    if contig_reduce == "allreduce" and info.world_size > 1:
        loc_off = torch.from_numpy(gdist.local_offsets(offsets, start, end)).to(dev)
        partials = gdist.allreduce_partials(segment_sum(local_t, loc_off), info.world_size)
        return gdist.finish_mean(partials).cpu().numpy()
    probs = gdist.gather_window_probs(local_t, n, info.world_size)
    off_t = torch.from_numpy(offsets.astype(np.int32)).to(dev)
    return segment_mean(probs, off_t).cpu().numpy()


def _classify_windows(clf, windows: np.ndarray, offsets: np.ndarray, info: gdist.DistInfo,
                      contig_reduce: str = "gather") -> np.ndarray:
    """Same reduction for a window matrix that is already in memory (tools/multigpu_check.py, tests)."""
    import torch
    n = windows.shape[0]
    start, end = gdist.shard_bounds(n, info.world_size, info.rank)
    local = clf.classify_host(windows[start:end])
    local_t = torch.from_numpy(local).to(torch.device("cuda", clf.device))
    return _reduce_probs(clf, local_t, offsets, start, end, n, info, contig_reduce)


def _write_tsv(path: Path, names, preds) -> None:
    with open(path, "w") as fout:
        fout.write(_HEADER)
        for name, s in zip(names, preds):
            fout.write(f"{name}\t{float(s[0]):.4f}\t{float(s[1]):.4f}\t{float(s[2]):.4f}\n")


_WINDOW_HEADER = "seq_name\tstart\tend\tchromosome_score\tplasmid_score\tvirus_score\n"


def window_scores_enabled() -> bool:
    """Opt-in (``--write-window-scores`` / GENOMAD_B200_WINDOW_SCORES=1): also write the class scores of every window."""
    return os.environ.get("GENOMAD_B200_WINDOW_SCORES", "0") not in ("", "0")


def _write_window_tsv(path: Path, names, offsets, starts, lengths, probs, threads: int = 1, header: str = _WINDOW_HEADER,
                      n_cols: int = 3) -> None:
    """One row per window: name, 1-based start, inclusive end (in the record's sequence before stripping n/N), and the three
    scores (a head's table: its n_cols) with the digits of f"{x:.4f}" -- formatted natively on `threads` threads
    (gnm_write_window_tsv[_cols]): a profile can have hundreds of millions of rows."""
    from . import engine
    lib = engine.load_library()
    blobs = [str(x).encode() for x in names]
    name_off = np.zeros(len(blobs) + 1, dtype=np.int64)
    np.cumsum([len(b) for b in blobs], out=name_off[1:])
    blob = b"".join(blobs) or b"\0"
    offsets = np.ascontiguousarray(offsets, dtype=np.int32)
    starts = np.ascontiguousarray(starts, dtype=np.int64)
    lengths = np.ascontiguousarray(lengths, dtype=np.int32)
    probs = np.ascontiguousarray(probs, dtype=np.float32)
    assert len(offsets) == len(blobs) + 1 and len(starts) == len(lengths) == len(probs) == offsets[-1]
    if n_cols == 3:
        rc = lib.gnm_write_window_tsv(str(path).encode(), header.encode(), blob, name_off.ctypes.data, len(blobs),
                                      offsets.ctypes.data, starts.ctypes.data, lengths.ctypes.data, probs.ctypes.data,
                                      max(1, int(threads)))
    else:
        assert probs.size == len(starts) * n_cols
        rc = lib.gnm_write_window_tsv_cols(str(path).encode(), header.encode(), blob, name_off.ctypes.data, len(blobs),
                                           offsets.ctypes.data, starts.ctypes.data, lengths.ctypes.data, probs.ctypes.data,
                                           int(n_cols), max(1, int(threads)))
    if rc != 0:
        raise RuntimeError(lib.gnm_tsv_last_error().decode())


def _write_window_scores(npz_path: Path, tsv_path: Path, names_key: str, names, offsets, starts, lengths, probs, stride: int,
                         threads: int) -> None:
    offsets = np.asarray(offsets, dtype=np.int32)
    np.savez(npz_path, **{names_key: names,
                          "window_contig": np.repeat(np.arange(len(offsets) - 1, dtype=np.int32), np.diff(offsets)),
                          "window_start": np.asarray(starts, dtype=np.int64),
                          "window_length": np.asarray(lengths, dtype=np.int32),
                          "predictions": np.asarray(probs, dtype=np.float32).reshape(-1, 3),
                          "window_stride": np.int32(stride)})
    _write_window_tsv(tsv_path, names, offsets, starts, lengths, probs, threads)


def _write_head_windows(npz_path: Path, tsv_path: Path, names_key: str, names, offsets, starts, lengths, preds, stride: int,
                        class_names, head_sha: str, threads: int) -> None:
    """<prefix>_nn_classification_head_windows.{npz,tsv}: the window-score files' windows and keys, with the head's scores
    float32 [W, C] as predictions, plus class_names and head_sha256."""
    C = len(class_names)
    offsets = np.asarray(offsets, dtype=np.int32)
    preds = np.asarray(preds, dtype=np.float32).reshape(-1, C)
    np.savez(npz_path, **{names_key: names,
                          "window_contig": np.repeat(np.arange(len(offsets) - 1, dtype=np.int32), np.diff(offsets)),
                          "window_start": np.asarray(starts, dtype=np.int64),
                          "window_length": np.asarray(lengths, dtype=np.int32),
                          "predictions": preds,
                          "window_stride": np.int32(stride),
                          "class_names": np.array(class_names),
                          "head_sha256": np.str_(head_sha)})
    header = "seq_name\tstart\tend\t" + "\t".join(f"{c}_score" for c in class_names) + "\n"
    _write_window_tsv(tsv_path, names, offsets, starts, lengths, preds, threads, header=header, n_cols=C)


def _window_scores_current(npz_path: Path, tsv_path: Path, stride: int) -> bool:
    """Both window-score files exist and were written at this stride."""
    if not (npz_path.exists() and tsv_path.exists()):
        return False
    try:
        with np.load(npz_path) as z:
            return int(z["window_stride"]) == stride
    except Exception:
        return False


def _classify_windows_of(clf, parsed, index, stride: int, single_window: bool, info, contig_reduce, embeddings: bool,
                         attributions=None, head=None):
    """Per-contig scores (+ embeddings) and the per-window scores at `stride`: (preds, emb or None, offsets, starts, lengths,
    probs); the window arrays are None off rank 0.  At stride 6000 without --single-window the profile windows are the
    contig pass's own windows and their probabilities come out of that pass; otherwise a second pass classifies the list.
    With `head`, the head's scores of the same windows are stored as head["window_preds"] (rank 0): the contig pass's own
    rows, or the second pass's, which then takes the embedding route with the head (the same probabilities, bitwise)."""
    emb = None
    ak = {"attributions": attributions} if attributions is not None else {}      # option off: the call of before
    if head is not None:
        ak["head"] = head
        head["windows"] = stride == sequence.WINDOW and not single_window
    if stride == sequence.WINDOW and not single_window:
        res = _classify_parsed(clf, parsed, index.offsets, info, contig_reduce, embeddings=embeddings, window_probs=True, **ak)
        preds, probs = res[0], res[-1]
        if embeddings:
            emb = res[1]
        starts, lengths = parsed.spans() if info.is_main else (None, None)
        return preds, emb, index.offsets, starts, lengths, probs
    if embeddings:
        preds, emb = _classify_parsed(clf, parsed, index.offsets, info, contig_reduce, embeddings=True, **ak)
    else:
        preds = _classify_parsed(clf, parsed, index.offsets, info, contig_reduce, **ak)
    wl = parsed.windows(stride)
    try:
        if head is not None:
            profile = {"head": head["head"], "windows": True, "novelty": bool(head.get("window_novelty_wanted"))}
            probs = _classify_parsed(clf, wl, None, info, window_probs=True, head=profile)
            head["window_preds"] = profile["window_preds"]
            if profile["novelty"]:
                head["window_novelty"] = profile["window_novelty"]
        else:
            probs = _classify_parsed(clf, wl, None, info, window_probs=True)
        offsets, starts, lengths = wl.spans() if info.is_main else (None, None, None)
    finally:
        wl.close()
    return preds, emb, offsets, starts, lengths, probs


ATTR_TOKENS = 5997
ATTR_CLASSES = ("chromosome", "plasmid", "virus")


def attributions_target(value=None):
    """The class whose attributions are written (``--write-attributions CLASS`` / GENOMAD_B200_ATTRIBUTIONS=CLASS /
    main(..., write_attributions=CLASS)), or None.  value None: the environment decides; False / "" / "0": off."""
    if value is None:
        value = os.environ.get("GENOMAD_B200_ATTRIBUTIONS", "")
    if value is False or value is None or str(value).strip() in ("", "0"):
        return None
    v = str(value).strip().lower()
    if v not in ATTR_CLASSES:
        raise ValueError(f"attributions target must be one of {ATTR_CLASSES}, not {value!r}")
    return v


ATTR_BASELINES = ("zero", "N")
IG_METHOD = "integrated_gradients"


def attribution_steps(value=None) -> int:
    """Integrated-gradients steps of the attributions (``--attribution-steps N`` / GENOMAD_B200_ATTRIBUTION_STEPS=N /
    main(..., attribution_steps=N)): 0 (the default) keeps gradient x input, N >= 1 selects integrated gradients."""
    if value is None:
        value = os.environ.get("GENOMAD_B200_ATTRIBUTION_STEPS", "").strip() or 0
    from .engine import ATTR_MAX_BATCH
    try:
        v = int(value)
    except (TypeError, ValueError):
        raise ValueError(f"attribution steps must be an integer in [0, {ATTR_MAX_BATCH}], not {value!r}") from None
    if not 0 <= v <= ATTR_MAX_BATCH:
        raise ValueError(f"attribution steps must be in [0, {ATTR_MAX_BATCH}], not {value!r}")
    return v


def _check_ig_steps_fit(clf, steps: int) -> None:
    """A window's `steps` rows share one chunk of the attribution context, which holds min(ATTR_MAX_BATCH, the classifier's
    windows per step) rows (Classifier._attr_ctx); the step can be smaller than ATTR_MAX_BATCH on a device short of memory
    (device_step)."""
    from .engine import ATTR_MAX_BATCH
    limit = min(ATTR_MAX_BATCH, int(clf.max_batch))
    if steps > limit:
        raise ValueError(f"attribution steps must be at most {limit} on this device (the attribution context holds {limit} "
                         f"rows), not {steps}")


def attribution_baseline(value=None) -> str:
    """Baseline of integrated gradients (``--attribution-baseline {zero,N}`` / GENOMAD_B200_ATTRIBUTION_BASELINE /
    main(..., attribution_baseline=)): "zero" (all-zero one-hot rows, the default) or "N" (the all-N window)."""
    if value is None:
        value = os.environ.get("GENOMAD_B200_ATTRIBUTION_BASELINE", "").strip() or "zero"
    v = str(value).strip()
    if v not in ATTR_BASELINES:
        raise ValueError(f"attribution baseline must be one of {ATTR_BASELINES}, not {value!r}")
    return v


def head_attributions_target(value=None):
    """The class of the --head classifier whose attributions are written (``--write-head-attributions CLASS`` /
    GENOMAD_B200_HEAD_ATTRIBUTIONS=CLASS / main(..., write_head_attributions=CLASS)), or None; it is checked against the head
    file's class names once that is loaded.  value None: the environment decides; False / "" / "0": off."""
    if value is None:
        value = os.environ.get("GENOMAD_B200_HEAD_ATTRIBUTIONS", "")
    if value is False or value is None or str(value).strip() in ("", "0"):
        return None
    return str(value).strip()


def novelty_attributions_enabled(value=None) -> bool:
    """``--write-novelty-attributions`` / GENOMAD_B200_NOVELTY_ATTRIBUTIONS=1 / main(..., write_novelty_attributions=True):
    attribute each window's distance to its sequence's nearest class of the --head novelty model."""
    if value is None:
        return os.environ.get("GENOMAD_B200_NOVELTY_ATTRIBUTIONS", "0") not in ("", "0")
    return bool(value)


def window_novelty_enabled(value=None) -> bool:
    """``--write-window-novelty`` / GENOMAD_B200_WINDOW_NOVELTY=1 / main(..., write_window_novelty=True): write every window's
    distances to the --head novelty model's classes."""
    if value is None:
        return os.environ.get("GENOMAD_B200_WINDOW_NOVELTY", "0") not in ("", "0")
    return bool(value)


NOVELTY_TARGET = "nearest_class"


def _write_attributions(path: Path, names_key: str, names, offsets, starts, lengths, target: str, attr, steps: int = 0,
                        baseline: str = "zero", logp=None, extra=None) -> None:
    # np.savez, as for the embeddings: 24 KB of fp32 per window barely compresses
    offsets = np.asarray(offsets, dtype=np.int32)
    keys = {names_key: names,
            "window_contig": np.repeat(np.arange(len(offsets) - 1, dtype=np.int32), np.diff(offsets)),
            "window_start": np.asarray(starts, dtype=np.int64),
            "window_length": np.asarray(lengths, dtype=np.int32),
            "target": np.str_(target),
            "attributions": np.asarray(attr, dtype=np.float32).reshape(-1, ATTR_TOKENS)}
    if steps:                                       # integrated gradients; a gradient x input file keeps the keys above only
        keys.update({"method": np.str_(IG_METHOD), "steps": np.int32(steps), "baseline": np.str_(baseline),
                     "log_p_target": np.asarray(logp, dtype=np.float32).reshape(-1, 2)})
    keys.update(extra or {})                        # the head attributions file: head_sha256, class_names
    np.savez(path, **keys)


def _attributions_current(path: Path, target: str, steps: int = 0, baseline: str = "zero") -> bool:
    """The attributions file exists and was written for this class by this method (a file without "method" is gradient x
    input), with these integrated-gradients steps and baseline."""
    if not path.exists():
        return False
    try:
        with np.load(path) as z:
            if str(z["target"]) != target:
                return False
            method = str(z["method"]) if "method" in z.files else "gradient_x_input"
            if not steps:
                return method == "gradient_x_input"
            return method == IG_METHOD and int(z["steps"]) == steps and str(z["baseline"]) == baseline
    except Exception:
        return False


def _head_attributions_current(path: Path, target: str, head_sha: str, steps: int = 0, baseline: str = "zero") -> bool:
    """The head attributions file is current for this class, method, steps and baseline, and was written for this head."""
    if not _attributions_current(path, target, steps, baseline):
        return False
    try:
        with np.load(path) as z:
            return str(z["head_sha256"]) == head_sha
    except Exception:
        return False


def _write_head(npz_path: Path, tsv_path: Path, names_key: str, names, preds, class_names, head_sha: str) -> None:
    """<prefix>_nn_classification_head.{npz,tsv}: the head's per-sequence scores, float32 [n, C], one column per class."""
    preds = np.asarray(preds, dtype=np.float32).reshape(len(names), len(class_names))
    np.savez_compressed(npz_path, **{names_key: names, "predictions": preds, "class_names": np.array(class_names),
                                     "head_sha256": np.str_(head_sha)})
    with open(tsv_path, "w") as fout:
        fout.write("seq_name\t" + "\t".join(f"{c}_score" for c in class_names) + "\n")
        for name, row in zip(names, preds):
            fout.write(f"{name}" + "".join(f"\t{float(x):.4f}" for x in row) + "\n")


def _write_head_strands(npz_path: Path, tsv_path: Path, names_key: str, names, forward, reverse, class_names,
                        head_sha: str) -> None:
    """<prefix>_nn_classification_head_strands.{npz,tsv}: the head's float32 [n, C] per strand and their mean, laid out as the
    strand files are (strand outermost, class innermost), plus class_names and head_sha256."""
    from .engine import both_strands
    C = len(class_names)
    fwd = np.asarray(forward, dtype=np.float32).reshape(len(names), C)
    rev = np.asarray(reverse, dtype=np.float32).reshape(len(names), C)
    both = both_strands(fwd, rev)
    np.savez_compressed(npz_path, **{names_key: names, "forward": fwd, "reverse": rev, "both_strands": both,
                                     "class_names": np.array(class_names), "head_sha256": np.str_(head_sha)})
    with open(tsv_path, "w") as fout:
        fout.write("seq_name\t" + "\t".join(f"{c}_score_{s}" for s in STRANDS for c in class_names) + "\n")
        for name, a, b, c in zip(names, fwd, rev, both):
            fout.write(f"{name}" + "".join(f"\t{float(x):.4f}" for x in (*a, *b, *c)) + "\n")


_NOVELTY_HEADER = "seq_name\tnearest_class\tnovelty\tp_value\n"


def _write_head_novelty(npz_path: Path, tsv_path: Path, names_key: str, names, dist, counts, calibration, class_names,
                        head_sha: str) -> None:
    """<prefix>_nn_classification_head_novelty.{npz,tsv}: per sequence, the mean window distance to each of the head's classes
    (distances float32 [n, C]), the smallest (novelty), its class (nearest_class; -1 / NA without a window or with a
    non-finite distance) and the conformal
    p-value against the head's calibration values (engine.novelty_scores), plus class_names and head_sha256."""
    from .engine import novelty_scores
    C = len(class_names)
    dist = np.asarray(dist, dtype=np.float32).reshape(len(names), C)
    nov, nearest, p = novelty_scores(dist, counts, calibration)
    np.savez_compressed(npz_path, **{names_key: names, "distances": dist, "novelty": nov, "nearest_class": nearest,
                                     "p_value": p, "class_names": np.array(class_names), "head_sha256": np.str_(head_sha)})
    with open(tsv_path, "w") as fout:
        fout.write(_NOVELTY_HEADER)
        for name, c, v, pv in zip(names, nearest, nov, p):
            if c < 0:
                fout.write(f"{name}\tNA\tNA\tNA\n")
            else:
                fout.write(f"{name}\t{class_names[c]}\t{float(v):.6g}\t{float(pv):.6g}\n")


def _write_novelty_attributions(path: Path, names_key: str, names, offsets, starts, lengths, rec, steps: int, baseline: str,
                                class_names, head_sha: str) -> None:
    """<prefix>_nn_classification_head_novelty_attributions.npz: the attribution file's keys with target "nearest_class",
    each window's target_class int32 [W] and distance float32 [W] (D of the window to that class), class_names, head_sha256;
    with integrated gradients also method, steps, baseline and distance_target float32 [W, 2] = (D_c(x), D_c(x'))."""
    extra = {"target_class": np.asarray(rec["target_class"], dtype=np.int32),
             "distance": np.asarray(rec["distance"], dtype=np.float32).reshape(-1),
             "class_names": np.array(class_names), "head_sha256": np.str_(head_sha)}
    if steps:
        extra.update({"method": np.str_(IG_METHOD), "steps": np.int32(steps), "baseline": np.str_(baseline),
                      "distance_target": np.asarray(rec["logp"], dtype=np.float32).reshape(-1, 2)})
    _write_attributions(path, names_key, names, offsets, starts, lengths, NOVELTY_TARGET, rec["attr"], extra=extra)


def _write_window_novelty(npz_path: Path, tsv_path: Path, names_key: str, names, offsets, starts, lengths, dist, stride: int,
                          class_names, head_sha: str, threads: int) -> None:
    """<prefix>_nn_classification_head_novelty_windows.{npz,tsv}: the window-score files' windows and coordinate keys, each
    window's distances float32 [W, C] to the head's classes, novelty [W] (the row minimum), nearest_class int32 [W] (lowest
    index on ties; -1 and NaN for a row that is not all finite), window_stride, class_names and head_sha256.  The TSV holds
    the coordinates, the novelty and one distance column per class."""
    C = len(class_names)
    offsets = np.asarray(offsets, dtype=np.int32)
    dist = np.asarray(dist, dtype=np.float32).reshape(-1, C)
    ok = np.isfinite(dist).all(1)
    nov = np.full(len(dist), np.nan, np.float32)
    nearest = np.full(len(dist), -1, np.int32)
    if ok.any():
        nov[ok] = dist[ok].min(1)
        nearest[ok] = dist[ok].argmin(1)
    np.savez(npz_path, **{names_key: names,
                          "window_contig": np.repeat(np.arange(len(offsets) - 1, dtype=np.int32), np.diff(offsets)),
                          "window_start": np.asarray(starts, dtype=np.int64),
                          "window_length": np.asarray(lengths, dtype=np.int32),
                          "window_stride": np.int32(stride),
                          "distances": dist, "novelty": nov, "nearest_class": nearest,
                          "class_names": np.array(class_names), "head_sha256": np.str_(head_sha)})
    header = "seq_name\tstart\tend\tnovelty\t" + "\t".join(f"{c}_distance" for c in class_names) + "\n"
    _write_window_tsv(tsv_path, names, offsets, starts, lengths, np.concatenate([nov[:, None], dist], 1), threads,
                      header=header, n_cols=C + 1)


def _novelty_window_targets(dist, counts, calibration, names) -> np.ndarray:
    """int32 [W]: every window of the contig pass gets its sequence's nearest class (engine.novelty_scores of the novelty
    file's distances).  A sequence with windows but no nearest class (a distance that is not finite) is refused by name."""
    from .engine import GnmError, novelty_scores
    counts = np.asarray(counts, np.int64)
    _, nearest, _ = novelty_scores(dist, counts, calibration)
    bad = np.flatnonzero((nearest < 0) & (counts > 0))
    if bad.size:
        raise GnmError(f"{names[int(bad[0])]}: its window distances to the head's classes are not finite, so it has no "
                       "nearest class to attribute")
    return np.repeat(nearest, counts).astype(np.int32)


def _head_has_novelty(path) -> bool:
    """Whether a --head file carries a novelty model (its keys present; load_head checks them)."""
    from .weights import NOVELTY_KEYS
    try:
        with np.load(Path(path), allow_pickle=False) as z:
            return any(k in z.files for k in NOVELTY_KEYS)
    except Exception:
        return False


def _head_windows_current(npz_path: Path, tsv_path: Path, head_sha: str, stride: int) -> bool:
    """Both head window files exist and were written for this head at this stride."""
    if not _head_current(npz_path, tsv_path, head_sha):
        return False
    try:
        with np.load(npz_path) as z:
            return int(z["window_stride"]) == stride
    except Exception:
        return False


def _head_current(npz_path: Path, tsv_path: Path, head_sha: str) -> bool:
    """Both head files exist and were written for the head file with this sha256."""
    if not (npz_path.exists() and tsv_path.exists()):
        return False
    try:
        with np.load(npz_path) as z:
            return str(z["head_sha256"]) == head_sha
    except Exception:
        return False


def _load_head_file(path):
    """(weights.HeadFile, sha256 of the file) of a --head file, checked against the shipped encoder (ValueError otherwise)."""
    import hashlib
    from . import weights as _w
    head = _w.load_head(path, _w.load_weights())
    return head, hashlib.sha256(Path(path).read_bytes()).hexdigest()


def _make_head(clf, head_file):
    """Factory (patched in CPU tests): the head on the classifier's device."""
    from .engine import Head
    return Head(clf, head_file)


def tfrecords_enabled() -> bool:
    """Opt-in (``--write-tfrecords`` / GENOMAD_B200_TFRECORDS=1): also leave the reference's ``<count>.tfrec`` files."""
    return os.environ.get("GENOMAD_B200_TFRECORDS", "0") not in ("", "0")


def _write_tfrecords(clf, parsed, enc_dir: Path) -> int:
    """
    Byte-compatible stand-in for the reference's generate_data/write_tfrecord (nn_classification.py:43-82): windows are
    tokenised on the GPU (gnm_encode), copied back as uint16 and serialised natively, 10,000 windows per file named by the
    cumulative window count.  Returns the number of files.
    """
    import torch
    from . import tfrecord
    n, per = parsed.n_windows, tfrecord.RECORDS_PER_FILE
    if n == 0:
        return 0
    keep, buf = _pinned_chunk(min(per, n))
    dev = torch.device("cuda", clf.device)
    files = 0
    for a in range(0, n, per):
        b = min(n, a + per)
        win = parsed.export_windows(a, b - a, buf)
        tokens = clf.encode(keep[: b - a].to(dev, non_blocking=True)).cpu().numpy()
        assert win.shape[0] == tokens.shape[0]
        tfrecord.write_tfrecord(enc_dir / f"{b}.tfrec", tokens)
        files += 1
    return files


def embeddings_enabled() -> bool:
    """Opt-in (``--write-embeddings`` / GENOMAD_B200_EMBEDDINGS=1): also write the per-contig mean encoder embeddings."""
    return os.environ.get("GENOMAD_B200_EMBEDDINGS", "0") not in ("", "0")


def _write_embeddings(path: Path, names_key: str, names, emb, emb_reverse=None) -> None:
    # np.savez, not savez_compressed: 2 KB of fp32 per contig barely compresses, and zlib would turn writing a large
    # input's embeddings into minutes of work
    keys = {names_key: names, "embeddings": np.asarray(emb, dtype=np.float32)}
    if emb_reverse is not None:                     # --both-strands: "embeddings" keeps its bytes, two keys follow it
        from .engine import both_strands
        keys["embeddings_reverse"] = np.asarray(emb_reverse, dtype=np.float32)
        keys["embeddings_both_strands"] = both_strands(keys["embeddings"], keys["embeddings_reverse"])
    np.savez(path, **keys)


def both_strands_enabled() -> bool:
    """Opt-in (``--both-strands`` / GENOMAD_B200_BOTH_STRANDS=1): also classify every sequence's reverse complement and write
    the scores of each strand and their mean (and, with embeddings, the reverse strand's and the mean embeddings)."""
    return os.environ.get("GENOMAD_B200_BOTH_STRANDS", "0") not in ("", "0")


STRANDS = ("forward", "reverse", "both_strands")
_STRANDS_HEADER = ("seq_name\t" + "\t".join(f"{c}_score_{s}" for s in STRANDS for c in ("chromosome", "plasmid", "virus"))
                   + "\n")


def _write_strands(npz_path: Path, tsv_path: Path, names_key: str, names, forward, reverse) -> None:
    """<prefix>_nn_classification_strands.{npz,tsv}: float32 [n, 3] per strand and their mean, nine scores per TSV row."""
    from .engine import both_strands
    fwd, rev = np.asarray(forward, dtype=np.float32), np.asarray(reverse, dtype=np.float32)
    both = both_strands(fwd, rev)
    np.savez_compressed(npz_path, **{names_key: names, "forward": fwd, "reverse": rev, "both_strands": both})
    with open(tsv_path, "w") as fout:
        fout.write(_STRANDS_HEADER)
        for name, a, b, c in zip(names, fwd, rev, both):
            fout.write(f"{name}" + "".join(f"\t{float(x):.4f}" for x in (*a, *b, *c)) + "\n")


def _strands_current(npz_path: Path, tsv_path: Path, emb_path: Path, embeddings: bool) -> bool:
    """Both strand files exist and, with embeddings, the embeddings file holds the reverse strand's keys."""
    if not (npz_path.exists() and tsv_path.exists()):
        return False
    if not embeddings:
        return True
    try:
        with np.load(emb_path) as z:
            return "embeddings_reverse" in z.files and "embeddings_both_strands" in z.files
    except Exception:
        return False


def _classify_reverse(clf, parsed, single_window: bool, info, contig_reduce, embeddings: bool, head=None):
    """The reverse strand: the windows of every record's reverse complement (sequence.WindowList, reverse=True) through the
    forward pass's chunk loop, per-contig reduction, embedding carry chain and multi-GPU routes.  A record keeps its row: it
    has at least one window on either strand.  Returns (preds, embeddings or None).  With `head` ({"head": engine.Head}), the
    list takes the embedding route with the head, as the forward pass does, and the head's per-contig means of the reverse
    windows are stored as head["reverse_preds"] (float32 [n_contigs, C], identical on all ranks)."""
    wl = parsed.windows(sequence.WINDOW, single_window, reverse=True)
    hk = {}
    if head is not None:
        hk["head"] = rev_head = {"head": head["head"]}
    try:
        offsets = wl.spans()[0]
        if embeddings:
            res = _classify_parsed(clf, wl, offsets, info, contig_reduce, embeddings=True, **hk)
        else:
            res = _classify_parsed(clf, wl, offsets, info, contig_reduce, **hk), None
        if head is not None:
            head["reverse_preds"] = rev_head["preds"]
        return res
    finally:
        wl.close()


def _encode_stage(console, enc_dir: Path, id_path: Path, names_key, ids_key, what, is_main, parsed, classifier=None):
    """
    The reference's "encoding" stage (nn_classification.py:215-246) wrote TFRecords of tokens; here tokens never exist on
    the host, so by default the stage only records which window belongs to which sequence (<prefix>_seq_window_id.npz,
    same keys).  With tfrecords_enabled() it also writes the reference's .tfrec files (rank 0 only).
    """
    if enc_dir.is_dir() and is_main:
        shutil.rmtree(enc_dir)
    console.log(f"Creating the {enc_dir} directory.")
    if is_main:
        enc_dir.mkdir()
    index = parsed.index()
    if is_main:
        np.savez_compressed(id_path, **{names_key: index.names, ids_key: index.contig_ids})
        if tfrecords_enabled() and classifier is not None and parsed.n_windows:
            n_files = _write_tfrecords(classifier(), parsed, enc_dir)
            console.log(f"{n_files} TFRecord file(s) of tokenised windows written to {enc_dir.name}.")
    console.log(f"Encoded {what} data written to {enc_dir.name}.")
    return index


def contig_reduce_mode(default: str = "gather") -> str:
    """How per-contig means are combined when windows are sharded over GPUs (genomad_b200.dist): "gather" (default; outputs
    bitwise independent of the number of GPUs) or "allreduce" (per-contig partial sums; for few, long contigs).
    Chosen with GENOMAD_B200_CONTIG_REDUCE or main(..., contig_reduce=...)."""
    mode = os.environ.get("GENOMAD_B200_CONTIG_REDUCE", default).strip().lower() or default
    if mode not in ("gather", "allreduce"):
        raise ValueError(f"GENOMAD_B200_CONTIG_REDUCE must be 'gather' or 'allreduce', not {mode!r}")
    return mode


_attribution_steps, _attribution_baseline = attribution_steps, attribution_baseline


def main(input_path, output_path, single_window, batch_size, restart, threads, verbose, cleanup, *, contig_reduce=None,
         write_embeddings=None, write_window_scores=None, window_stride=None, write_attributions=None,
         attribution_steps=None, attribution_baseline=None, both_strands=None, head=None, write_head_attributions=None,
         write_novelty_attributions=None, write_window_novelty=None):
    import time as _time
    t_start = _time.perf_counter()
    last_timings.clear()
    input_path, output_path = Path(input_path), Path(output_path)
    info = gdist.init_process_group_if_needed()
    is_main = info.is_main
    contig_reduce = contig_reduce or contig_reduce_mode()
    write_embeddings = embeddings_enabled() if write_embeddings is None else bool(write_embeddings)
    strands = both_strands_enabled() if both_strands is None else bool(both_strands)
    # a stride asks for a profile: it implies the window scores unless they are switched off explicitly
    write_window_scores = ((window_scores_enabled() or window_stride is not None) if write_window_scores is None
                           else bool(write_window_scores))
    window_stride = sequence.WINDOW if window_stride is None else int(window_stride)
    attr_target = attributions_target(write_attributions)
    head_attr_target = head_attributions_target(write_head_attributions)
    if head_attr_target is not None and head is None:
        raise ValueError("--write-head-attributions needs --head: it names a class of the head file")
    if head_attr_target is not None and attr_target:
        raise ValueError("--write-head-attributions and --write-attributions cannot be combined in one run: the contig pass "
                         "runs through one kind of attribution call")
    nov_attr = novelty_attributions_enabled(write_novelty_attributions)
    window_nov = window_novelty_enabled(write_window_novelty)
    if nov_attr and head is None:
        raise ValueError("--write-novelty-attributions needs --head: it attributes the distance to the head's novelty model")
    if nov_attr and (attr_target or head_attr_target):
        raise ValueError("--write-novelty-attributions cannot be combined with --write-attributions or "
                         "--write-head-attributions: a run writes one attribution file")
    if window_nov and head is None:
        raise ValueError("--write-window-novelty needs --head: it scores the windows by the head's novelty model")
    any_attr = bool(attr_target or head_attr_target or nov_attr)
    # both options are validated whether or not they take effect; an option without effect is reported in the log
    steps_opt, baseline_opt = _attribution_steps(attribution_steps), _attribution_baseline(attribution_baseline)
    baseline_given = attribution_baseline is not None or bool(os.environ.get("GENOMAD_B200_ATTRIBUTION_BASELINE", "").strip())
    ig_notes = []
    if not any_attr and (steps_opt or baseline_given):
        ig_notes.append("--attribution-steps / --attribution-baseline have no effect without --write-attributions or "
                        "--write-head-attributions.")
    elif any_attr and baseline_given and not steps_opt:
        ig_notes.append("--attribution-baseline has no effect with --attribution-steps 0 (gradient x input).")
    ig_steps = steps_opt if any_attr else 0
    ig_baseline = baseline_opt if ig_steps else "zero"
    attr_method = f", integrated gradients, {ig_steps} steps, baseline {ig_baseline}" if ig_steps else ""
    if not 1 <= window_stride <= sequence.WINDOW:
        raise ValueError(f"window_stride must be in [1, {sequence.WINDOW}], not {window_stride}")
    if is_main:
        utils.start_md5(input_path)                      # hashed in the background while the file is indexed (rank 0 only)
    if not output_path.is_dir() and is_main:
        output_path.mkdir()
    prefix = input_path.stem
    if sequence.is_compressed(input_path) != sequence.Compression.uncompressed:
        prefix = prefix.rsplit(".", 1)[0]
    outputs = NNOutputs(prefix, output_path)
    console = utils.HybridConsole(output_file=outputs.nn_classification_log if is_main else None,
                                  verbose=verbose and is_main)
    parameter_dict = {"single_window": single_window}
    # Every decision that depends on what is on disk is taken by rank 0 alone and broadcast: the other ranks never consult
    # the file system for control flow (rank 0 rewrites the execution-info JSON and the outputs while they would look).
    classify_proviruses = gdist.broadcast_object(
        utils.check_provirus_execution(prefix, input_path, output_path) if is_main else None, info)

    files = [outputs.nn_classification_execution_info, outputs.encoded_sequences_dir,
             outputs.nn_classification_output, outputs.nn_classification_npz_output]
    descr = ["execution parameters", "directory containing encoded sequence data",
             "contig classification: tabular format", "contig classification: binary format"]
    if write_embeddings:
        files.append(outputs.nn_classification_embeddings_output)
        descr.append("contig embeddings: binary format")
    if write_window_scores:
        files += [outputs.nn_classification_windows_output, outputs.nn_classification_windows_npz_output]
        descr += ["window classification: tabular format", "window classification: binary format"]
    if attr_target:
        files.append(outputs.nn_classification_attributions_output)
        descr.append(f"window attributions ({attr_target}{attr_method}): binary format")
    if strands:
        files += [outputs.nn_classification_strands_output, outputs.nn_classification_strands_npz_output]
        descr += ["classification of both strands: tabular format", "classification of both strands: binary format"]
    if head is not None:
        files += [outputs.nn_classification_head_output, outputs.nn_classification_head_npz_output]
        descr += ["classification by the --head classifier: tabular format",
                  "classification by the --head classifier: binary format"]
    if head is not None and strands:
        files += [outputs.nn_classification_head_strands_output, outputs.nn_classification_head_strands_npz_output]
        descr += ["classification of both strands by the --head classifier: tabular format",
                  "classification of both strands by the --head classifier: binary format"]
    if head is not None and write_window_scores:
        files += [outputs.nn_classification_head_windows_output, outputs.nn_classification_head_windows_npz_output]
        descr += ["window classification by the --head classifier: tabular format",
                  "window classification by the --head classifier: binary format"]
    head_novelty = head is not None and _head_has_novelty(head)
    if head_novelty:
        files += [outputs.nn_classification_head_novelty_output, outputs.nn_classification_head_novelty_npz_output]
        descr += ["novelty with respect to the --head classifier's classes: tabular format",
                  "novelty with respect to the --head classifier's classes: binary format"]
    if head_attr_target:
        files.append(outputs.nn_classification_head_attributions_output)
        descr.append(f"window attributions of the --head classifier ({head_attr_target}{attr_method}): binary format")
    if nov_attr:
        files.append(outputs.nn_classification_head_novelty_attributions_output)
        descr.append(f"window attributions of the distance to the nearest class of the --head novelty model{attr_method}: "
                     "binary format")
    if window_nov:
        files += [outputs.nn_classification_head_novelty_windows_output,
                  outputs.nn_classification_head_novelty_windows_npz_output]
        descr += ["window novelty with respect to the --head classifier's classes: tabular format",
                  "window novelty with respect to the --head classifier's classes: binary format"]
    if classify_proviruses:
        files += [outputs.encoded_proviruses_dir, outputs.provirus_nn_classification_output,
                  outputs.provirus_nn_classification_npz_output]
        descr += ["directory containing encoded sequence data", "provirus classification: tabular format",
                  "provirus classification: binary format"]
        if write_embeddings:
            files.append(outputs.provirus_nn_classification_embeddings_output)
            descr.append("provirus embeddings: binary format")
        if write_window_scores:
            files += [outputs.provirus_nn_classification_windows_output, outputs.provirus_nn_classification_windows_npz_output]
            descr += ["provirus window classification: tabular format", "provirus window classification: binary format"]
        if attr_target:
            files.append(outputs.provirus_nn_classification_attributions_output)
            descr.append(f"provirus window attributions ({attr_target}{attr_method}): binary format")
        if strands:
            files += [outputs.provirus_nn_classification_strands_output, outputs.provirus_nn_classification_strands_npz_output]
            descr += ["provirus classification of both strands: tabular format",
                      "provirus classification of both strands: binary format"]
        if head is not None:
            files += [outputs.provirus_nn_classification_head_output, outputs.provirus_nn_classification_head_npz_output]
            descr += ["provirus classification by the --head classifier: tabular format",
                      "provirus classification by the --head classifier: binary format"]
        if head is not None and strands:
            files += [outputs.provirus_nn_classification_head_strands_output,
                      outputs.provirus_nn_classification_head_strands_npz_output]
            descr += ["provirus classification of both strands by the --head classifier: tabular format",
                      "provirus classification of both strands by the --head classifier: binary format"]
        if head is not None and write_window_scores:
            files += [outputs.provirus_nn_classification_head_windows_output,
                      outputs.provirus_nn_classification_head_windows_npz_output]
            descr += ["provirus window classification by the --head classifier: tabular format",
                      "provirus window classification by the --head classifier: binary format"]
        if head_novelty:
            files += [outputs.provirus_nn_classification_head_novelty_output,
                      outputs.provirus_nn_classification_head_novelty_npz_output]
            descr += ["provirus novelty with respect to the --head classifier's classes: tabular format",
                      "provirus novelty with respect to the --head classifier's classes: binary format"]
        if head_attr_target:
            files.append(outputs.provirus_nn_classification_head_attributions_output)
            descr.append(f"provirus window attributions of the --head classifier ({head_attr_target}{attr_method}): "
                         "binary format")
        if nov_attr:
            files.append(outputs.provirus_nn_classification_head_novelty_attributions_output)
            descr.append("provirus window attributions of the distance to the nearest class of the --head novelty model"
                         f"{attr_method}: binary format")
        if window_nov:
            files += [outputs.provirus_nn_classification_head_novelty_windows_output,
                      outputs.provirus_nn_classification_head_novelty_windows_npz_output]
            descr += ["provirus window novelty with respect to the --head classifier's classes: tabular format",
                      "provirus window novelty with respect to the --head classifier's classes: binary format"]
    utils.display_header(console, __version__, "nn-classification",
                         "This will classify the input sequences into chromosome, plasmid, or virus based on the "
                         "nucleotide sequence.", outputs.nn_classification_dir, files, descr)
    for note in ig_notes:
        console.log(f"Warning: {note}")
    head_file = head_sha = None
    if head is not None:             # a head for another encoder (or a malformed file) is refused before any work
        try:
            head_file, head_sha = _load_head_file(head)
        except (OSError, ValueError, KeyError) as e:
            console.error(f"{head} is not a usable head file: {e}")
            sys.exit(1)
        if head_attr_target is not None and head_attr_target not in head_file.class_names:
            console.error(f"--write-head-attributions {head_attr_target}: not a class of {head} "
                          f"({', '.join(head_file.class_names)})")
            sys.exit(1)
        if (nov_attr or window_nov) and head_file.novelty is None:
            opt = "--write-novelty-attributions" if nov_attr else "--write-window-novelty"
            console.error(f"{opt}: {head} carries no novelty model (train-head --novelty)")
            sys.exit(1)
    ig_clf = None
    if ig_steps:                     # the steps must fit this device's attribution context: fail before any work
        ig_clf = _make_classifier(batch_size, info.local_rank)
        _check_ig_steps_fit(ig_clf, ig_steps)

    parsed_input = sequence.ParsedFasta(input_path, single_window, threads)      # one native index pass: check + windows
    last_timings["index_s"] = _time.perf_counter() - t_start
    if not parsed_input.check():
        console.error(f"{input_path} is either empty or contains multiple entries with the same identifier. "
                      "Please check your input FASTA file and execute genomad nn-classification again.")
        sys.exit(1)
    console.log("Executing genomad nn-classification.")

    jobs = [("sequence", "contig", input_path, outputs.encoded_sequences_dir, outputs.seq_window_id_output,
             "contig_names", "contig_ids", outputs.nn_classification_npz_output, outputs.nn_classification_output, True,
             outputs.nn_classification_embeddings_output, outputs.nn_classification_windows_npz_output,
             outputs.nn_classification_windows_output, outputs.nn_classification_attributions_output,
             outputs.nn_classification_strands_npz_output, outputs.nn_classification_strands_output,
             outputs.nn_classification_head_npz_output, outputs.nn_classification_head_output,
             outputs.nn_classification_head_attributions_output,
             outputs.nn_classification_head_strands_npz_output, outputs.nn_classification_head_strands_output,
             outputs.nn_classification_head_windows_npz_output, outputs.nn_classification_head_windows_output,
             outputs.nn_classification_head_novelty_npz_output, outputs.nn_classification_head_novelty_output,
             outputs.nn_classification_head_novelty_attributions_output,
             outputs.nn_classification_head_novelty_windows_npz_output,
             outputs.nn_classification_head_novelty_windows_output)]
    if classify_proviruses:
        jobs.append(("provirus", "provirus", outputs.find_proviruses_nucleotide_output, outputs.encoded_proviruses_dir,
                     outputs.provirus_window_id_output, "provirus_names", "provirus_ids",
                     outputs.provirus_nn_classification_npz_output, outputs.provirus_nn_classification_output, False,
                     outputs.provirus_nn_classification_embeddings_output, outputs.provirus_nn_classification_windows_npz_output,
                     outputs.provirus_nn_classification_windows_output, outputs.provirus_nn_classification_attributions_output,
                     outputs.provirus_nn_classification_strands_npz_output, outputs.provirus_nn_classification_strands_output,
                     outputs.provirus_nn_classification_head_npz_output, outputs.provirus_nn_classification_head_output,
                     outputs.provirus_nn_classification_head_attributions_output,
                     outputs.provirus_nn_classification_head_strands_npz_output,
                     outputs.provirus_nn_classification_head_strands_output,
                     outputs.provirus_nn_classification_head_windows_npz_output,
                     outputs.provirus_nn_classification_head_windows_output,
                     outputs.provirus_nn_classification_head_novelty_npz_output,
                     outputs.provirus_nn_classification_head_novelty_output,
                     outputs.provirus_nn_classification_head_novelty_attributions_output,
                     outputs.provirus_nn_classification_head_novelty_windows_npz_output,
                     outputs.provirus_nn_classification_head_novelty_windows_output))

    plan = None
    info_writer = None
    if is_main:
        skip = False
        if outputs.nn_classification_execution_info.exists() and any(p.exists() for p in files) and not restart:
            if utils.compare_executions(input_path, parameter_dict, outputs.nn_classification_execution_info):
                skip = True
                console.log("Previous execution detected. Steps will be skipped unless their outputs are not found. "
                            "Use the --restart option to force the execution of all the steps again.")
            else:
                console.log("The input file or the parameters changed since the last execution. "
                            "Previous outputs will be overwritten.")
        if not outputs.nn_classification_dir.is_dir():
            console.log(f"Creating the {outputs.nn_classification_dir} directory.")
            outputs.nn_classification_dir.mkdir()
        # per job: (skip the encoding stage, skip the classification) -- decided BEFORE anything is rewritten
        # (with embeddings or window scores requested, a classification whose embeddings file is missing, or whose window
        # scores are missing or were written at another stride, or whose attributions are missing or were written for another
        # class, or whose strand files are missing, or whose head files are missing or were written for another head or
        # stride, is redone: same predictions, bit for bit)
        plan = [(bool(skip and j[4].exists()),
                 bool(skip and j[7].exists() and (not write_embeddings or j[10].exists())
                      and (not write_window_scores or _window_scores_current(j[11], j[12], window_stride))
                      and (not attr_target or _attributions_current(j[13], attr_target, ig_steps, ig_baseline))
                      and (not strands or _strands_current(j[14], j[15], j[10], write_embeddings))
                      and (head_file is None or _head_current(j[16], j[17], head_sha))
                      and (head_file is None or not strands or _head_current(j[19], j[20], head_sha))
                      and (head_file is None or not write_window_scores
                           or _head_windows_current(j[21], j[22], head_sha, window_stride))
                      and (not head_attr_target
                           or _head_attributions_current(j[18], head_attr_target, head_sha, ig_steps, ig_baseline))
                      and (head_file is None or head_file.novelty is None or _head_current(j[23], j[24], head_sha))
                      and (not nov_attr
                           or _head_attributions_current(j[25], NOVELTY_TARGET, head_sha, ig_steps, ig_baseline))
                      and (not window_nov or _head_windows_current(j[26], j[27], head_sha, window_stride))))
                for j in jobs]
        # The execution info carries the input's md5 (aggregated-classification cross-checks it).  md5 is sequential
        # (~0.6 GB/s): writing the JSON here, as the reference does, would hold the GPUs back until the whole file is hashed,
        # so it is written by a helper thread as soon as the background hash is done and joined before main() returns.
        import threading
        info_writer = threading.Thread(target=utils.write_execution_info, daemon=True,
                                       args=("nn_classification", input_path, parameter_dict,
                                             outputs.nn_classification_execution_info))
        info_writer.start()
    plan = gdist.broadcast_object(plan, info)

    # the classifier (CUDA context, weight upload, TMA descriptors: ~0.3 s) is built on a helper thread while the host
    # indexes; it is only joined when a job really has windows to classify
    from concurrent.futures import ThreadPoolExecutor
    clf_pool = ThreadPoolExecutor(max_workers=1)
    clf_future = None

    def classifier():
        nonlocal clf_future
        if ig_clf is not None:
            return ig_clf
        if clf_future is None:
            clf_future = clf_pool.submit(_make_classifier, batch_size, info.local_rank)
        return clf_future.result()

    scorer = None

    def head_scorer():
        nonlocal scorer
        if scorer is None:
            scorer = _make_head(classifier(), head_file)
        return scorer

    if not all(cls_skip for _, cls_skip in plan) and ig_clf is None:
        clf_future = clf_pool.submit(_make_classifier, batch_size, info.local_rank)      # start now, overlap with indexing

    # ---- stage 1, every job: "encode" (here: record the window -> sequence map; the windows themselves are streamed to the GPU in
    # stage 2).  Like the reference, sequences AND proviruses are encoded before either is classified (nn_classification.py:215-281).
    staged = []
    for (what, noun, fasta, enc_dir, id_path, names_key, ids_key, npz_path, tsv_path, must_have_windows, emb_path, *_), \
            (enc_skip, cls_skip) in zip(jobs, plan):
        parsed = index = None
        if enc_skip:
            console.log(f"{enc_dir.name} was found. Skipping {what} encoding.")
        else:
            parsed = parsed_input if what == "sequence" else sequence.ParsedFasta(fasta, single_window, threads)
            index = _encode_stage(console, enc_dir, id_path, names_key, ids_key, what, is_main, parsed, classifier)
        staged.append((parsed, index))

    # ---- stage 2, every job: classify, write NPZ, clean up, write TSV (nn_classification.py:283-353, 355-425)
    for (what, noun, fasta, enc_dir, id_path, names_key, ids_key, npz_path, tsv_path, must_have_windows, emb_path,
         win_npz_path, win_tsv_path, attr_path, strands_npz_path, strands_tsv_path, head_npz_path, head_tsv_path,
         head_attr_path, head_strands_npz_path, head_strands_tsv_path, head_win_npz_path, head_win_tsv_path,
         head_nov_npz_path, head_nov_tsv_path, nov_attr_path, win_nov_npz_path, win_nov_tsv_path), \
            (enc_skip, cls_skip), (parsed, index) \
            in zip(jobs, plan, staged):
        names = preds = emb = None
        rev_preds = rev_emb = None      # --both-strands: the reverse strand's scores and embeddings
        attr = None                     # the contig pass runs through the attribution calls
        if attr_target:
            attr = {"target": attr_target, **({"steps": ig_steps, "baseline": ig_baseline} if ig_steps else {})}
        elif head_attr_target:          # the same, through the head's attribution calls
            attr = {"target": head_attr_target, "head": True,
                    **({"steps": ig_steps, "baseline": ig_baseline} if ig_steps else {})}
        win = None                      # (offsets, starts, lengths, probs) of the window scores, on rank 0
        hd = None                       # --head: the chunk loop also scores every window with the head
        label = "Sequence" if what == "sequence" else "Provirus"      # the reference's log wording (nn_classification.py:333, 351, 407, 425)
        # ---- classify
        if cls_skip:
            console.log(f"{npz_path.name} was found. Skipping {what} classification.")
            if is_main:
                z = np.load(npz_path)
                names, preds = z[names_key], z["predictions"]
        else:
            if parsed is None:
                parsed = parsed_input if what == "sequence" else sequence.ParsedFasta(fasta, single_window, threads)
                index = parsed.index()
            if parsed.n_windows == 0:
                if must_have_windows:
                    console.error("No sequences were found. Please check your input FASTA.")
                    if info_writer is not None:
                        info_writer.join()                    # the reference has written the JSON by this point
                    sys.exit(1)
                names, preds = index.names, np.zeros((len(index.names), 3), np.float32)
                if head_file is not None:
                    C = len(head_file.class_names)
                    hd = {"preds": np.zeros((len(index.names), C), np.float32), "window_preds": np.zeros((0, C), np.float32)}
                    hd["reverse_preds"] = hd["preds"]
                    hd["novelty_dist"], hd["counts"] = hd["preds"], np.zeros(len(index.names), np.int64)
                    hd["window_novelty"] = hd["window_preds"]
                emb = np.zeros((len(index.names), 512), np.float32)
                win = (np.zeros(len(index.names) + 1, np.int32), np.zeros(0, np.int64), np.zeros(0, np.int32),
                       np.zeros((0, 3), np.float32))
                if attr is not None:
                    attr.update(attr=np.zeros((0, ATTR_TOKENS), np.float32), logp=np.zeros((0, 2), np.float32), spans=win[:3])
                if nov_attr:
                    nov_rec = {"attr": np.zeros((0, ATTR_TOKENS), np.float32), "logp": np.zeros((0, 2), np.float32),
                               "distance": np.zeros(0, np.float32), "target_class": np.zeros(0, np.int32), "spans": win[:3]}
                rev_preds, rev_emb = preds, emb
            else:
                t_c = _time.perf_counter()
                ak = {"attributions": attr} if attr is not None else {}      # option off: the calls of before
                if head_file is not None:
                    hd = {"head": head_scorer()}
                    if head_file.novelty is not None:
                        hd["novelty"] = True
                        hd["counts"] = np.diff(np.asarray(index.offsets, np.int64))
                        hd["window_novelty_wanted"] = window_nov
                    ak["head"] = hd
                if write_window_scores or window_nov:
                    preds, emb, *win = _classify_windows_of(classifier(), parsed, index, window_stride, single_window, info,
                                                            contig_reduce, write_embeddings, **ak)
                elif write_embeddings:
                    preds, emb = _classify_parsed(classifier(), parsed, index.offsets, info, contig_reduce, embeddings=True, **ak)
                else:
                    preds = _classify_parsed(classifier(), parsed, index.offsets, info, contig_reduce, **ak)
                if attr is not None:
                    attr["spans"] = (index.offsets, *parsed.spans()) if is_main else None
                if nov_attr:
                    # a second pass over the contig pass's windows through the novelty attribution calls, each window
                    # against its sequence's nearest class (head["novelty_dist"] is the same on every rank)
                    t_n = _time.perf_counter()
                    try:
                        targets = _novelty_window_targets(hd["novelty_dist"], hd["counts"],
                                                          head_file.novelty["novelty_calibration"], index.names)
                    except Exception as e:
                        console.error(str(e))
                        sys.exit(1)
                    nov_rec = {"target": NOVELTY_TARGET, "novelty": targets,
                               **({"steps": ig_steps, "baseline": ig_baseline} if ig_steps else {})}
                    _classify_parsed(classifier(), parsed, None, info, attributions=nov_rec, head={"head": head_scorer()})
                    nov_rec["target_class"] = targets
                    nov_rec["spans"] = (index.offsets, *parsed.spans()) if is_main else None
                    last_timings[f"novelty_attributions_{what}_s"] = _time.perf_counter() - t_n
                if strands:
                    rev_preds, rev_emb = _classify_reverse(classifier(), parsed, single_window, info, contig_reduce,
                                                           write_embeddings, head=hd)
                last_timings[f"classify_{what}_s"] = _time.perf_counter() - t_c          # incl. waiting for the CUDA context
                names = index.names
            console.log(f"{'Sequences' if what == 'sequence' else 'Proviruses'} classified.")
            if is_main:
                np.savez_compressed(npz_path, **{names_key: names, "predictions": preds.astype(np.float32)})
            console.log(f"{label} classification in binary format written to {npz_path.name}.")
            if write_embeddings:
                if is_main:
                    _write_embeddings(emb_path, names_key, names, emb, rev_emb if strands else None)
                console.log(f"{label} embeddings in binary format written to {emb_path.name}.")
            if strands:
                if is_main:
                    _write_strands(strands_npz_path, strands_tsv_path, names_key, names, preds.astype(np.float32), rev_preds)
                console.log(f"{label} classification of both strands written to {strands_tsv_path.name} and "
                            f"{strands_npz_path.name}.")
            if hd is not None:
                if is_main:
                    _write_head(head_npz_path, head_tsv_path, names_key, names, hd["preds"], head_file.class_names, head_sha)
                console.log(f"{label} classification by the head written to {head_tsv_path.name} and {head_npz_path.name}.")
                if strands:
                    if is_main:
                        _write_head_strands(head_strands_npz_path, head_strands_tsv_path, names_key, names, hd["preds"],
                                            hd["reverse_preds"], head_file.class_names, head_sha)
                    console.log(f"{label} classification of both strands by the head written to "
                                f"{head_strands_tsv_path.name} and {head_strands_npz_path.name}.")
                if head_file.novelty is not None:
                    if is_main:
                        _write_head_novelty(head_nov_npz_path, head_nov_tsv_path, names_key, names, hd["novelty_dist"],
                                            hd["counts"], head_file.novelty["novelty_calibration"], head_file.class_names,
                                            head_sha)
                    console.log(f"{label} novelty with respect to the head's classes (forward strand) written to "
                                f"{head_nov_tsv_path.name} and {head_nov_npz_path.name}.")
            if window_nov:
                if is_main:
                    _write_window_novelty(win_nov_npz_path, win_nov_tsv_path, names_key, names, *win[:3], hd["window_novelty"],
                                          window_stride, head_file.class_names, head_sha, threads or 1)
                console.log(f"{label} window novelty (stride {window_stride}) written to {win_nov_tsv_path.name} and "
                            f"{win_nov_npz_path.name}.")
            if nov_attr:
                if is_main:
                    _write_novelty_attributions(nov_attr_path, names_key, names, *nov_rec["spans"], nov_rec, ig_steps,
                                                ig_baseline, head_file.class_names, head_sha)
                console.log(f"{label} window attributions of the distance to the nearest class{attr_method} in binary "
                            f"format written to {nov_attr_path.name}.")
            if write_window_scores:
                if is_main:
                    _write_window_scores(win_npz_path, win_tsv_path, names_key, names, *win, window_stride,
                                         threads or 1)
                console.log(f"{label} window scores (stride {window_stride}) written to {win_tsv_path.name} and "
                            f"{win_npz_path.name}.")
                if hd is not None:
                    if is_main:
                        _write_head_windows(head_win_npz_path, head_win_tsv_path, names_key, names, *win[:3],
                                            hd["window_preds"], window_stride, head_file.class_names, head_sha, threads or 1)
                    console.log(f"{label} window scores of the head (stride {window_stride}) written to "
                                f"{head_win_tsv_path.name} and {head_win_npz_path.name}.")
            if attr is not None and head_attr_target:
                if is_main:
                    _write_attributions(head_attr_path, names_key, names, *attr["spans"], head_attr_target, attr["attr"],
                                        ig_steps, ig_baseline, attr.get("logp"),
                                        extra={"head_sha256": np.str_(head_sha),
                                               "class_names": np.array(head_file.class_names)})
                console.log(f"{label} window attributions of the head ({head_attr_target}{attr_method}) in binary format "
                            f"written to {head_attr_path.name}.")
            elif attr is not None:
                if is_main:
                    _write_attributions(attr_path, names_key, names, *attr["spans"], attr_target, attr["attr"], ig_steps,
                                        ig_baseline, attr.get("logp"))
                console.log(f"{label} window attributions ({attr_target}{attr_method}) in binary format written to "
                            f"{attr_path.name}.")
        if parsed is not None:
            parsed.close()
        if cleanup and is_main and enc_dir.is_dir():
            console.log(f"Deleting encoded {what} data.")
            shutil.rmtree(enc_dir)
        if is_main:
            _write_tsv(tsv_path, names, preds)
        console.log(f"{label} classification in tabular format written to {tsv_path.name}.")

    clf_pool.shutdown(wait=True)
    t_j = _time.perf_counter()
    if info_writer is not None:
        info_writer.join()
    last_timings["wait_for_md5_json_s"] = _time.perf_counter() - t_j
    gdist.barrier(info)
    last_timings["total_s"] = _time.perf_counter() - t_start                                   # rank 0 has written everything before any rank returns
    console.log("geNomad nn-classification finished!")
