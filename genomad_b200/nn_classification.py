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
from dataclasses import dataclass, replace
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


@dataclass(frozen=True)
class AttributionSpec:
    """What a chunk pass attributes to 4-mers: a class of the classifier (`target`), a class of the request's head (`target`,
    `head` true), or each window's distance to its target class of the head's novelty model (`novelty_targets`, int32
    [n_windows] in global window order).  `steps` >= 1 selects integrated gradients from `baseline`."""
    target: "str | None" = None
    head: bool = False
    novelty_targets: "np.ndarray | None" = None
    steps: int = 0
    baseline: str = "zero"


@dataclass(frozen=True)
class ChunkRequest:
    """What a chunk pass computes besides the class scores.  `head` (engine.Head) scores every window's embedding, and with
    `novelty` also its distances to the head's novelty classes.  `window_probs`, `window_head` and `window_novelty` collect
    those per-window rows on rank 0 in window order.  `window_embeddings` (float32 cuda [shard windows, 512]) keeps each
    window's embedding in its row."""
    embeddings: bool = False
    head: object = None
    novelty: bool = False
    window_probs: bool = False
    window_head: bool = False
    window_novelty: bool = False
    attribution: "AttributionSpec | None" = None
    window_embeddings: object = None


@dataclass(frozen=True)
class ChunkResult:
    """A chunk pass's results.  Per contig (only with offsets), identical on all ranks: preds float32 [n_contigs, 3],
    head_preds and novelty [n_contigs, C]; embeddings [n_contigs, 512] on rank 0.  Per window, on rank 0 (None on the other
    ranks): window_probs [n_windows, 3], head_window_preds and window_novelty [n_windows, C], attributions [n_windows, 5997],
    logp [n_windows, 2] (integrated gradients: log p_target, or the novelty distance, at the window and at the baseline) and
    distance [n_windows] (the novelty route: each window's distance to its target class)."""
    preds: "np.ndarray | None" = None
    embeddings: "np.ndarray | None" = None
    head_preds: "np.ndarray | None" = None
    novelty: "np.ndarray | None" = None
    window_probs: "np.ndarray | None" = None
    head_window_preds: "np.ndarray | None" = None
    window_novelty: "np.ndarray | None" = None
    attributions: "np.ndarray | None" = None
    logp: "np.ndarray | None" = None
    distance: "np.ndarray | None" = None


def _chunk_pass(clf, parsed, offsets, info: gdist.DistInfo, contig_reduce: str = "gather",
                req: ChunkRequest = ChunkRequest()) -> ChunkResult:
    """
    Indexed FASTA -> per-contig means of the class scores (and of whatever `req` asks for), reduced over `offsets`, or with
    offsets None only the per-window rows `req` collects.

    `parsed` is the window source: a ParsedFasta (the reference's windows) or a sequence.WindowList (windows at another
    stride); all the loop needs is n_windows, export_windows and release_before.

    This rank's contiguous block of the global window list is streamed in chunks: the native reader fills one pinned
    chunk straight from the mmap'ed file (upper-case + pad, multi-threaded) while the GPU classifies the previous one
    (on a worker thread; the C calls release the GIL) into a pinned result buffer, so neither copy direction blocks the
    host.  Windows never exist on disk, and file pages behind the cursor are released.

    Each chunk takes one route:
    * gnm_classify_host, when nothing but the class scores is asked for;
    * gnm_embed_host (the same probabilities, plus each window's encoder output on the device), with embeddings, a head or
      window_embeddings: the head scores the embeddings on the device, and the embeddings are summed per contig right away
      (segment_sum_rows, carried from chunk to chunk) and combined over the ranks by genomad_b200.dist's carry chain;
    * with an attribution, the classifier's or the head's attribution calls (the same forward step, so bitwise the same
      probabilities; a head route call also gives the head's scores), plus Classifier.embed_ascii only for embeddings,
      novelty or head scores that call does not give.
    Per-window rows live in device buffers of this rank's shard and are reduced per contig by the routes of the class
    scores (gather or allreduce, any width) or collected on rank 0 in window order.
    """
    import torch
    from concurrent.futures import ThreadPoolExecutor
    n = parsed.n_windows
    start, end = gdist.shard_bounds(n, info.world_size, info.rank)
    chunk = max(4 * clf.max_batch, 4096)
    keep, bufs = zip(*(_pinned_chunk(min(chunk, max(1, end - start))) for _ in range(2)))
    out_t = _pinned_probs(max(1, end - start))
    dev = _device(clf)
    scorer, nov, att, embeddings = req.head, req.head is not None and req.novelty, req.attribution, req.embeddings

    def sync():
        if dev.type == "cuda":
            torch.cuda.current_stream(dev).synchronize()

    if scorer is not None:
        d_head = torch.empty((end - start, scorer.n_classes), dtype=torch.float32, device=dev)
    if nov:
        d_nov = torch.empty((end - start, scorer.n_classes), dtype=torch.float32, device=dev)
    if embeddings:
        shard = gdist.EmbeddingShard(offsets, start, end, clf.segment_sum_rows, device=dev)

    if att is not None:
        d_attr = torch.empty((end - start, ATTR_TOKENS), dtype=torch.float32, device=dev)
        if att.steps:
            d_logp = torch.empty((end - start, 2), dtype=torch.float32, device=dev)
        nov_targets = att.novelty_targets
        assert not (att.head or nov_targets is not None) or scorer is not None
        if nov_targets is not None:
            d_distance = torch.empty((end - start, 1), dtype=torch.float32, device=dev)
        head_by_embedding = scorer is not None and not att.head and nov_targets is None

        def run(win, m, row):                                # one chunk: windows win[:m] are rows [row, row + m) of the shard
            d_win = torch.from_numpy(win[:m]).to(dev)
            if nov_targets is not None:                      # the head's novelty distance to each window's target
                tg = np.ascontiguousarray(nov_targets[start + row: start + row + m], dtype=np.int32)
                if att.steps:
                    probs, dist, dt, attr = scorer.integrated_gradients_novelty_ascii(d_win, tg, att.steps, att.baseline)
                    d_logp[row: row + m].copy_(dt)
                else:
                    probs, dist, attr = scorer.attribute_novelty_ascii(d_win, tg)
                d_distance[row: row + m].copy_(dist.gather(1, torch.from_numpy(tg).to(dist.device, torch.int64)[:, None]))
            elif att.head:                                   # the head's scores come out of the same call
                if att.steps:
                    probs, head_probs, logp, attr = scorer.integrated_gradients_ascii(d_win, att.target, att.steps,
                                                                                      att.baseline)
                    d_logp[row: row + m].copy_(logp)
                else:
                    probs, head_probs, attr = scorer.attribute_ascii(d_win, att.target)
                d_head[row: row + m].copy_(head_probs)
            elif att.steps:
                probs, logp, attr = clf.integrated_gradients_ascii(d_win, att.target, att.steps, att.baseline)
                d_logp[row: row + m].copy_(logp)
            else:
                probs, attr = clf.attribute_ascii(d_win, att.target)
            out_t[row: row + m].copy_(probs)
            d_attr[row: row + m].copy_(attr)
            if embeddings or nov or head_by_embedding:
                e = clf.embed_ascii(d_win)[1]
                if embeddings:
                    shard.add(e)
                if head_by_embedding:
                    scorer.predict(e, out=d_head[row: row + m])
                if nov:
                    scorer.novelty(e, out=d_nov[row: row + m])
            sync()
    elif embeddings or scorer is not None or req.window_embeddings is not None:
        if req.window_embeddings is None:
            d_emb = torch.empty((min(chunk, max(1, end - start)), 512), dtype=torch.float32, device=dev)

        def run(win, m, row):                                # the worker owns d_emb: one chunk at a time
            e = req.window_embeddings[row: row + m] if req.window_embeddings is not None else d_emb[:m]
            clf.embed_host_into(win.ctypes.data, m, out_t.data_ptr() + row * 12, e.data_ptr())
            if scorer is not None:
                scorer.predict(e, out=d_head[row: row + m])
            if nov:
                scorer.novelty(e, out=d_nov[row: row + m])
            if embeddings:
                shard.add(e)
            sync()
    else:
        def run(win, m, row):
            clf.classify_host_into(win.ctypes.data, m, out_t.data_ptr() + row * 12)
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

    def collect(rows):                                       # per-window rows -> rank 0, in window order
        full = gdist.collect_window_probs(rows, n, info)
        return full.cpu().numpy() if full is not None else None

    def reduce(mean, total, rows):
        return _reduce_rows(mean, total, rows, offsets, start, end, n, info, contig_reduce)
    res = {}
    if offsets is not None:
        res["preds"] = _reduce_probs(clf, local_t, offsets, start, end, n, info, contig_reduce)
        if embeddings:
            lo, means = shard.finish(info)
            emb = gdist.gather_contig_means(lo, means, len(offsets) - 1, info)
            res["embeddings"] = emb.cpu().numpy() if emb is not None else None
        if scorer is not None:
            res["head_preds"] = reduce(scorer.segment_mean, scorer.segment_sum, d_head)
            if nov:
                res["novelty"] = reduce(scorer.segment_mean, scorer.segment_sum, d_nov)
    if req.window_probs:
        res["window_probs"] = collect(local_t)
    if scorer is not None and req.window_head:
        res["head_window_preds"] = collect(d_head)
        if nov and req.window_novelty:
            res["window_novelty"] = collect(d_nov)
    if att is not None:
        res["attributions"] = collect(d_attr)
        if att.steps:
            res["logp"] = collect(d_logp)
        if nov_targets is not None:
            distance = collect(d_distance)
            res["distance"] = distance.reshape(-1) if distance is not None else None
    return ChunkResult(**res)


def _classify_parsed(clf, parsed, offsets, info: gdist.DistInfo, contig_reduce: str = "gather", embeddings: bool = False):
    """Per-contig class scores float32 [n_contigs, 3] (identical on all ranks), and with `embeddings` the pair (scores,
    per-contig mean embeddings float32 [n_contigs, 512] on rank 0, None on the other ranks): the chunk pass when nothing else
    is asked for.  It is the seam where tests substitute the classification of a whole window source."""
    res = _chunk_pass(clf, parsed, offsets, info, contig_reduce, ChunkRequest(embeddings=embeddings))
    return (res.preds, res.embeddings) if embeddings else res.preds


def _contig_pass(clf, parsed, offsets, info: gdist.DistInfo, contig_reduce: str, req: ChunkRequest) -> ChunkResult:
    """_chunk_pass of a per-contig request; one that asks for the class scores and embeddings only goes through
    _classify_parsed."""
    if req.head is not None or req.attribution is not None:
        return _chunk_pass(clf, parsed, offsets, info, contig_reduce, req)
    if req.embeddings:
        preds, emb = _classify_parsed(clf, parsed, offsets, info, contig_reduce, embeddings=True)
        return ChunkResult(preds=preds, embeddings=emb)
    return ChunkResult(preds=_classify_parsed(clf, parsed, offsets, info, contig_reduce))


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


def _write_score_tsv(path: Path, header: str, names, rows) -> None:
    """One line per sequence: its name, then every score of its row with the digits of f"{x:.4f}"."""
    with open(path, "w") as fout:
        fout.write(header)
        for name, row in zip(names, rows):
            fout.write(f"{name}" + "".join(f"\t{float(x):.4f}" for x in row) + "\n")


def _write_tsv(path: Path, names, preds) -> None:
    _write_score_tsv(path, _HEADER, names, preds)


def _window_coords(offsets, starts, lengths) -> dict:
    """The coordinate keys of every per-window file: each window's contig, 0-based start and length."""
    offsets = np.asarray(offsets, dtype=np.int32)
    return {"window_contig": np.repeat(np.arange(len(offsets) - 1, dtype=np.int32), np.diff(offsets)),
            "window_start": np.asarray(starts, dtype=np.int64),
            "window_length": np.asarray(lengths, dtype=np.int32)}


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
    np.savez(npz_path, **{names_key: names, **_window_coords(offsets, starts, lengths),
                          "predictions": np.asarray(probs, dtype=np.float32).reshape(-1, 3),
                          "window_stride": np.int32(stride)})
    _write_window_tsv(tsv_path, names, offsets, starts, lengths, probs, threads)


def _write_head_windows(npz_path: Path, tsv_path: Path, names_key: str, names, offsets, starts, lengths, preds, stride: int,
                        class_names, head_sha: str, threads: int) -> None:
    """<prefix>_nn_classification_head_windows.{npz,tsv}: the window-score files' windows and keys, with the head's scores
    float32 [W, C] as predictions, plus class_names and head_sha256."""
    C = len(class_names)
    preds = np.asarray(preds, dtype=np.float32).reshape(-1, C)
    np.savez(npz_path, **{names_key: names, **_window_coords(offsets, starts, lengths),
                          "predictions": preds,
                          "window_stride": np.int32(stride),
                          "class_names": np.array(class_names),
                          "head_sha256": np.str_(head_sha)})
    header = "seq_name\tstart\tend\t" + "\t".join(f"{c}_score" for c in class_names) + "\n"
    _write_window_tsv(tsv_path, names, offsets, starts, lengths, preds, threads, header=header, n_cols=C)


def _classify_windows_of(clf, parsed, index, stride: int, single_window: bool, info, contig_reduce, req: ChunkRequest,
                         window_novelty: bool = False):
    """The contig pass of `req`, plus the class scores of every window at `stride` (and with a head, the head's scores and,
    with `window_novelty`, its novelty rows): (ChunkResult, (offsets, starts, lengths) of those windows on rank 0).  At
    stride 6000 without --single-window the profile windows are the contig pass's own windows and their rows come out of that
    pass; otherwise a second pass over the window list collects them, with the head taking the embedding route (the same
    probabilities, bitwise)."""
    head = req.head is not None
    if stride == sequence.WINDOW and not single_window:
        res = _chunk_pass(clf, parsed, index.offsets, info, contig_reduce,
                          replace(req, window_probs=True, window_head=head, window_novelty=window_novelty))
        return res, (index.offsets, *(parsed.spans() if info.is_main else (None, None)))
    res = _chunk_pass(clf, parsed, index.offsets, info, contig_reduce, req)
    wl = parsed.windows(stride)
    try:
        prof = _chunk_pass(clf, wl, None, info, req=ChunkRequest(window_probs=True, head=req.head, window_head=head,
                                                                 novelty=window_novelty, window_novelty=window_novelty))
        spans = wl.spans() if info.is_main else (None, None, None)
    finally:
        wl.close()
    return replace(res, window_probs=prof.window_probs, head_window_preds=prof.head_window_preds,
                   window_novelty=prof.window_novelty), spans


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
    keys = {names_key: names, **_window_coords(offsets, starts, lengths),
            "target": np.str_(target),
            "attributions": np.asarray(attr, dtype=np.float32).reshape(-1, ATTR_TOKENS)}
    if steps:                                       # integrated gradients; a gradient x input file keeps the keys above only
        keys.update({"method": np.str_(IG_METHOD), "steps": np.int32(steps), "baseline": np.str_(baseline),
                     "log_p_target": np.asarray(logp, dtype=np.float32).reshape(-1, 2)})
    keys.update(extra or {})                        # the head attributions file: head_sha256, class_names
    np.savez(path, **keys)


# the value of a key that an output file may lack: an attributions file without "method" is gradient x input
_NPZ_ABSENT = {"method": "gradient_x_input"}


def _npz_current(paths, npz_path: Path, **keys) -> bool:
    """Every file of `paths` exists and the NPZ file `npz_path` holds each of `keys` with that value."""
    if not all(p.exists() for p in paths):
        return False
    try:
        with np.load(npz_path) as z:
            return all((z[k].item() if k in z.files else _NPZ_ABSENT.get(k)) == v for k, v in keys.items())
    except Exception:
        return False


def _write_head(npz_path: Path, tsv_path: Path, names_key: str, names, preds, class_names, head_sha: str) -> None:
    """<prefix>_nn_classification_head.{npz,tsv}: the head's per-sequence scores, float32 [n, C], one column per class."""
    preds = np.asarray(preds, dtype=np.float32).reshape(len(names), len(class_names))
    np.savez_compressed(npz_path, **{names_key: names, "predictions": preds, "class_names": np.array(class_names),
                                     "head_sha256": np.str_(head_sha)})
    _write_score_tsv(tsv_path, "seq_name\t" + "\t".join(f"{c}_score" for c in class_names) + "\n", names, preds)


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
    _write_score_tsv(tsv_path, "seq_name\t" + "\t".join(f"{c}_score_{s}" for s in STRANDS for c in class_names) + "\n",
                     names, np.concatenate([fwd, rev, both], 1))


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


def _write_novelty_attributions(path: Path, names_key: str, names, offsets, starts, lengths, target_class, res: ChunkResult,
                                steps: int, baseline: str, class_names, head_sha: str) -> None:
    """<prefix>_nn_classification_head_novelty_attributions.npz: the attribution file's keys with target "nearest_class",
    each window's target_class int32 [W] and distance float32 [W] (D of the window to that class), class_names, head_sha256;
    with integrated gradients also method, steps, baseline and distance_target float32 [W, 2] = (D_c(x), D_c(x'))."""
    extra = {"target_class": np.asarray(target_class, dtype=np.int32),
             "distance": np.asarray(res.distance, dtype=np.float32).reshape(-1),
             "class_names": np.array(class_names), "head_sha256": np.str_(head_sha)}
    if steps:
        extra.update({"method": np.str_(IG_METHOD), "steps": np.int32(steps), "baseline": np.str_(baseline),
                      "distance_target": np.asarray(res.logp, dtype=np.float32).reshape(-1, 2)})
    _write_attributions(path, names_key, names, offsets, starts, lengths, NOVELTY_TARGET, res.attributions, extra=extra)


def _write_window_novelty(npz_path: Path, tsv_path: Path, names_key: str, names, offsets, starts, lengths, dist, stride: int,
                          class_names, head_sha: str, threads: int) -> None:
    """<prefix>_nn_classification_head_novelty_windows.{npz,tsv}: the window-score files' windows and coordinate keys, each
    window's distances float32 [W, C] to the head's classes, novelty [W] (the row minimum), nearest_class int32 [W] (lowest
    index on ties; -1 and NaN for a row that is not all finite), window_stride, class_names and head_sha256.  The TSV holds
    the coordinates, the novelty and one distance column per class."""
    C = len(class_names)
    dist = np.asarray(dist, dtype=np.float32).reshape(-1, C)
    ok = np.isfinite(dist).all(1)
    nov = np.full(len(dist), np.nan, np.float32)
    nearest = np.full(len(dist), -1, np.int32)
    if ok.any():
        nov[ok] = dist[ok].min(1)
        nearest[ok] = dist[ok].argmin(1)
    np.savez(npz_path, **{names_key: names, **_window_coords(offsets, starts, lengths),
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
    _write_score_tsv(tsv_path, _STRANDS_HEADER, names, np.concatenate([fwd, rev, both], 1))


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


def _classify_reverse(clf, parsed, single_window: bool, info, contig_reduce, req: ChunkRequest) -> ChunkResult:
    """The reverse strand: the windows of every record's reverse complement (sequence.WindowList, reverse=True) through the
    forward pass's chunk loop, per-contig reduction, embedding carry chain and multi-GPU routes.  A record keeps its row: it
    has at least one window on either strand."""
    wl = parsed.windows(sequence.WINDOW, single_window, reverse=True)
    try:
        return _contig_pass(clf, wl, wl.spans()[0], info, contig_reduce, req)
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


@dataclass(frozen=True)
class _Options:
    """nn-classification's options, parsed and checked once.  attr_kind is the one attribution file of the run: "classifier",
    "head" or "novelty" (attr_target then is NOVELTY_TARGET); head_file and head_sha are set once the --head file is loaded."""
    contig_reduce: str
    embeddings: bool
    strands: bool
    window_scores: bool
    stride: int
    attr_kind: "str | None"
    attr_target: "str | None"
    steps: int
    baseline: str
    window_novelty: bool
    head: object
    head_novelty: bool
    notes: tuple
    threads: int
    head_file: object = None
    head_sha: "str | None" = None

    @property
    def attr_method(self) -> str:
        return f", integrated gradients, {self.steps} steps, baseline {self.baseline}" if self.steps else ""


def _parse_options(threads, contig_reduce, write_embeddings, write_window_scores, window_stride, write_attributions,
                   attribution_steps, attribution_baseline, both_strands, head, write_head_attributions,
                   write_novelty_attributions, write_window_novelty) -> _Options:
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
    attr_kind = "classifier" if attr_target else "head" if head_attr_target else "novelty" if nov_attr else None
    # both options are validated whether or not they take effect; an option without effect is reported in the log
    steps_opt, baseline_opt = _attribution_steps(attribution_steps), _attribution_baseline(attribution_baseline)
    baseline_given = attribution_baseline is not None or bool(os.environ.get("GENOMAD_B200_ATTRIBUTION_BASELINE", "").strip())
    notes = []
    if not attr_kind and (steps_opt or baseline_given):
        notes.append("--attribution-steps / --attribution-baseline have no effect without --write-attributions or "
                     "--write-head-attributions.")
    elif attr_kind and baseline_given and not steps_opt:
        notes.append("--attribution-baseline has no effect with --attribution-steps 0 (gradient x input).")
    steps = steps_opt if attr_kind else 0
    if not 1 <= window_stride <= sequence.WINDOW:
        raise ValueError(f"window_stride must be in [1, {sequence.WINDOW}], not {window_stride}")
    return _Options(contig_reduce=contig_reduce, embeddings=write_embeddings, strands=strands,
                    window_scores=write_window_scores, stride=window_stride, attr_kind=attr_kind,
                    attr_target={"classifier": attr_target, "head": head_attr_target, "novelty": NOVELTY_TARGET}.get(attr_kind),
                    steps=steps, baseline=baseline_opt if steps else "zero", window_novelty=window_nov, head=head,
                    head_novelty=head is not None and _head_has_novelty(head), notes=tuple(notes),
                    threads=threads or 1)


@dataclass(frozen=True)
class _Job:
    """One classification of the module: the input's sequences, or find-proviruses' proviruses.  Its output paths are the
    NNOutputs properties of the sequence job's names with `prefix` in front."""
    what: str
    noun: str
    fasta: Path
    enc_dir: Path
    id_path: Path
    names_key: str
    ids_key: str
    must_have_windows: bool
    outputs: NNOutputs
    prefix: str

    def path(self, name: str) -> Path:
        return getattr(self.outputs, self.prefix + name)

    @property
    def label(self) -> str:                  # the reference's log wording (nn_classification.py:333, 351, 407, 425)
        return "Sequence" if self.what == "sequence" else "Provirus"


@dataclass
class _Classified:
    """One job's classification, as the writers read it on rank 0: the contig pass (fwd), the reverse strand's (rev), the
    pass whose attributions are written (attr), the windows of the window files and of the attribution files (offsets,
    starts, lengths), the head's window count per sequence and each window's novelty target class."""
    names: object
    fwd: ChunkResult
    rev: "ChunkResult | None" = None
    attr: "ChunkResult | None" = None
    windows: tuple = (None, None, None)
    spans: tuple = (None, None, None)
    counts: "np.ndarray | None" = None
    target_class: "np.ndarray | None" = None

    @classmethod
    def empty(cls, names, n_classes: int) -> "_Classified":
        """A job without windows: zero scores and embeddings per sequence, no window rows."""
        n, C = len(names), n_classes
        rows = np.zeros((n, C), np.float32)
        none = np.zeros((0, C), np.float32)
        fwd = ChunkResult(preds=np.zeros((n, 3), np.float32), embeddings=np.zeros((n, 512), np.float32), head_preds=rows,
                          novelty=rows, window_probs=np.zeros((0, 3), np.float32), head_window_preds=none,
                          window_novelty=none, attributions=np.zeros((0, ATTR_TOKENS), np.float32),
                          logp=np.zeros((0, 2), np.float32), distance=np.zeros(0, np.float32))
        spans = (np.zeros(n + 1, np.int32), np.zeros(0, np.int64), np.zeros(0, np.int32))
        return cls(names, fwd, fwd, fwd, spans, spans, np.zeros(n, np.int64), np.zeros(0, np.int32))


@dataclass(frozen=True)
class _Product:
    """One opt-in output of a job: the NNOutputs properties of its files (a .tsv is described as tabular, a .npz as binary),
    when it is written, its header description and log line (str.format templates of _Product.fields), whether a previous
    run's files are current, and its writer (rank 0)."""
    files: tuple
    enabled: object
    descr: str
    log: str
    current: object
    write: object

    def fields(self, o: _Options, job: _Job) -> dict:
        named = {job.path(f).suffix[1:]: job.path(f).name for f in self.files}
        return {"p": "" if job.what == "sequence" else "provirus ", "noun": job.noun, "label": job.label, "stride": o.stride,
                "target": o.attr_target, "method": o.attr_method, **named}


def _attributions_keys(o: _Options, **keys) -> dict:
    """The keys that make an attributions file current: its class, method and integrated-gradients steps and baseline."""
    if not o.steps:
        return {"target": o.attr_target, "method": "gradient_x_input", **keys}
    return {"target": o.attr_target, "method": IG_METHOD, "steps": o.steps, "baseline": o.baseline, **keys}


def _write_attributions_of(o: _Options, j: _Job, r: _Classified, npz: Path, extra=None) -> None:
    _write_attributions(npz, j.names_key, r.names, *r.spans, o.attr_target, r.attr.attributions, o.steps, o.baseline,
                        r.attr.logp, extra=extra)


# Every opt-in output of a job, in the order the header lists them and the module writes them.  `current` and `write` take
# the options, the job and (write) its _Classified, then the row's files.
_PRODUCTS = (
    _Product(("nn_classification_embeddings_output",), lambda o: o.embeddings,
             "{noun} embeddings", "{label} embeddings in binary format written to {npz}.",
             lambda o, j, npz: npz.exists(),
             lambda o, j, r, npz: _write_embeddings(npz, j.names_key, r.names, r.fwd.embeddings,
                                                    r.rev.embeddings if o.strands else None)),
    _Product(("nn_classification_windows_output", "nn_classification_windows_npz_output"), lambda o: o.window_scores,
             "{p}window classification", "{label} window scores (stride {stride}) written to {tsv} and {npz}.",
             lambda o, j, tsv, npz: _npz_current((tsv, npz), npz, window_stride=o.stride),
             lambda o, j, r, tsv, npz: _write_window_scores(npz, tsv, j.names_key, r.names, *r.windows, r.fwd.window_probs,
                                                            o.stride, o.threads)),
    _Product(("nn_classification_attributions_output",), lambda o: o.attr_kind == "classifier",
             "{p}window attributions ({target}{method})",
             "{label} window attributions ({target}{method}) in binary format written to {npz}.",
             lambda o, j, npz: _npz_current((npz,), npz, **_attributions_keys(o)),
             _write_attributions_of),
    _Product(("nn_classification_strands_output", "nn_classification_strands_npz_output"), lambda o: o.strands,
             "{p}classification of both strands", "{label} classification of both strands written to {tsv} and {npz}.",
             lambda o, j, tsv, npz: _strands_current(npz, tsv, j.path("nn_classification_embeddings_output"), o.embeddings),
             lambda o, j, r, tsv, npz: _write_strands(npz, tsv, j.names_key, r.names, r.fwd.preds.astype(np.float32),
                                                      r.rev.preds)),
    _Product(("nn_classification_head_output", "nn_classification_head_npz_output"), lambda o: o.head is not None,
             "{p}classification by the --head classifier", "{label} classification by the head written to {tsv} and {npz}.",
             lambda o, j, tsv, npz: _npz_current((tsv, npz), npz, head_sha256=o.head_sha),
             lambda o, j, r, tsv, npz: _write_head(npz, tsv, j.names_key, r.names, r.fwd.head_preds, o.head_file.class_names,
                                                   o.head_sha)),
    _Product(("nn_classification_head_strands_output", "nn_classification_head_strands_npz_output"),
             lambda o: o.head is not None and o.strands,
             "{p}classification of both strands by the --head classifier",
             "{label} classification of both strands by the head written to {tsv} and {npz}.",
             lambda o, j, tsv, npz: _npz_current((tsv, npz), npz, head_sha256=o.head_sha),
             lambda o, j, r, tsv, npz: _write_head_strands(npz, tsv, j.names_key, r.names, r.fwd.head_preds,
                                                           r.rev.head_preds, o.head_file.class_names, o.head_sha)),
    _Product(("nn_classification_head_windows_output", "nn_classification_head_windows_npz_output"),
             lambda o: o.head is not None and o.window_scores,
             "{p}window classification by the --head classifier",
             "{label} window scores of the head (stride {stride}) written to {tsv} and {npz}.",
             lambda o, j, tsv, npz: _npz_current((tsv, npz), npz, head_sha256=o.head_sha, window_stride=o.stride),
             lambda o, j, r, tsv, npz: _write_head_windows(npz, tsv, j.names_key, r.names, *r.windows,
                                                           r.fwd.head_window_preds, o.stride, o.head_file.class_names,
                                                           o.head_sha, o.threads)),
    _Product(("nn_classification_head_novelty_output", "nn_classification_head_novelty_npz_output"),
             lambda o: o.head_novelty,
             "{p}novelty with respect to the --head classifier's classes",
             "{label} novelty with respect to the head's classes (forward strand) written to {tsv} and {npz}.",
             lambda o, j, tsv, npz: _npz_current((tsv, npz), npz, head_sha256=o.head_sha),
             lambda o, j, r, tsv, npz: _write_head_novelty(npz, tsv, j.names_key, r.names, r.fwd.novelty, r.counts,
                                                           o.head_file.novelty["novelty_calibration"],
                                                           o.head_file.class_names, o.head_sha)),
    _Product(("nn_classification_head_attributions_output",), lambda o: o.attr_kind == "head",
             "{p}window attributions of the --head classifier ({target}{method})",
             "{label} window attributions of the head ({target}{method}) in binary format written to {npz}.",
             lambda o, j, npz: _npz_current((npz,), npz, **_attributions_keys(o, head_sha256=o.head_sha)),
             lambda o, j, r, npz: _write_attributions_of(o, j, r, npz, extra={
                 "head_sha256": np.str_(o.head_sha), "class_names": np.array(o.head_file.class_names)})),
    _Product(("nn_classification_head_novelty_attributions_output",), lambda o: o.attr_kind == "novelty",
             "{p}window attributions of the distance to the nearest class of the --head novelty model{method}",
             "{label} window attributions of the distance to the nearest class{method} in binary format written to {npz}.",
             lambda o, j, npz: _npz_current((npz,), npz, **_attributions_keys(o, head_sha256=o.head_sha)),
             lambda o, j, r, npz: _write_novelty_attributions(npz, j.names_key, r.names, *r.spans, r.target_class, r.attr,
                                                              o.steps, o.baseline, o.head_file.class_names, o.head_sha)),
    _Product(("nn_classification_head_novelty_windows_output", "nn_classification_head_novelty_windows_npz_output"),
             lambda o: o.window_novelty,
             "{p}window novelty with respect to the --head classifier's classes",
             "{label} window novelty (stride {stride}) written to {tsv} and {npz}.",
             lambda o, j, tsv, npz: _npz_current((tsv, npz), npz, head_sha256=o.head_sha, window_stride=o.stride),
             lambda o, j, r, tsv, npz: _write_window_novelty(npz, tsv, j.names_key, r.names, *r.windows,
                                                             r.fwd.window_novelty, o.stride, o.head_file.class_names,
                                                             o.head_sha, o.threads)),
)


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
    opts = _parse_options(threads, contig_reduce, write_embeddings, write_window_scores, window_stride, write_attributions,
                          attribution_steps, attribution_baseline, both_strands, head, write_head_attributions,
                          write_novelty_attributions, write_window_novelty)
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

    jobs = [_Job("sequence", "contig", input_path, outputs.encoded_sequences_dir, outputs.seq_window_id_output,
                 "contig_names", "contig_ids", True, outputs, "")]
    if classify_proviruses:
        jobs.append(_Job("provirus", "provirus", outputs.find_proviruses_nucleotide_output, outputs.encoded_proviruses_dir,
                         outputs.provirus_window_id_output, "provirus_names", "provirus_ids", False, outputs, "provirus_"))
    products = [p for p in _PRODUCTS if p.enabled(opts)]
    files, descr = [outputs.nn_classification_execution_info], ["execution parameters"]
    for job in jobs:
        files += [job.enc_dir, job.path("nn_classification_output"), job.path("nn_classification_npz_output")]
        descr += ["directory containing encoded sequence data", f"{job.noun} classification: tabular format",
                  f"{job.noun} classification: binary format"]
        for p in products:
            files += [job.path(f) for f in p.files]
            descr += [p.descr.format(**p.fields(opts, job)) + (": tabular format" if job.path(f).suffix == ".tsv"
                                                               else ": binary format") for f in p.files]
    utils.display_header(console, __version__, "nn-classification",
                         "This will classify the input sequences into chromosome, plasmid, or virus based on the "
                         "nucleotide sequence.", outputs.nn_classification_dir, files, descr)
    for note in opts.notes:
        console.log(f"Warning: {note}")
    if head is not None:             # a head for another encoder (or a malformed file) is refused before any work
        try:
            head_file, head_sha = _load_head_file(head)
        except (OSError, ValueError, KeyError) as e:
            console.error(f"{head} is not a usable head file: {e}")
            sys.exit(1)
        if opts.attr_kind == "head" and opts.attr_target not in head_file.class_names:
            console.error(f"--write-head-attributions {opts.attr_target}: not a class of {head} "
                          f"({', '.join(head_file.class_names)})")
            sys.exit(1)
        if (opts.attr_kind == "novelty" or opts.window_novelty) and head_file.novelty is None:
            opt = "--write-novelty-attributions" if opts.attr_kind == "novelty" else "--write-window-novelty"
            console.error(f"{opt}: {head} carries no novelty model (train-head --novelty)")
            sys.exit(1)
        opts = replace(opts, head_file=head_file, head_sha=head_sha)
    ig_clf = None
    if opts.steps:                   # the steps must fit this device's attribution context: fail before any work
        ig_clf = _make_classifier(batch_size, info.local_rank)
        _check_ig_steps_fit(ig_clf, opts.steps)

    parsed_input = sequence.ParsedFasta(input_path, single_window, threads)      # one native index pass: check + windows
    last_timings["index_s"] = _time.perf_counter() - t_start
    if not parsed_input.check():
        console.error(f"{input_path} is either empty or contains multiple entries with the same identifier. "
                      "Please check your input FASTA file and execute genomad nn-classification again.")
        sys.exit(1)
    console.log("Executing genomad nn-classification.")

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
        # per job: (skip the encoding stage, skip the classification) -- decided BEFORE anything is rewritten; a
        # classification any of whose opt-in outputs is missing or was written for other options is redone (same
        # predictions, bit for bit)
        plan = [(bool(skip and job.id_path.exists()),
                 bool(skip and job.path("nn_classification_npz_output").exists()
                      and all(p.current(opts, job, *map(job.path, p.files)) for p in products)))
                for job in jobs]
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
            scorer = _make_head(classifier(), opts.head_file)
        return scorer

    if not all(cls_skip for _, cls_skip in plan) and ig_clf is None:
        clf_future = clf_pool.submit(_make_classifier, batch_size, info.local_rank)      # start now, overlap with indexing

    # ---- stage 1, every job: "encode" (here: record the window -> sequence map; the windows themselves are streamed to the GPU in
    # stage 2).  Like the reference, sequences AND proviruses are encoded before either is classified (nn_classification.py:215-281).
    staged = []
    for job, (enc_skip, cls_skip) in zip(jobs, plan):
        parsed = index = None
        if enc_skip:
            console.log(f"{job.enc_dir.name} was found. Skipping {job.what} encoding.")
        else:
            parsed = parsed_input if job.what == "sequence" else sequence.ParsedFasta(job.fasta, single_window, threads)
            index = _encode_stage(console, job.enc_dir, job.id_path, job.names_key, job.ids_key, job.what, is_main, parsed,
                                  classifier)
        staged.append((parsed, index))

    # ---- stage 2, every job: classify, write NPZ, clean up, write TSV (nn_classification.py:283-353, 355-425)
    for job, (enc_skip, cls_skip), (parsed, index) in zip(jobs, plan, staged):
        what, npz_path, tsv_path = job.what, job.path("nn_classification_npz_output"), job.path("nn_classification_output")
        # ---- classify
        if cls_skip:
            console.log(f"{npz_path.name} was found. Skipping {what} classification.")
            names = preds = None
            if is_main:
                z = np.load(npz_path)
                names, preds = z[job.names_key], z["predictions"]
        else:
            if parsed is None:
                parsed = parsed_input if what == "sequence" else sequence.ParsedFasta(job.fasta, single_window, threads)
                index = parsed.index()
            if parsed.n_windows == 0:
                if job.must_have_windows:
                    console.error("No sequences were found. Please check your input FASTA.")
                    if info_writer is not None:
                        info_writer.join()                    # the reference has written the JSON by this point
                    sys.exit(1)
                r = _Classified.empty(index.names, len(opts.head_file.class_names) if opts.head_file else 0)
            else:
                r = _classify_job(opts, classifier, head_scorer, parsed, index, single_window, info, what, console)
            names, preds = r.names, r.fwd.preds
            console.log(f"{'Sequences' if what == 'sequence' else 'Proviruses'} classified.")
            if is_main:
                np.savez_compressed(npz_path, **{job.names_key: names, "predictions": preds.astype(np.float32)})
            console.log(f"{job.label} classification in binary format written to {npz_path.name}.")
            for p in products:
                if is_main:
                    p.write(opts, job, r, *map(job.path, p.files))
                console.log(p.log.format(**p.fields(opts, job)))
        if parsed is not None:
            parsed.close()
        if cleanup and is_main and job.enc_dir.is_dir():
            console.log(f"Deleting encoded {what} data.")
            shutil.rmtree(job.enc_dir)
        if is_main:
            _write_tsv(tsv_path, names, preds)
        console.log(f"{job.label} classification in tabular format written to {tsv_path.name}.")

    clf_pool.shutdown(wait=True)
    t_j = _time.perf_counter()
    if info_writer is not None:
        info_writer.join()
    last_timings["wait_for_md5_json_s"] = _time.perf_counter() - t_j
    gdist.barrier(info)
    last_timings["total_s"] = _time.perf_counter() - t_start                                   # rank 0 has written everything before any rank returns
    console.log("geNomad nn-classification finished!")


def _classify_job(opts: _Options, classifier, head_scorer, parsed, index, single_window: bool, info, what: str,
                  console) -> _Classified:
    """The passes of one job with windows: the contig pass (with the window profile when window files are written), the
    novelty attribution pass and the reverse strand."""
    import time as _time
    t_c = _time.perf_counter()
    scorer = head_scorer() if opts.head is not None else None
    clf = classifier()
    att = None                       # the contig pass runs through the classifier's or the head's attribution calls
    if opts.attr_kind in ("classifier", "head"):
        att = AttributionSpec(opts.attr_target, opts.attr_kind == "head", steps=opts.steps, baseline=opts.baseline)
    req = ChunkRequest(embeddings=opts.embeddings, head=scorer, novelty=opts.head_novelty, attribution=att)
    windows = spans = (None, None, None)
    counts = target_class = rev = None
    if opts.window_scores or opts.window_novelty:
        fwd, windows = _classify_windows_of(clf, parsed, index, opts.stride, single_window, info, opts.contig_reduce, req,
                                            opts.window_novelty)
    else:
        fwd = _contig_pass(clf, parsed, index.offsets, info, opts.contig_reduce, req)
    attr = fwd
    if opts.attr_kind and info.is_main:
        spans = (index.offsets, *parsed.spans())
    if opts.head_novelty:
        counts = np.diff(np.asarray(index.offsets, np.int64))
    if opts.attr_kind == "novelty":
        # a second pass over the contig pass's windows through the novelty attribution calls, each window against its
        # sequence's nearest class (the per-contig novelty is the same on every rank)
        t_n = _time.perf_counter()
        try:
            target_class = _novelty_window_targets(fwd.novelty, counts, opts.head_file.novelty["novelty_calibration"],
                                                   index.names)
        except Exception as e:
            console.error(str(e))
            sys.exit(1)
        att = AttributionSpec(novelty_targets=target_class, steps=opts.steps, baseline=opts.baseline)
        attr = _chunk_pass(clf, parsed, None, info, req=ChunkRequest(head=scorer, attribution=att))
        last_timings[f"novelty_attributions_{what}_s"] = _time.perf_counter() - t_n
    if opts.strands:
        rev = _classify_reverse(clf, parsed, single_window, info, opts.contig_reduce,
                                ChunkRequest(embeddings=opts.embeddings, head=scorer))
    last_timings[f"classify_{what}_s"] = _time.perf_counter() - t_c          # incl. waiting for the CUDA context
    return _Classified(index.names, fwd, rev, attr, windows, spans, counts, target_class)
