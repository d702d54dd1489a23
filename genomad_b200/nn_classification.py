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


def _classify_parsed(clf, parsed, offsets: np.ndarray, info: gdist.DistInfo, contig_reduce: str = "gather") -> np.ndarray:
    """
    Indexed FASTA -> float32 [n_contigs, 3] per-contig mean (identical on all ranks).

    This rank's contiguous block of the global window list is streamed in chunks: the native reader fills one pinned
    chunk straight from the mmap'ed file (upper-case + pad, multi-threaded) while the GPU classifies the previous one
    (gnm_classify_host on a worker thread; the C call releases the GIL) into a pinned result buffer, so neither copy
    direction blocks the host.  Windows never exist on disk, and file pages behind the cursor are released.
    """
    import torch
    from concurrent.futures import ThreadPoolExecutor
    n = parsed.n_windows
    start, end = gdist.shard_bounds(n, info.world_size, info.rank)
    chunk = max(4 * clf.max_batch, 4096)
    keep, bufs = zip(*(_pinned_chunk(min(chunk, max(1, end - start))) for _ in range(2)))
    out_t = torch.empty((max(1, end - start), 3), dtype=torch.float32).pin_memory()
    futures = []
    with ThreadPoolExecutor(max_workers=1) as gpu:
        for i, a in enumerate(range(start, end, chunk)):
            b = min(end, a + chunk)
            if i >= 2:
                futures[i - 2].result()                          # buffer i%2 is free again
                parsed.release_before(a - chunk)
            win = parsed.export_windows(a, b - a, bufs[i % 2])
            futures.append(gpu.submit(clf.classify_host_into, win.ctypes.data, b - a,
                                      out_t.data_ptr() + (a - start) * 12))
        for f in futures:
            f.result()
    del keep
    dev = torch.device("cuda", clf.device)
    local_t = out_t[: end - start].to(dev, non_blocking=True)
    if contig_reduce == "allreduce" and info.world_size > 1:
        loc_off = torch.from_numpy(gdist.local_offsets(offsets, start, end)).to(dev)
        partials = gdist.allreduce_partials(clf.segment_sum(local_t, loc_off), info.world_size)
        return gdist.finish_mean(partials).cpu().numpy()
    probs = gdist.gather_window_probs(local_t, n, info.world_size)
    off_t = torch.from_numpy(offsets.astype(np.int32)).to(dev)
    return clf.segment_mean(probs, off_t).cpu().numpy()


def _classify_windows(clf, windows: np.ndarray, offsets: np.ndarray, info: gdist.DistInfo,
                      contig_reduce: str = "gather") -> np.ndarray:
    """Same reduction for a window matrix that is already in memory (tools/multigpu_check.py, tests)."""
    import torch
    n = windows.shape[0]
    start, end = gdist.shard_bounds(n, info.world_size, info.rank)
    local = clf.classify_host(windows[start:end])
    dev = torch.device("cuda", clf.device)
    local_t = torch.from_numpy(local).to(dev)
    if contig_reduce == "allreduce" and info.world_size > 1:
        loc_off = torch.from_numpy(gdist.local_offsets(offsets, start, end)).to(dev)
        partials = gdist.allreduce_partials(clf.segment_sum(local_t, loc_off), info.world_size)
        return gdist.finish_mean(partials).cpu().numpy()
    probs = gdist.gather_window_probs(local_t, n, info.world_size)
    off_t = torch.from_numpy(offsets.astype(np.int32)).to(dev)
    return clf.segment_mean(probs, off_t).cpu().numpy()


def _write_tsv(path: Path, names, preds) -> None:
    with open(path, "w") as fout:
        fout.write(_HEADER)
        for name, s in zip(names, preds):
            fout.write(f"{name}\t{float(s[0]):.4f}\t{float(s[1]):.4f}\t{float(s[2]):.4f}\n")


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


def main(input_path, output_path, single_window, batch_size, restart, threads, verbose, cleanup, *, contig_reduce=None):
    import time as _time
    t_start = _time.perf_counter()
    last_timings.clear()
    input_path, output_path = Path(input_path), Path(output_path)
    info = gdist.init_process_group_if_needed()
    is_main = info.is_main
    contig_reduce = contig_reduce or contig_reduce_mode()
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
    if classify_proviruses:
        files += [outputs.encoded_proviruses_dir, outputs.provirus_nn_classification_output,
                  outputs.provirus_nn_classification_npz_output]
        descr += ["directory containing encoded sequence data", "provirus classification: tabular format",
                  "provirus classification: binary format"]
    utils.display_header(console, __version__, "nn-classification",
                         "This will classify the input sequences into chromosome, plasmid, or virus based on the "
                         "nucleotide sequence.", outputs.nn_classification_dir, files, descr)

    parsed_input = sequence.ParsedFasta(input_path, single_window, threads)      # one native index pass: check + windows
    last_timings["index_s"] = _time.perf_counter() - t_start
    if not parsed_input.check():
        console.error(f"{input_path} is either empty or contains multiple entries with the same identifier. "
                      "Please check your input FASTA file and execute genomad nn-classification again.")
        sys.exit(1)
    console.log("Executing genomad nn-classification.")

    jobs = [("sequence", "contig", input_path, outputs.encoded_sequences_dir, outputs.seq_window_id_output,
             "contig_names", "contig_ids", outputs.nn_classification_npz_output, outputs.nn_classification_output, True)]
    if classify_proviruses:
        jobs.append(("provirus", "provirus", outputs.find_proviruses_nucleotide_output, outputs.encoded_proviruses_dir,
                     outputs.provirus_window_id_output, "provirus_names", "provirus_ids",
                     outputs.provirus_nn_classification_npz_output, outputs.provirus_nn_classification_output, False))

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
        plan = [(bool(skip and j[4].exists()), bool(skip and j[7].exists())) for j in jobs]
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
        if clf_future is None:
            clf_future = clf_pool.submit(_make_classifier, batch_size, info.local_rank)
        return clf_future.result()

    if not all(cls_skip for _, cls_skip in plan):
        clf_future = clf_pool.submit(_make_classifier, batch_size, info.local_rank)      # start now, overlap with indexing

    # ---- stage 1, every job: "encode" (here: record the window -> sequence map; the windows themselves are streamed to the GPU in
    # stage 2).  Like the reference, sequences AND proviruses are encoded before either is classified (nn_classification.py:215-281).
    staged = []
    for (what, noun, fasta, enc_dir, id_path, names_key, ids_key, npz_path, tsv_path, must_have_windows), \
            (enc_skip, cls_skip) in zip(jobs, plan):
        parsed = index = None
        if enc_skip:
            console.log(f"{enc_dir.name} was found. Skipping {what} encoding.")
        else:
            parsed = parsed_input if what == "sequence" else sequence.ParsedFasta(fasta, single_window, threads)
            index = _encode_stage(console, enc_dir, id_path, names_key, ids_key, what, is_main, parsed, classifier)
        staged.append((parsed, index))

    # ---- stage 2, every job: classify, write NPZ, clean up, write TSV (nn_classification.py:283-353, 355-425)
    for (what, noun, fasta, enc_dir, id_path, names_key, ids_key, npz_path, tsv_path, must_have_windows), \
            (enc_skip, cls_skip), (parsed, index) in zip(jobs, plan, staged):
        names = preds = None
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
            else:
                t_c = _time.perf_counter()
                preds = _classify_parsed(classifier(), parsed, index.offsets, info, contig_reduce)
                last_timings[f"classify_{what}_s"] = _time.perf_counter() - t_c          # incl. waiting for the CUDA context
                names = index.names
            console.log(f"{'Sequences' if what == 'sequence' else 'Proviruses'} classified.")
            if is_main:
                np.savez_compressed(npz_path, **{names_key: names, "predictions": preds.astype(np.float32)})
            console.log(f"{label} classification in binary format written to {npz_path.name}.")
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
