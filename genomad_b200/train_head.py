"""
``train-head``: train a classifier head for the user's own classes on the frozen encoder, the way the reference built its
classifier (genomad/neural_network/model.py:34-45, create_classifier: the encoder's layers frozen, Dense(512) +
BatchNormalization + ReLU + Dropout(0.2) + Dense(C, softmax) trained on its 512-value output).

The windows of the labelled sequences (the reference's windows: stride 6000, N rule) go once through nn-classification's
chunk loop on the embedding route; every window's embedding stays in a device matrix and takes its sequence's label.  The
head is then trained on that matrix (engine.HeadTrainer, include/gnm.h for the exact semantics).  The encoder runs in
inference mode: Keras' fit would also run the encoder's SpatialDropout layers, here the embeddings are computed once and cached,
which is what makes training cheap.  The head of the epoch with the lowest validation loss is written as
<prefix>_head.npz, for ``nn-classification --head``.

With ``--both-strands`` the windows of the same records' reverse complements (nn-classification --both-strands' reverse list)
are embedded too, into rows after the forward ones, and take the same labels: the head then learns from both strands, the
split stays by sequence (both strands of a sequence on the same side), and a validation sequence is scored by the mean of its
two strands' scores, as ``nn-classification --head --both-strands`` reports it.

With ``--novelty`` a novelty model is fitted once the best epoch is chosen (engine.novelty_fit on the training rows of the
embedding matrix: class means, shared covariance, whitening; DESIGN.md, "Head novelty") and calibrated on the validation
sequences: the novelty of each, from its forward-strand windows through the same device path nn-classification --head takes
(Head.novelty, then the head's segment mean, then the minimum over classes), sorted, is the head file's novelty_calibration.
"""
from __future__ import annotations

import sys
from pathlib import Path
from typing import List, Tuple

import numpy as np

from . import dist as gdist, sequence, utils, weights as _weights

MAX_LISTED = 10
EMBED_BYTES = 512 * 4
_TSV_HEADER = "epoch\ttrain_loss\tvalidation_loss\tvalidation_window_accuracy\tvalidation_sequence_accuracy\n"


def read_labels(path) -> Tuple[List[str], List[str]]:
    """LABELS.tsv -> (sequence names, class labels) in file order.  Header `seq_name<TAB>class`; blank lines are ignored."""
    lines = Path(path).read_text().splitlines()
    if not lines or lines[0].rstrip("\r").split("\t") != ["seq_name", "class"]:
        raise ValueError(f"{path}: the first line must be the header 'seq_name<TAB>class'")
    names, classes = [], []
    for i, line in enumerate(lines[1:], 2):
        line = line.rstrip("\r")
        if not line.strip():
            continue
        parts = line.split("\t")
        if len(parts) != 2 or not parts[0] or not parts[1]:
            raise ValueError(f"{path}, line {i}: expected two non-empty tab-separated fields (seq_name, class)")
        names.append(parts[0])
        classes.append(parts[1])
    return names, classes


def _listed(items) -> str:
    items = list(items)
    more = f" and {len(items) - MAX_LISTED} more" if len(items) > MAX_LISTED else ""
    return ", ".join(items[:MAX_LISTED]) + more


def class_names_of(classes) -> Tuple[str, ...]:
    """The head's classes: the sorted unique labels (the class-name rule and 2 <= C <= 32 enforced)."""
    return _weights.check_class_names(sorted(set(classes)))


def label_records(fasta_names, names, classes, class_names, skip=()) -> np.ndarray:
    """int32 [n_records]: each FASTA record's class index, -1 without a label.  A name labelled twice, or one that is not in
    the FASTA, is an error listing up to MAX_LISTED such names; names in `skip` (records without a sequence) are ignored."""
    seen, dup = set(), []
    for n in names:
        if n in seen and n not in dup:
            dup.append(n)
        seen.add(n)
    if dup:
        raise ValueError(f"{len(dup)} sequence name(s) labelled more than once: {_listed(dup)}")
    pos = {str(n): i for i, n in enumerate(fasta_names)}
    unknown = [n for n in names if n not in pos and n not in skip]
    if unknown:
        raise ValueError(f"{len(unknown)} labelled name(s) not found in the FASTA: {_listed(unknown)}")
    cidx = {c: i for i, c in enumerate(class_names)}
    out = np.full(len(fasta_names), -1, np.int32)
    for n, c in zip(names, classes):
        if n in pos:
            out[pos[n]] = cidx[c]
    return out


def split_sequences(seq_class: np.ndarray, n_classes: int, fraction: float, seed: int) -> np.ndarray:
    """bool [n_seq]: held out for validation.  Per class (in class order) the class's sequences are shuffled with
    numpy.random.default_rng(seed) and the first k = round(fraction * n_c) (half up) are held out; k >= 1 when n_c >= 2 and
    fraction > 0, and k <= n_c - 1, so every class keeps a training sequence."""
    rng = np.random.default_rng(seed)
    val = np.zeros(len(seq_class), bool)
    for c in range(n_classes):
        members = np.nonzero(seq_class == c)[0]
        n_c = len(members)
        k = int(np.floor(fraction * n_c + 0.5))
        if n_c >= 2 and fraction > 0:
            k = max(k, 1)
        k = min(k, max(n_c - 1, 0))
        val[rng.permutation(members)[:k]] = True
    return val


def class_weights(train_window_class: np.ndarray, n_classes: int, mode: str) -> np.ndarray:
    """float32 [C]: "balanced" = N / (C * N_c) over the training windows, "none" = 1."""
    if mode == "none":
        return np.ones(n_classes, np.float32)
    if mode != "balanced":
        raise ValueError(f"class weight must be 'balanced' or 'none', not {mode!r}")
    counts = np.bincount(train_window_class, minlength=n_classes).astype(np.float64)
    return (len(train_window_class) / (n_classes * counts)).astype(np.float32)


def epoch_order(train_rows: np.ndarray, seed: int, epoch: int) -> np.ndarray:
    """The training windows of one epoch in their seeded order."""
    return train_rows[np.random.default_rng([int(seed), int(epoch)]).permutation(len(train_rows))]


def validation_metrics(probs: np.ndarray, window_class: np.ndarray, seq_probs: np.ndarray, seq_class: np.ndarray,
                       cw: np.ndarray) -> Tuple[float, float, float]:
    """(weighted loss, window accuracy, sequence accuracy).  The loss is sum_i w_y (-log p_y) / n with p clipped to
    [1e-7, 1] as Keras clips probabilities in its cross-entropy."""
    p = np.clip(probs[np.arange(len(window_class)), window_class].astype(np.float64), 1e-7, 1.0)
    loss = float((cw[window_class].astype(np.float64) * -np.log(p)).sum() / len(window_class))
    win_acc = float((probs.argmax(1) == window_class).mean())
    seq_acc = float((seq_probs.argmax(1) == seq_class).mean())
    return loss, win_acc, seq_acc


class RecordWindows:
    """The windows of chosen records of a ParsedFasta, in file order: a window source of nn-classification's chunk loop
    (n_windows, export_windows, release_before), so only those records' windows are read and embedded.  Window w of this list
    is window starts[i] + (w - local[i]) of the file's list for its record i."""

    def __init__(self, parsed, offsets: np.ndarray, records: np.ndarray):
        offsets = np.asarray(offsets, np.int64)
        records = np.asarray(records, np.int64)
        self._parsed = parsed
        starts, counts = offsets[records], offsets[records + 1] - offsets[records]
        keep = counts > 0
        starts, counts = starts[keep], counts[keep]
        # runs of records whose windows follow each other in the file's list are exported in one call
        brk = np.r_[True, starts[1:] != starts[:-1] + counts[:-1]] if len(starts) else np.zeros(0, bool)
        first = np.nonzero(brk)[0]
        self._starts = starts[first]
        self._local = np.zeros(len(first) + 1, np.int64)
        np.cumsum(np.add.reduceat(counts, first) if len(first) else np.zeros(0, np.int64), out=self._local[1:])
        self.n_windows = int(self._local[-1])

    def _run(self, w: int) -> int:
        return int(np.searchsorted(self._local, w, side="right")) - 1

    def export_windows(self, first: int, count: int, out: np.ndarray) -> np.ndarray:
        pos = 0
        i = self._run(first)
        while pos < count:
            a = first + pos
            take = min(int(self._local[i + 1]) - a, count - pos)
            self._parsed.export_windows(int(self._starts[i]) + a - int(self._local[i]), take, out[pos: pos + take])
            pos += take
            i += 1
        return out[:count]

    def release_before(self, upto: int) -> None:
        if 0 < upto < self.n_windows:
            i = self._run(upto)
            self._parsed.release_before(int(self._starts[i]) + upto - int(self._local[i]))


def _make_classifier(device: int):
    """Factory (patched in CPU tests)."""
    from .nn_classification import _make_classifier as make
    return make(1024, device)


def _free_bytes(clf) -> int:
    import torch
    return int(torch.cuda.mem_get_info(clf.device)[0])


def _make_trainer(init, device, max_batch, seed, learning_rate):
    from .engine import HeadTrainer
    return HeadTrainer(init, device=device, max_batch=max_batch, seed=seed, learning_rate=learning_rate)


def _make_head(clf, head_file):
    from .engine import Head
    return Head(clf, head_file)


def _fit_novelty(clf, X, rows, labels, n_classes):
    """Factory (patched in CPU tests): engine.novelty_fit."""
    from .engine import novelty_fit
    return novelty_fit(clf, X, rows, labels, n_classes)


def calibration_values(head, X, rows, offsets) -> np.ndarray:
    """Sorted float32 novelty of the sequences whose windows are rows `rows` of X (int64 cuda, sequence by sequence, each
    sequence's rows delimited by `offsets`, int32 cuda [n + 1]): Head.novelty, the head's segment mean, the minimum over
    classes -- the values nn-classification --head computes for the same windows."""
    dist = head.segment_mean(head.novelty(X[rows]), offsets).cpu().numpy()
    return np.sort(dist.min(1)).astype(np.float32)


def main(input_path, labels_path, output_path, epochs: int = 10, batch_size: int = 256, learning_rate: float = 1e-3,
         validation_fraction: float = 0.1, class_weight: str = "balanced", seed: int = 0, threads=None,
         verbose: bool = True, both_strands: bool = False, novelty: bool = False) -> None:
    import torch
    from . import nn_classification as nnc
    from .engine import both_strands as both_strands_mean
    input_path, output_path = Path(input_path), Path(output_path)
    info = gdist.dist_info_from_env()
    if info.world_size > 1:
        utils.HybridConsole(verbose=True).error(
            f"train-head runs on one GPU; it was started with {info.world_size} processes. Run it without torchrun.")
        sys.exit(1)
    if epochs < 1 or batch_size < 1 or not 0.0 <= validation_fraction < 1.0 or not learning_rate > 0 or seed < 0:
        raise ValueError("epochs >= 1, batch_size >= 1, 0 <= validation_fraction < 1, learning_rate > 0 and seed >= 0 "
                         "are required")
    if novelty and validation_fraction == 0:
        raise ValueError("--novelty needs validation sequences to calibrate against: use a validation fraction > 0")
    output_path.mkdir(parents=True, exist_ok=True)
    prefix = input_path.stem
    if sequence.is_compressed(input_path) != sequence.Compression.uncompressed:
        prefix = prefix.rsplit(".", 1)[0]
    npz_path = output_path / f"{prefix}_head.npz"
    tsv_path = output_path / f"{prefix}_head_training.tsv"
    console = utils.HybridConsole(output_file=output_path / f"{prefix}_head_training.log", verbose=verbose)
    console.log(f"Executing genomad train-head on {input_path} with labels {labels_path}.")
    try:
        names, classes = read_labels(labels_path)
        class_names = class_names_of(classes)
    except ValueError as e:
        console.error(str(e))
        sys.exit(1)
    C = len(class_names)
    parsed = sequence.ParsedFasta(input_path, False, threads)
    rev_list = None
    try:
        if not parsed.check():
            console.error(f"{input_path} is either empty or contains multiple entries with the same identifier.")
            sys.exit(1)
        index = parsed.index()
        # the index lists the records that keep a sequence after stripping n/N; a labelled name outside it is either such an
        # empty record (no window: skipped) or not in the FASTA (an error), which only a pass over the headers can tell
        indexed = set(str(x) for x in index.names)
        outside = set(n for n in names if n not in indexed)
        empty = outside & {sequence.accession(h) for h, _ in sequence.iter_fasta(input_path, strip_n=False)} if outside else set()
        try:
            rec_class = label_records(index.names, names, classes, class_names, skip=empty)
        except ValueError as e:
            console.error(str(e))
            sys.exit(1)
        offsets = np.asarray(index.offsets, np.int64)
        counts = np.diff(offsets)
        labelled = rec_class >= 0
        n_records = len(index.names) + len(empty)     # records dropped by the index without a label are not counted
        console.log(f"{n_records - len(names)} FASTA record(s) without a label skipped; "
                    f"{len(empty) + int((labelled & (counts == 0)).sum())} labelled record(s) without a window skipped.")
        used = np.nonzero(labelled & (counts > 0))[0]
        seq_class = rec_class[used]
        missing = [class_names[c] for c in range(C) if not (seq_class == c).any()]
        if missing:
            console.error(f"class(es) without a sequence that has a window: {_listed(missing)}")
            sys.exit(1)
        val_seq = split_sequences(seq_class, C, validation_fraction, seed)
        if novelty and not val_seq.any():
            console.error("--novelty needs validation sequences to calibrate against, and this split holds none out (no class "
                          "has two sequences with a window); label more sequences or train without --novelty")
            sys.exit(1)
        # rows of X: the windows of the used records only, in file order; with both strands, then the same records' reverse
        # windows in file order (a record can have another number of windows on that strand: the N rule)
        strand_lists = [(RecordWindows(parsed, offsets, used), counts[used])]
        if both_strands:
            rev_list = parsed.windows(sequence.WINDOW, False, reverse=True)
            rev_offsets = np.asarray(rev_list.spans()[0], np.int64)
            strand_lists.append((RecordWindows(rev_list, rev_offsets, used), np.diff(rev_offsets)[used]))
        rows, base = [], 0                          # rows[k][i]: the rows of X of strand k of used record i
        for _, n_win in strand_lists:
            local = np.zeros(len(used) + 1, np.int64)
            np.cumsum(n_win, out=local[1:])
            rows.append([base + np.arange(local[i], local[i + 1]) for i in range(len(used))])
            base += int(local[-1])
        train_idx, val_idx = np.nonzero(~val_seq)[0], np.nonzero(val_seq)[0]
        train_rows = np.concatenate([r[i] for r in rows for i in train_idx]).astype(np.int64)
        val_rows = (np.concatenate([r[i] for r in rows for i in val_idx]) if len(val_idx) else np.zeros(0)).astype(np.int64)
        win_class = np.concatenate([np.repeat(seq_class, n_win) for _, n_win in strand_lists]).astype(np.int32)
        cw = class_weights(win_class[train_rows], C, class_weight)
        console.log(f"{C} classes ({', '.join(class_names)}); {len(used)} sequences: {int((~val_seq).sum())} for training "
                    f"({len(train_rows)} windows), {len(val_idx)} for validation ({len(val_rows)} windows); class weights "
                    + ", ".join(f"{x:.6g}" for x in cw) + ".")
        if both_strands:
            console.log("Training on both strands: every sequence's forward windows "
                        f"({strand_lists[0][0].n_windows} in all) and the windows of its reverse complement "
                        f"({strand_lists[1][0].n_windows}); validation sequences are scored by the mean of their two strands.")

        clf = _make_classifier(0)
        W = sum(src.n_windows for src, _ in strand_lists)
        if W * EMBED_BYTES > 0.9 * _free_bytes(clf):
            console.error(f"the embeddings of {W} windows ({W * EMBED_BYTES / 2**30:.1f} GiB) do not fit in the GPU's free "
                          "memory; train on fewer sequences")
            sys.exit(1)
        dev = torch.device("cuda", clf.device) if torch.cuda.is_available() else torch.device("cpu")
        X = torch.empty((W, 512), dtype=torch.float32, device=dev)
        console.log(f"Computing the encoder embeddings of {W} windows.")
        row = 0
        for src, _ in strand_lists:
            nnc._chunk_pass(clf, src, None, info, req=nnc.ChunkRequest(window_embeddings=X[row: row + src.n_windows]))
            row += src.n_windows
    finally:
        if rev_list is not None:
            rev_list.close()
        parsed.close()

    enc_w = _weights.load_weights()
    enc_sha = _weights.encoder_sha256(enc_w)
    trainer = _make_trainer(_weights.initial_head(C, seed), clf.device, batch_size, seed, learning_rate)
    labels_d = torch.from_numpy(win_class).to(dev)
    cw_d = torch.from_numpy(cw).to(dev)
    Xv = X[torch.from_numpy(val_rows).to(dev)] if len(val_rows) else None
    # validation rows are strand by strand; v_off[k] delimits strand k's windows of each validation sequence
    v_off, at = [], 0
    for r in rows:
        o = np.zeros(len(val_idx) + 1, np.int32)
        np.cumsum([len(r[i]) for i in val_idx], out=o[1:])
        v_off.append((at, torch.from_numpy(o).to(dev)))
        at += int(o[-1])
    N = len(train_rows)
    steps = -(-N // batch_size)
    sizes = torch.tensor([min(batch_size, N - s * batch_size) for s in range(steps)], dtype=torch.float64)
    best = None
    with open(tsv_path, "w") as tsv:
        tsv.write(_TSV_HEADER)
        for epoch in range(1, epochs + 1):
            order = torch.from_numpy(epoch_order(train_rows, seed, epoch)).to(dev)
            losses = torch.empty(steps, dtype=torch.float32, device=dev)
            for s in range(steps):
                trainer.step(X, order[s * batch_size: (s + 1) * batch_size], labels_d, cw_d, loss=losses[s: s + 1])
            train_loss = float((losses.double().cpu() * sizes).sum() / N)
            arrays = trainer.weights()
            metrics = (float("nan"),) * 3
            if Xv is not None:
                head = _make_head(clf, _weights.HeadFile(arrays, class_names, enc_sha))
                probs = head.predict(Xv)
                means = [head.segment_mean(probs[a: a + int(o[-1])], o) for a, o in v_off]
                seq_probs = (means[0] if len(means) == 1 else both_strands_mean(*means)).cpu().numpy()
                metrics = validation_metrics(probs.cpu().numpy(), win_class[val_rows], seq_probs, seq_class[val_idx], cw)
                head.close()
            tsv.write(f"{epoch}\t{train_loss:.6f}\t{metrics[0]:.6f}\t{metrics[1]:.6f}\t{metrics[2]:.6f}\n")
            console.log(f"Epoch {epoch}/{epochs}: train loss {train_loss:.4f}, validation loss {metrics[0]:.4f}, window "
                        f"accuracy {metrics[1]:.4f}, sequence accuracy {metrics[2]:.4f}.")
            if Xv is None or best is None or metrics[0] < best[1]:
                best = (epoch, metrics[0], arrays)
    trainer.close()
    nov = None
    if novelty:
        train_d = torch.from_numpy(train_rows).to(dev)
        fit = _fit_novelty(clf, X, train_d, labels_d, C)
        head = _make_head(clf, _weights.HeadFile(best[2], class_names, enc_sha))
        head.set_novelty(fit.center, fit.whitening, fit.means)
        fwd = [rows[0][i] for i in val_idx]                  # the validation sequences' forward-strand rows
        o = np.zeros(len(fwd) + 1, np.int32)
        np.cumsum([len(r) for r in fwd], out=o[1:])
        cal = calibration_values(head, X, torch.from_numpy(np.concatenate(fwd).astype(np.int64)).to(dev),
                                 torch.from_numpy(o).to(dev))
        head.close()
        nov = {"novelty_center": fit.center, "novelty_whitening": fit.whitening, "novelty_means": fit.means,
               "novelty_calibration": cal}
        console.log(f"Novelty model fitted on {len(train_rows)} training windows (shrinkage alpha 0.01, smallest Cholesky pivot "
                    f"{fit.min_pivot:.6g}) and calibrated on {len(cal)} validation sequences (novelty median "
                    f"{float(np.median(cal)):.4g}, max {float(cal[-1]):.4g}).")
    _weights.save_head(npz_path, best[2], class_names, enc_w, novelty=nov)
    console.log(f"Head of epoch {best[0]} written to {npz_path.name}; training record in {tsv_path.name}.")
    console.log("geNomad train-head finished!")
