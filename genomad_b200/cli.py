"""
Command line of the nn-classification module -- same arguments and options as
``genomad nn-classification`` (reference genomad/cli.py:714-774) -- and of its direct consumer
``genomad aggregated-classification`` (reference cli.py:776-803).  rich-click is not a dependency;
plain click gives the same option surface.

    python -m genomad_b200.cli nn-classification [OPTIONS] INPUT OUTPUT
    torchrun --nproc-per-node 8 -m genomad_b200.cli nn-classification INPUT OUTPUT     # 8 GPUs
"""
from __future__ import annotations

from pathlib import Path

import click

from . import __version__
from .utils import get_n_available_cpus

CONTEXT_SETTINGS = dict(help_option_names=["-h", "--help"])


@click.group(context_settings=CONTEXT_SETTINGS)
@click.version_option(version=__version__, prog_name="geNomad-H100")
def cli():
    """geNomad nn-classification on NVIDIA H100."""


@cli.command(name="nn-classification", context_settings=CONTEXT_SETTINGS)
@click.argument("input", type=click.Path(path_type=Path, exists=True))
@click.argument("output", type=click.Path(path_type=Path))
@click.option("--restart", is_flag=True, default=False, show_default=True,
              help="Overwrite existing intermediate files.")
@click.option("--threads", "-t", type=int, default=get_n_available_cpus(), show_default=True,
              help="Number of threads to use.")
@click.option("--verbose/--quiet", "-v/-q", is_flag=True, default=True, show_default=True,
              help="Display the execution log.")
@click.option("--cleanup", is_flag=True, default=False, show_default=True,
              help="Delete intermediate files after execution.")
@click.option("--single-window", is_flag=True, default=False, show_default=True,
              help="Use only the first window (6,000 bases) of each sequence to perform the classification.")
@click.option("--batch-size", type=int, default=128, show_default=True,
              help="Number of data points per batch of prediction.")
@click.option("--write-tfrecords", is_flag=True, default=False, show_default=True,
              help="Also write the reference's TFRecord intermediates (<count>.tfrec) to the encoded-sequences "
                   "directory. Not an option of the reference: it always writes them; here nothing reads them.")
@click.option("--write-embeddings", is_flag=True, default=False, show_default=True,
              help="Also write each sequence's mean encoder embedding (512 values, the network's vector representation) to "
                   "<prefix>_nn_classification_embeddings.npz. Not an option of the reference.")
@click.option("--write-window-scores", is_flag=True, default=False, show_default=True,
              help="Also write the class scores of every window, with its coordinates in the sequence, to "
                   "<prefix>_nn_classification_windows.{tsv,npz}: where along a sequence the chromosome, plasmid and virus "
                   "signal lies. With --head, the head's scores of the same windows also go to "
                   "<prefix>_nn_classification_head_windows.{tsv,npz}; every other file is unchanged. Not an option of the "
                   "reference.")
@click.option("--window-stride", type=click.IntRange(1, 6000), default=None, show_default="6000",
              help="Write the window scores (implies --write-window-scores) for a 6,000-base window every N bases (overlapping "
                   "windows when N < 6000), a finer score profile. Sequence scores always use the reference's windows. Not an "
                   "option of the reference.")
@click.option("--write-attributions", type=click.Choice(["chromosome", "plasmid", "virus"]), default=None,
              help="Also write, for every window of the classification, the gradient of the log-probability of this class "
                   "with respect to each one-hot 4-mer (gradient x input; position t covers bases t..t+3 of the window) to "
                   "<prefix>_nn_classification_attributions.npz: 5,997 float32 values, 24 KB per window, ~4 GB per Gbp of "
                   "input. About 4x the classification's GPU time. Not an option of the reference.")
@click.option("--attribution-steps", type=click.IntRange(0, 256), default=None, show_default="0",
              help="With --write-attributions: 0 writes gradient x input; N >= 1 writes integrated gradients with N steps "
                   "instead, attributions that add up to the change in log-probability from a baseline to the window, also for "
                   "windows classified with near certainty (where gradient x input is ~0). About 1 + 4.2 N times the "
                   "classification's GPU time; the file adds log_p_target (window, baseline). At most 256, and at most the windows per GPU "
                   "step of the device (checked before any work). Also applies to --write-head-attributions. Without either "
                   "option it has no effect (a warning is logged). Not an option of the reference.")
@click.option("--attribution-baseline", type=click.Choice(["zero", "N"]), default=None, show_default="zero",
              help="Baseline of integrated gradients: zero (all-zero one-hot input) or N (a window of N). Not an option of the "
                   "reference.")
@click.option("--both-strands", is_flag=True, default=False, show_default=True,
              help="Also classify every sequence's reverse complement and write the scores of the forward strand, the reverse "
                   "strand and their mean to <prefix>_nn_classification_strands.{tsv,npz}; with --write-embeddings the "
                   "embeddings file also gets embeddings_reverse and embeddings_both_strands. With --head, the head's scores "
                   "of both strands and their mean also go to <prefix>_nn_classification_head_strands.{tsv,npz}. The main "
                   "outputs are unchanged. About twice the GPU time. Not an option of the reference.")
@click.option("--head", "head", type=click.Path(path_type=Path, exists=True, dir_okay=False), default=None,
              help="Also score every sequence with this classifier head (a train-head output, <prefix>_head.npz) and write "
                   "the scores of its classes to <prefix>_nn_classification_head.{tsv,npz}. The head must have been trained "
                   "on this encoder (checked before any work). That file holds the forward strand's scores; with "
                   "--both-strands the head also scores the reverse strand (<prefix>_nn_classification_head_strands.{tsv,npz}) "
                   "and with --write-window-scores every window (<prefix>_nn_classification_head_windows.{tsv,npz}). The main "
                   "outputs are unchanged. Not an option of the reference.")
@click.option("--write-head-attributions", "write_head_attributions", metavar="CLASS", default=None,
              help="With --head: also write, for every window, the attributions of this class of the head (one of its "
                   "class names) to <prefix>_nn_classification_head_attributions.npz, as --write-attributions does for the "
                   "shipped classes; --attribution-steps and --attribution-baseline apply to it. Cannot be combined with "
                   "--write-attributions. Not an option of the reference.")
@click.option("--write-novelty-attributions", is_flag=True, default=False, show_default=True,
              help="With a --head that carries a novelty model: also attribute every window's distance to its sequence's "
                   "nearest class (the class of the novelty file) to the window's 4-mers, and write them to "
                   "<prefix>_nn_classification_head_novelty_attributions.npz; --attribution-steps and --attribution-baseline "
                   "apply to it. Cannot be combined with --write-attributions or --write-head-attributions. Costs one more "
                   "pass over the windows. Not an option of the reference.")
@click.option("--write-window-novelty", is_flag=True, default=False, show_default=True,
              help="With a --head that carries a novelty model: also write every window's distance to each of the head's "
                   "classes and its novelty (the smallest) to <prefix>_nn_classification_head_novelty_windows.{tsv,npz}, for "
                   "the windows of the window-score files (--window-stride applies). There are no per-window p-values: the "
                   "calibration set holds per-sequence means, whose quantiles do not describe single windows, whose "
                   "distances spread wider. Not an option of the reference.")
def nn_classification(input, output, single_window, batch_size, restart, threads, verbose, cleanup, write_tfrecords,
                      write_embeddings, write_window_scores, window_stride, write_attributions, attribution_steps,
                      attribution_baseline, both_strands, head, write_head_attributions, write_novelty_attributions,
                      write_window_novelty):
    """Classify the sequences in the INPUT file (FASTA format) using the geNomad neural network and write
    the results to the OUTPUT directory."""
    import os
    from . import nn_classification as module
    if write_tfrecords:
        os.environ["GENOMAD_B200_TFRECORDS"] = "1"
    extra = {}
    if write_window_scores:
        extra["write_window_scores"] = True
    if window_stride is not None:
        extra["window_stride"] = window_stride
    if write_attributions is not None:
        extra["write_attributions"] = write_attributions
    if attribution_steps is not None:
        extra["attribution_steps"] = attribution_steps
    if attribution_baseline is not None:
        extra["attribution_baseline"] = attribution_baseline
    if both_strands:
        extra["both_strands"] = True
    if head is not None:
        extra["head"] = head
    if write_head_attributions is not None:
        extra["write_head_attributions"] = write_head_attributions
    if write_novelty_attributions:
        extra["write_novelty_attributions"] = True
    if write_window_novelty:
        extra["write_window_novelty"] = True
    module.main(input, output, single_window, batch_size, restart, threads, verbose, cleanup,
                write_embeddings=True if write_embeddings else None, **extra)


@cli.command(name="train-head", context_settings=CONTEXT_SETTINGS)
@click.argument("input", type=click.Path(path_type=Path, exists=True, dir_okay=False))
@click.argument("labels", type=click.Path(path_type=Path, exists=True, dir_okay=False))
@click.argument("output", type=click.Path(path_type=Path))
@click.option("--epochs", type=click.IntRange(1), default=10, show_default=True, help="Passes over the training windows.")
@click.option("--batch-size", type=click.IntRange(1, 65536), default=256, show_default=True, help="Windows per training step.")
@click.option("--learning-rate", type=click.FloatRange(0, min_open=True), default=1e-3, show_default=True,
              help="Adam learning rate.")
@click.option("--validation-fraction", type=click.FloatRange(0, 1, max_open=True), default=0.1, show_default=True,
              help="Share of each class's sequences held out for validation (split by sequence, never by window).")
@click.option("--class-weight", type=click.Choice(["balanced", "none"]), default="balanced", show_default=True,
              help="balanced: class c weighs N / (C * N_c) in the loss, over the training windows; none: 1.")
@click.option("--seed", type=click.IntRange(0), default=0, show_default=True,
              help="Seed of the initialisation, split, order and dropout (>= 0).")
@click.option("--both-strands", is_flag=True, default=False, show_default=True,
              help="Also train on the windows of every labelled sequence's reverse complement, so the head scores a sequence "
                   "alike on either strand; the validation sequence accuracy then uses the strand-averaged scores that "
                   "nn-classification --head --both-strands writes. About twice the embedding time and time per epoch.")
@click.option("--novelty", is_flag=True, default=False, show_default=True,
              help="Also fit a novelty model (one Gaussian per class with a shared covariance, on the training windows' "
                   "embeddings) and calibrate it on the validation sequences, so nn-classification --head flags sequences "
                   "far from every class (<prefix>_nn_classification_head_novelty.{tsv,npz}). Needs a validation fraction > 0.")
@click.option("--threads", "-t", type=int, default=get_n_available_cpus(), show_default=True,
              help="Number of threads to use.")
@click.option("--verbose/--quiet", "-v/-q", is_flag=True, default=True, show_default=True,
              help="Display the execution log.")
def train_head(input, labels, output, epochs, batch_size, learning_rate, validation_fraction, class_weight, seed, both_strands,
               novelty, threads, verbose):
    """Train a classifier head for your own classes on the frozen encoder. LABELS is a TSV with the header
    seq_name<TAB>class and one row per labelled sequence of the INPUT FASTA (seq_name as nn-classification writes it).
    Writes <prefix>_head.npz (the epoch with the lowest validation loss), <prefix>_head_training.tsv and
    <prefix>_head_training.log to OUTPUT; score sequences with it by nn-classification --head. One GPU. Not a module of
    the reference."""
    from . import train_head as module
    extra = {"both_strands": True} if both_strands else {}
    if novelty:
        extra["novelty"] = True
    module.main(input, labels, output, epochs, batch_size, learning_rate, validation_fraction, class_weight, seed, threads,
                verbose, **extra)


@cli.command(name="embedding-neighbours", context_settings=CONTEXT_SETTINGS)
@click.argument("query", type=click.Path(path_type=Path, exists=True, dir_okay=False))
@click.argument("output", type=click.Path(path_type=Path))
@click.option("--reference", type=click.Path(path_type=Path, exists=True, dir_okay=False), default=None,
              help="Embeddings file of the sequences to search (nn-classification --write-embeddings output). Without it, the "
                   "query sequences are searched against each other, a sequence never being its own neighbour.")
@click.option("--neighbours", "-k", type=click.IntRange(1, 64), default=10, show_default=True,
              help="Neighbours per query sequence.")
@click.option("--both-strands", is_flag=True, default=False, show_default=True,
              help="Search the mean of both strands' embeddings (embeddings_both_strands, written by nn-classification "
                   "--write-embeddings --both-strands) of every input file, so a sequence and its reverse complement match.")
@click.option("--index", "index", type=click.Path(path_type=Path, exists=True, dir_okay=False), default=None,
              help="Search through this embedding-index file (embedding-index output) instead of comparing every pair: each "
                   "sequence scans only the sequences of its --nprobe nearest lists. The index must have been built on the reference file (the query file without --reference) "
                   "with the same --both-strands; checked before any work.")
@click.option("--nprobe", type=int, default=None,
              help="With --index: lists each sequence scans (1 to min(64, lists)); required with --index, since recall "
                   "against the exact search depends on it. At nprobe = lists the result is the exact search's.")
@click.option("--verbose/--quiet", "-v/-q", is_flag=True, default=True, show_default=True,
              help="Display the execution log.")
def embedding_neighbours(query, output, reference, neighbours, both_strands, index, nprobe, verbose):
    """Find the nearest neighbours, in cosine similarity of the encoder embeddings, of every sequence of the QUERY embeddings
    file (nn-classification --write-embeddings output) and write them to the OUTPUT directory as
    <prefix>_embedding_neighbours.{tsv,npz}. Not a module of the reference."""
    from . import embedding_neighbours as module
    extra = {} if index is None and nprobe is None else {"index": index, "nprobe": nprobe}
    module.main(query, reference, output, neighbours, verbose, both_strands=both_strands, **extra)


@cli.command(name="embedding-clusters", context_settings=CONTEXT_SETTINGS)
@click.argument("input", type=click.Path(path_type=Path, exists=True, dir_okay=False))
@click.argument("output", type=click.Path(path_type=Path))
@click.option("--min-similarity", type=click.FloatRange(0, 1, min_open=True), required=True,
              help="Cosine similarity a sequence needs with a representative to join its cluster, in (0, 1]. No default: "
                   "which level separates what in this embedding space has not been measured.")
@click.option("--both-strands", is_flag=True, default=False, show_default=True,
              help="Cluster the mean of both strands' embeddings (embeddings_both_strands, written by nn-classification "
                   "--write-embeddings --both-strands), so a sequence and its reverse complement share a cluster.")
@click.option("--index", "index", type=click.Path(path_type=Path, exists=True, dir_okay=False), default=None,
              help="Cluster through this embedding-index file (embedding-index output) instead of comparing every sequence with "
                   "every representative: a sequence is compared only with the representatives of its --nprobe nearest lists. "
                   "The index must have been built on the INPUT file (with --both-strands if given here).")
@click.option("--nprobe", type=int, default=None,
              help="With --index: lists each sequence is compared in (1 to min(64, lists)); required with --index. At "
                   "nprobe = lists the clusters are the exact ones.")
@click.option("--verbose/--quiet", "-v/-q", is_flag=True, default=True, show_default=True,
              help="Display the execution log.")
def embedding_clusters(input, output, min_similarity, both_strands, index, nprobe, verbose):
    """Cluster the sequences of the INPUT embeddings file (nn-classification --write-embeddings output) greedily, in file
    order, at a cosine similarity threshold of the encoder embeddings, and write each sequence's representative to the OUTPUT
    directory as <prefix>_embedding_clusters.{tsv,npz}. A representative is the first member of its cluster in file order.
    Not a module of the reference."""
    from . import embedding_clusters as module
    extra = {} if index is None and nprobe is None else {"index": index, "nprobe": nprobe}
    module.main(input, output, min_similarity, verbose, both_strands=both_strands, **extra)


@cli.command(name="embedding-map", context_settings=CONTEXT_SETTINGS)
@click.argument("input", type=click.Path(path_type=Path, exists=True, dir_okay=False))
@click.argument("output", type=click.Path(path_type=Path))
@click.option("-k", "k", type=int, default=15, show_default=True,
              help="Neighbours of each sequence the map keeps close, other sequences only (1 to 64, fewer than the sequences; "
                   "umap-learn's n_neighbors = k + 1).")
@click.option("--epochs", type=int, default=None, show_default="500 for up to 10,000 sequences, else 200",
              help="Layout epochs.")
@click.option("--seed", type=int, default=0, show_default=True,
              help="Seed of the initial noise and the negative samples: the same seed gives bitwise the same map.")
@click.option("--both-strands", is_flag=True, default=False, show_default=True,
              help="Map the mean of both strands' embeddings (embeddings_both_strands, written by nn-classification "
                   "--write-embeddings --both-strands), so a sequence and its reverse complement get the same point.")
@click.option("--index", "index", type=click.Path(path_type=Path, exists=True, dir_okay=False), default=None,
              help="Search through this embedding-index file (embedding-index output) instead of comparing every pair: each "
                   "sequence scans only the sequences of its --nprobe nearest lists. The index must have been built on the INPUT file "
                   "with the same --both-strands; checked before any work.")
@click.option("--nprobe", type=int, default=None,
              help="With --index: lists each sequence scans (1 to min(64, lists)); required with --index, since recall "
                   "against the exact search depends on it. At nprobe = lists the result is the exact search's.")
@click.option("--verbose/--quiet", "-v/-q", is_flag=True, default=True, show_default=True,
              help="Display the execution log.")
def embedding_map(input, output, k, epochs, seed, both_strands, index, nprobe, verbose):
    """Map the sequences of the INPUT embeddings file (nn-classification --write-embeddings output) onto two dimensions with
    UMAP on the GPU, and write each sequence's coordinates to the OUTPUT directory as <prefix>_embedding_map.{tsv,npz}.
    Not a module of the reference."""
    from . import embedding_map as module
    extra = {} if index is None and nprobe is None else {"index": index, "nprobe": nprobe}
    module.main(input, output, k, epochs, seed, verbose, both_strands=both_strands, **extra)


@cli.command(name="embedding-index", context_settings=CONTEXT_SETTINGS)
@click.argument("reference", type=click.Path(path_type=Path, exists=True, dir_okay=False))
@click.argument("output", type=click.Path(path_type=Path))
@click.option("--lists", type=int, default=None, show_default="ceil(4 sqrt(n))",
              help="Lists the sequences are split into by spherical k-means (1 to the number of sequences).")
@click.option("--iterations", type=int, default=20, show_default=True, help="k-means iterations (>= 0).")
@click.option("--seed", type=int, default=0, show_default=True,
              help="Seed of the training sample and the initial centroids: the same seed gives bitwise the same index.")
@click.option("--both-strands", is_flag=True, default=False, show_default=True,
              help="Index the mean of both strands' embeddings (embeddings_both_strands); searches with the index must then "
                   "use --both-strands too.")
@click.option("--verbose/--quiet", "-v/-q", is_flag=True, default=True, show_default=True,
              help="Display the execution log.")
def embedding_index(reference, output, lists, iterations, seed, both_strands, verbose):
    """Build an inverted-file index of the sequences of the REFERENCE embeddings file (nn-classification --write-embeddings
    output) for embedding-neighbours --index and embedding-map --index, and write it to the OUTPUT directory as
    <prefix>_embedding_index.npz. Runs in one process on one GPU (not a torchrun job). Not a module of the reference."""
    from . import embedding_index as module
    module.main(reference, output, lists, iterations, seed, verbose, both_strands=both_strands)


@cli.command(name="window-regions", context_settings=CONTEXT_SETTINGS)
@click.argument("windows", type=click.Path(path_type=Path, exists=True, dir_okay=False))
@click.argument("output", type=click.Path(path_type=Path))
@click.option("--mean-region-length", type=click.FloatRange(12000), required=True,
              help="Mean length, in bases, of a region of one class (>= 12,000): sets the switch rate between classes per "
                   "stride to stride / L. No default: no region length has been measured to suit this model.")
@click.option("--verbose/--quiet", "-v/-q", is_flag=True, default=True, show_default=True,
              help="Display the execution log.")
def window_regions(windows, output, mean_region_length, verbose):
    """Call class regions along each sequence of the WINDOWS file (nn-classification --write-window-scores output,
    <prefix>_nn_classification_windows.npz, a head's <prefix>_nn_classification_head_windows.npz, or their provirus_ twins)
    by an HMM decode of its window-score profile, and write them with coordinates and posterior confidence to the OUTPUT
    directory as <prefix>_nn_classification[_head]_regions.{tsv,npz}. Runs in one process on one GPU (not a torchrun job).
    Not a module of the reference."""
    from . import window_regions as module
    module.main(windows, output, mean_region_length, verbose)


@cli.command(name="aggregated-classification", context_settings=CONTEXT_SETTINGS)
@click.argument("input", type=click.Path(path_type=Path, exists=True))
@click.argument("output", type=click.Path(path_type=Path))
@click.option("--restart", is_flag=True, default=False, show_default=True,
              help="Overwrite existing intermediate files.")
@click.option("--verbose/--quiet", "-v/-q", is_flag=True, default=True, show_default=True,
              help="Display the execution log.")
def aggregated_classification(input, output, restart, verbose):
    """Aggregate the results of the marker-classification and nn-classification modules to classify the sequences in
    the INPUT file (FASTA format) and write the results to the OUTPUT directory (reference cli.py:776-803)."""
    from . import aggregated_classification as module
    module.main(input, output, restart, verbose)


if __name__ == "__main__":
    cli()
