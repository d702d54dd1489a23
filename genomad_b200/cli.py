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
def nn_classification(input, output, single_window, batch_size, restart, threads, verbose, cleanup, write_tfrecords):
    """Classify the sequences in the INPUT file (FASTA format) using the geNomad neural network and write
    the results to the OUTPUT directory."""
    import os
    from . import nn_classification as module
    if write_tfrecords:
        os.environ["GENOMAD_B200_TFRECORDS"] = "1"
    module.main(input, output, single_window, batch_size, restart, threads, verbose, cleanup)


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
