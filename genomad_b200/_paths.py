"""
Output path schema of the nn-classification module -- the on-disk half of the drop-in boundary.
Same file names as the reference's ``GenomadOutputs`` (reference genomad/_paths.py:188-236, and
:100-140 for the find-proviruses files this module only reads).
"""
from __future__ import annotations

from dataclasses import dataclass
from pathlib import Path


@dataclass(frozen=True)
class NNOutputs:
    prefix: str
    output_dir: Path

    def _nn(self, name: str) -> Path:
        return self.nn_classification_dir / f"{self.prefix}_{name}"

    @property
    def nn_classification_log(self) -> Path:
        return self.output_dir / f"{self.prefix}_nn_classification.log"

    @property
    def nn_classification_dir(self) -> Path:
        return self.output_dir / f"{self.prefix}_nn_classification"

    @property
    def nn_classification_execution_info(self) -> Path:
        return self._nn("nn_classification.json")

    @property
    def encoded_sequences_dir(self) -> Path:
        return self._nn("encoded_sequences")

    @property
    def seq_window_id_output(self) -> Path:
        return self.encoded_sequences_dir / f"{self.prefix}_seq_window_id.npz"

    @property
    def nn_classification_output(self) -> Path:
        return self._nn("nn_classification.tsv")

    @property
    def nn_classification_npz_output(self) -> Path:
        return self._nn("nn_classification.npz")

    @property
    def encoded_proviruses_dir(self) -> Path:
        return self._nn("encoded_proviruses")

    @property
    def provirus_window_id_output(self) -> Path:
        return self.encoded_proviruses_dir / f"{self.prefix}_provirus_window_id.npz"

    @property
    def provirus_nn_classification_output(self) -> Path:
        return self._nn("provirus_nn_classification.tsv")

    @property
    def provirus_nn_classification_npz_output(self) -> Path:
        return self._nn("provirus_nn_classification.npz")

    # ---- opt-in (--write-embeddings), not a reference output: per-contig mean encoder embeddings
    @property
    def nn_classification_embeddings_output(self) -> Path:
        return self._nn("nn_classification_embeddings.npz")

    @property
    def provirus_nn_classification_embeddings_output(self) -> Path:
        return self._nn("provirus_nn_classification_embeddings.npz")

    # ---- opt-in (--write-window-scores), not a reference output: class scores of every window, with its coordinates
    @property
    def nn_classification_windows_output(self) -> Path:
        return self._nn("nn_classification_windows.tsv")

    @property
    def nn_classification_windows_npz_output(self) -> Path:
        return self._nn("nn_classification_windows.npz")

    @property
    def provirus_nn_classification_windows_output(self) -> Path:
        return self._nn("provirus_nn_classification_windows.tsv")

    @property
    def provirus_nn_classification_windows_npz_output(self) -> Path:
        return self._nn("provirus_nn_classification_windows.npz")

    # ---- opt-in (--write-attributions), not a reference output: per-token input gradients of one class, per window
    @property
    def nn_classification_attributions_output(self) -> Path:
        return self._nn("nn_classification_attributions.npz")

    @property
    def provirus_nn_classification_attributions_output(self) -> Path:
        return self._nn("provirus_nn_classification_attributions.npz")

    # ---- opt-in (--both-strands), not a reference output: scores of the forward strand, the reverse strand and their mean
    @property
    def nn_classification_strands_output(self) -> Path:
        return self._nn("nn_classification_strands.tsv")

    @property
    def nn_classification_strands_npz_output(self) -> Path:
        return self._nn("nn_classification_strands.npz")

    @property
    def provirus_nn_classification_strands_output(self) -> Path:
        return self._nn("provirus_nn_classification_strands.tsv")

    @property
    def provirus_nn_classification_strands_npz_output(self) -> Path:
        return self._nn("provirus_nn_classification_strands.npz")

    # ---- opt-in (--head), not a reference output: scores of a user-trained classifier head
    @property
    def nn_classification_head_output(self) -> Path:
        return self._nn("nn_classification_head.tsv")

    @property
    def nn_classification_head_npz_output(self) -> Path:
        return self._nn("nn_classification_head.npz")

    @property
    def provirus_nn_classification_head_output(self) -> Path:
        return self._nn("provirus_nn_classification_head.tsv")

    @property
    def provirus_nn_classification_head_npz_output(self) -> Path:
        return self._nn("provirus_nn_classification_head.npz")

    # ---- opt-in (--head with --both-strands), not a reference output: the head's scores of each strand and their mean
    @property
    def nn_classification_head_strands_output(self) -> Path:
        return self._nn("nn_classification_head_strands.tsv")

    @property
    def nn_classification_head_strands_npz_output(self) -> Path:
        return self._nn("nn_classification_head_strands.npz")

    @property
    def provirus_nn_classification_head_strands_output(self) -> Path:
        return self._nn("provirus_nn_classification_head_strands.tsv")

    @property
    def provirus_nn_classification_head_strands_npz_output(self) -> Path:
        return self._nn("provirus_nn_classification_head_strands.npz")

    # ---- opt-in (--head with --write-window-scores), not a reference output: the head's scores of every window
    @property
    def nn_classification_head_windows_output(self) -> Path:
        return self._nn("nn_classification_head_windows.tsv")

    @property
    def nn_classification_head_windows_npz_output(self) -> Path:
        return self._nn("nn_classification_head_windows.npz")

    @property
    def provirus_nn_classification_head_windows_output(self) -> Path:
        return self._nn("provirus_nn_classification_head_windows.tsv")

    @property
    def provirus_nn_classification_head_windows_npz_output(self) -> Path:
        return self._nn("provirus_nn_classification_head_windows.npz")

    # ---- opt-in (--head with a head that carries a novelty model), not a reference output: distance to the head's classes
    @property
    def nn_classification_head_novelty_output(self) -> Path:
        return self._nn("nn_classification_head_novelty.tsv")

    @property
    def nn_classification_head_novelty_npz_output(self) -> Path:
        return self._nn("nn_classification_head_novelty.npz")

    @property
    def provirus_nn_classification_head_novelty_output(self) -> Path:
        return self._nn("provirus_nn_classification_head_novelty.tsv")

    @property
    def provirus_nn_classification_head_novelty_npz_output(self) -> Path:
        return self._nn("provirus_nn_classification_head_novelty.npz")

    # ---- opt-in (--write-head-attributions), not a reference output: per-token input gradients of one of the head's classes
    @property
    def nn_classification_head_attributions_output(self) -> Path:
        return self._nn("nn_classification_head_attributions.npz")

    @property
    def provirus_nn_classification_head_attributions_output(self) -> Path:
        return self._nn("provirus_nn_classification_head_attributions.npz")

    # ---- opt-in (--write-novelty-attributions, --write-window-novelty), not reference outputs: where and why a sequence is novel
    @property
    def nn_classification_head_novelty_attributions_output(self) -> Path:
        return self._nn("nn_classification_head_novelty_attributions.npz")

    @property
    def provirus_nn_classification_head_novelty_attributions_output(self) -> Path:
        return self._nn("provirus_nn_classification_head_novelty_attributions.npz")

    @property
    def nn_classification_head_novelty_windows_output(self) -> Path:
        return self._nn("nn_classification_head_novelty_windows.tsv")

    @property
    def nn_classification_head_novelty_windows_npz_output(self) -> Path:
        return self._nn("nn_classification_head_novelty_windows.npz")

    @property
    def provirus_nn_classification_head_novelty_windows_output(self) -> Path:
        return self._nn("provirus_nn_classification_head_novelty_windows.tsv")

    @property
    def provirus_nn_classification_head_novelty_windows_npz_output(self) -> Path:
        return self._nn("provirus_nn_classification_head_novelty_windows.npz")

    # ---- produced by find-proviruses, only read here (reference utils.py:280-297)
    @property
    def find_proviruses_dir(self) -> Path:
        return self.output_dir / f"{self.prefix}_find_proviruses"

    @property
    def find_proviruses_execution_info(self) -> Path:
        return self.find_proviruses_dir / f"{self.prefix}_find_proviruses.json"

    @property
    def find_proviruses_output(self) -> Path:
        return self.find_proviruses_dir / f"{self.prefix}_provirus.tsv"

    @property
    def find_proviruses_nucleotide_output(self) -> Path:
        return self.find_proviruses_dir / f"{self.prefix}_provirus.fna"

    @property
    def find_proviruses_proteins_output(self) -> Path:
        return self.find_proviruses_dir / f"{self.prefix}_provirus_proteins.faa"

    @property
    def find_proviruses_genes_output(self) -> Path:
        return self.find_proviruses_dir / f"{self.prefix}_provirus_genes.tsv"


@dataclass(frozen=True)
class AggregatedOutputs(NNOutputs):
    """
    What aggregated-classification reads (marker-classification's NPZ files, reference _paths.py:129-181) and writes
    (reference _paths.py:238-281), on top of the nn-classification files above.
    """

    def _mk(self, name: str) -> Path:
        return self.marker_classification_dir / f"{self.prefix}_{name}"

    def _agg(self, name: str) -> Path:
        return self.aggregated_classification_dir / f"{self.prefix}_{name}"

    # ---- produced by marker-classification, only read here
    @property
    def marker_classification_dir(self) -> Path:
        return self.output_dir / f"{self.prefix}_marker_classification"

    @property
    def marker_classification_execution_info(self) -> Path:
        return self._mk("marker_classification.json")

    @property
    def features_npz_output(self) -> Path:
        return self._mk("features.npz")

    @property
    def marker_classification_npz_output(self) -> Path:
        return self._mk("marker_classification.npz")

    @property
    def provirus_features_npz_output(self) -> Path:
        return self._mk("provirus_features.npz")

    @property
    def provirus_marker_classification_npz_output(self) -> Path:
        return self._mk("provirus_marker_classification.npz")

    # ---- written by aggregated-classification
    @property
    def aggregated_classification_log(self) -> Path:
        return self.output_dir / f"{self.prefix}_aggregated_classification.log"

    @property
    def aggregated_classification_dir(self) -> Path:
        return self.output_dir / f"{self.prefix}_aggregated_classification"

    @property
    def aggregated_classification_execution_info(self) -> Path:
        return self._agg("aggregated_classification.json")

    @property
    def aggregated_classification_output(self) -> Path:
        return self._agg("aggregated_classification.tsv")

    @property
    def aggregated_classification_npz_output(self) -> Path:
        return self._agg("aggregated_classification.npz")

    @property
    def provirus_aggregated_classification_output(self) -> Path:
        return self._agg("provirus_aggregated_classification.tsv")

    @property
    def provirus_aggregated_classification_npz_output(self) -> Path:
        return self._agg("provirus_aggregated_classification.npz")
