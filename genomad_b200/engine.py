"""
ctypes binding of libgnm.so (C ABI: include/gnm.h) and the ``Classifier`` object the host code uses.

This is the device-facing half of the drop-in: ``Classifier`` plays the role of the Keras model the
reference builds with ``neural_network.create_classifier()`` + ``load_weights`` and calls with
``predict(batch)`` (reference genomad/modules/nn_classification.py:309-317).  Tensors live in PyTorch
(device memory, streams); all arithmetic happens in the hand-written sm_90a kernels of libgnm.so.
There is no CPU or PyTorch fallback: if the library or an H100 is missing, construction fails.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path
from typing import Dict, List, NamedTuple, Optional, Tuple

import numpy as np

from . import weights as _weights

_PKG = Path(__file__).resolve().parent
_LIB_PATH = Path(os.environ["GENOMAD_B200_LIB"]) if os.environ.get("GENOMAD_B200_LIB") else _PKG / "libgnm.so"   # dev: A/B two builds
_lib = None

WINDOW = 6000
TOKENS = 5997
EMBED = 512                      # encoder output width (GNM_EMBED)


class GnmError(RuntimeError):
    pass


class _IglooW(C.Structure):
    _fields_ = [("w_mult", C.c_void_p), ("w_summer", C.c_void_p), ("w_bias", C.c_void_p),
                ("w_qk", C.c_void_p), ("w_v", C.c_void_p), ("patches", C.c_void_p)]


class _BnW(C.Structure):
    _fields_ = [("gamma", C.c_void_p), ("beta", C.c_void_p), ("moving_mean", C.c_void_p),
                ("moving_variance", C.c_void_p)]


class _Weights(C.Structure):
    _fields_ = [("conv1_kernel", C.c_void_p), ("conv1_bias", C.c_void_p),
                ("conv2_kernel", C.c_void_p), ("conv2_bias", C.c_void_p),
                ("conv3_kernel", C.c_void_p), ("conv3_bias", C.c_void_p),
                ("igloo", _IglooW * 2),
                ("dense0_kernel", C.c_void_p), ("dense0_bias", C.c_void_p), ("bn0", _BnW),
                ("dense1_kernel", C.c_void_p), ("dense1_bias", C.c_void_p), ("bn1", _BnW),
                ("dense2_kernel", C.c_void_p), ("dense2_bias", C.c_void_p)]


class _HeadW(C.Structure):
    _fields_ = [("n_classes", C.c_int), ("dense1_kernel", C.c_void_p), ("dense1_bias", C.c_void_p), ("bn1", _BnW),
                ("dense2_kernel", C.c_void_p), ("dense2_bias", C.c_void_p)]


EXPORTS = {
    # name: (restype, argtypes)
    "gnm_last_error": (C.c_char_p, []),
    "gnm_version": (C.c_char_p, []),
    "gnm_create": (C.c_int, [C.c_int, C.POINTER(_Weights), C.c_int, C.POINTER(C.c_void_p)]),
    "gnm_destroy": (C.c_int, [C.c_void_p]),
    "gnm_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_forward_ascii": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_forward_tokens": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_segment_mean": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_segment_sum": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_classify_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "gnm_check_status": (C.c_int, [C.c_void_p, C.c_void_p]),
    "gnm_contig_windows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64,
                                     C.c_void_p, C.POINTER(C.c_int64), C.c_void_p]),
    "gnm_contig_windows_stride": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                            C.c_int64, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p]),
    "gnm_contig_windows_rc": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                        C.c_int64, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p]),
    "gnm_gather_windows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_gather_windows_rc": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_forward_windows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_forward_windows_rc": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_embed_tokens": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_embed_ascii": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_embed_windows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_embed_windows_rc": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                       C.c_void_p]),
    "gnm_embed_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_segment_sum_rows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int]),
    "gnm_get_option": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_int)]),
    "gnm_kernel_launches": (C.c_longlong, [C.c_void_p]),
    "gnm_stage_times": (C.c_int, [C.c_void_p, C.POINTER(C.c_char_p), C.POINTER(C.c_float), C.POINTER(C.c_int)]),
    "gnm_debug_fetch": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_pack_patches": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.POINTER(C.c_int), C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.c_void_p]),
    "gnm_attr_create": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]),
    "gnm_attr_destroy": (C.c_int, [C.c_void_p]),
    "gnm_attr_bytes_per_window": (C.c_longlong, []),
    "gnm_attribute_ascii": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_attribute_windows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                        C.c_void_p, C.c_void_p]),
    "gnm_attribute_ig_ascii": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_attribute_ig_windows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                           C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_attribute_head_ascii": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_attribute_head_windows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                             C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_attribute_head_ig_ascii": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_attribute_head_ig_windows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                                C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_void_p]),
    "gnm_attribute_novelty_ascii": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_attribute_novelty_windows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_attribute_novelty_ig_ascii": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                                 C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_attribute_novelty_ig_windows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_void_p, C.c_void_p]),
    "gnm_neighbours_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64, C.c_int]),
    "gnm_embedding_neighbours": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "gnm_neighbours_merge": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]),
    "gnm_ivf_normalize": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "gnm_ivf_centroids": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_ivf_prepare": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_ivf_search_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64, C.c_void_p, C.c_int, C.c_int]),
    "gnm_ivf_search": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                 C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                 C.c_void_p]),
    "gnm_ivf_search_ranges_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64, C.c_void_p, C.c_int, C.c_int]),
    "gnm_ivf_search_ranges": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                        C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_size_t, C.c_void_p]),
    "gnm_cluster_block_probed": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_float, C.c_void_p, C.c_int, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "gnm_cluster_block_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "gnm_cluster_block": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                    C.c_void_p]),
    "gnm_map_membership": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p]),
    "gnm_map_pca_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "gnm_map_pca": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                              C.c_void_p]),
    "gnm_map_init_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "gnm_map_init": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t,
                               C.c_void_p]),
    "gnm_map_epochs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_void_p,
                                 C.c_void_p, C.c_void_p]),
    "gnm_window_regions_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "gnm_window_regions": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                     C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "gnm_head_create": (C.c_int, [C.c_void_p, C.POINTER(_HeadW), C.POINTER(C.c_void_p)]),
    "gnm_head_destroy": (C.c_int, [C.c_void_p]),
    "gnm_head_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_head_segment_mean": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_head_segment_sum": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_novelty_fit_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "gnm_novelty_fit": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.POINTER(C.c_double), C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                  C.c_void_p]),
    "gnm_head_set_novelty": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_head_novelty": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_head_train_create": (C.c_int, [C.c_int, C.POINTER(_HeadW), C.c_int, C.c_uint64, C.c_float, C.POINTER(C.c_void_p)]),
    "gnm_head_train_destroy": (C.c_int, [C.c_void_p]),
    "gnm_head_train_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                      C.c_void_p, C.c_void_p]),
    "gnm_head_train_read": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_longlong), C.c_void_p]),
    "gnm_head_train_fetch": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p]),
    "gnm_fasta_last_error": (C.c_char_p, []),
    "gnm_fasta_open": (C.c_int, [C.c_char_p, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "gnm_fasta_open_gz": (C.c_int, [C.c_char_p, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "gnm_fasta_release_before": (C.c_int, [C.c_void_p, C.c_int64]),
    "gnm_fasta_parse": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "gnm_fasta_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int), C.POINTER(C.c_int64),
                                 C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "gnm_fasta_export": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "gnm_fasta_export_windows": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int]),
    "gnm_fasta_free": (None, [C.c_void_p]),
    "gnm_fasta_windows_plan": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "gnm_fasta_windows_plan_rc": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "gnm_fasta_windows_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "gnm_fasta_windows_spans": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_fasta_windows_export": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int]),
    "gnm_fasta_windows_release_before": (C.c_int, [C.c_void_p, C.c_int64]),
    "gnm_fasta_windows_free": (None, [C.c_void_p]),
    "gnm_fasta_spans": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "gnm_tsv_last_error": (C.c_char_p, []),
    "gnm_write_window_tsv": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_int]),
    "gnm_write_window_tsv_cols": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "gnm_format_scores": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.POINTER(C.c_int64)]),
    "gnm_tfrecord_last_error": (C.c_char_p, []),
    "gnm_tfrecord_write": (C.c_int, [C.c_char_p, C.c_void_p, C.c_int64, C.c_int]),
    "gnm_tfrecord_read": (C.c_int, [C.c_char_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]),
    "gnm_crc32c": (C.c_uint32, [C.c_void_p, C.c_size_t]),
}


def load_library(path: Optional[Path] = None):
    """dlopen libgnm.so (built in-tree by ``python -m genomad_b200.build``) and declare every symbol."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = Path(path) if path else _LIB_PATH
    if not p.exists():
        raise GnmError(f"{p} not found: build it with `python -m genomad_b200.build` "
                       "(the CUDA extension is mandatory; there is no CPU fallback)")
    lib = C.CDLL(str(p))
    for name, (res, args) in EXPORTS.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if path is None:
        _lib = lib
    return lib


def _check(lib, rc: int):
    if rc != 0:
        raise GnmError(lib.gnm_last_error().decode(errors="replace"))


def _ptr(a: np.ndarray) -> int:
    return a.ctypes.data


NEIGHBOURS_MAX_K = 64
NEIGHBOURS_CHUNK = 1 << 18       # reference rows per gnm_embedding_neighbours call: 1 GB of TF32 halves, whatever the input size


def _neighbours_args(t, rows, name):
    assert rows.dtype == t.float32 and rows.dim() == 2 and rows.shape[1] == EMBED and rows.is_cuda, \
        f"{name}: float32 cuda tensor [n, {EMBED}] expected"
    return rows.contiguous()


def _neighbours_k(k) -> int:
    k = int(k)
    if not 1 <= k <= NEIGHBOURS_MAX_K:
        raise ValueError(f"k must be in [1, {NEIGHBOURS_MAX_K}], not {k}")
    return k


def embedding_neighbours(query, reference=None, k: int = 10, *, ref_index0: int = 0, self_index0: Optional[int] = None):
    """The k nearest reference rows of every query row in cosine similarity (gnm_embedding_neighbours, include/gnm.h).

    query float32 cuda [nq, 512]; reference float32 cuda [nr, 512] on the same device, or None for all-vs-all: the query rows
    are the reference and query i never returns itself.  Returns cuda tensors (sim float32 [nq, k], idx int64 [nq, k]), row q
    sorted by (similarity descending, index ascending) and padded with (-inf, -1) when fewer than k references qualify.
    Indices are ref_index0 + reference row; self_index0 (default: ref_index0 for all-vs-all, none otherwise) excludes global
    index self_index0 + q from query q's list.  The reference is searched NEIGHBOURS_CHUNK rows per call, the lists merged on
    the device (gnm_neighbours_merge): the result is bitwise that of one call over all rows."""
    import torch as t
    k = _neighbours_k(k)
    q = _neighbours_args(t, query, "query")
    ref = q if reference is None else _neighbours_args(t, reference, "reference")
    if ref.device != q.device:
        raise ValueError("query and reference must be on the same device")
    self0 = (ref_index0 if reference is None else -1) if self_index0 is None else int(self_index0)
    lib = load_library()
    nq, nr = q.shape[0], ref.shape[0]
    sim = t.empty((nq, k), dtype=t.float32, device=q.device)
    idx = t.empty((nq, k), dtype=t.int64, device=q.device)
    with t.cuda.device(q.device):
        stream = t.cuda.current_stream(q.device).cuda_stream
        work = t.empty(0, dtype=t.uint8, device=q.device)
        part = None
        for a in range(0, max(nr, 1), NEIGHBOURS_CHUNK):
            b = min(nr, a + NEIGHBOURS_CHUNK)
            need = int(lib.gnm_neighbours_workspace_bytes(nq, b - a, k))
            if need == 0 and nq:
                _check(lib, 1)
            if need > work.numel():
                work = t.empty(need, dtype=t.uint8, device=q.device)
            if a and part is None:
                part = (t.empty_like(sim), t.empty_like(idx))
            s_out, i_out = (sim, idx) if a == 0 else part
            _check(lib, lib.gnm_embedding_neighbours(q.data_ptr(), nq, ref[a:b].data_ptr() if b > a else None, b - a,
                                                     int(ref_index0) + a, self0, k, s_out.data_ptr(), i_out.data_ptr(),
                                                     work.data_ptr(), work.numel(), stream))
            if a:
                _check(lib, lib.gnm_neighbours_merge(sim.data_ptr(), idx.data_ptr(), s_out.data_ptr(), i_out.data_ptr(), nq, k,
                                                     stream))
    return sim, idx


def neighbours_merge(sim, idx, sim_b, idx_b):
    """Merge the neighbour lists (sim_b, idx_b) into (sim, idx) in place (cuda float32 / int64 [nq, k]; gnm_neighbours_merge)."""
    import torch as t
    assert sim.dtype == sim_b.dtype == t.float32 and idx.dtype == idx_b.dtype == t.int64 and sim.is_cuda
    assert sim.shape == idx.shape == sim_b.shape == idx_b.shape and sim.dim() == 2
    assert sim.is_contiguous() and idx.is_contiguous()
    sb, ib = sim_b.contiguous(), idx_b.contiguous()
    k = _neighbours_k(sim.shape[1])
    lib = load_library()
    with t.cuda.device(sim.device):
        _check(lib, lib.gnm_neighbours_merge(sim.data_ptr(), idx.data_ptr(), sb.data_ptr(), ib.data_ptr(), sim.shape[0], k,
                                             t.cuda.current_stream(sim.device).cuda_stream))
    return sim, idx


IVF_MAX_PROBE = 64
IVF_TRAIN_PER_LIST = 256         # training rows per list at most (the first 256 L rows of the hashed order)
IVF_QUERY_BYTES = 1 << 31        # per gnm_ivf_search call: the live (query, list) pairs' rows, halves and partial lists
IVF_REF_ROWS = NEIGHBOURS_CHUNK  # reference rows per gnm_ivf_search call: whole lists, or pieces of a longer list


class IvfIndex(NamedTuple):
    """An inverted-file index of n reference rows (cuda tensors; DESIGN.md, "Embedding index")."""
    centroids: "object"       # float32 [L, 512], unit rows (or zero)
    rows: "object"            # int64 [n]: the reference rows in (list, row) order
    offsets: "object"         # int64 [L + 1]: list l is rows[offsets[l]:offsets[l + 1]]


def ivf_default_lists(n: int) -> int:
    """ceil(4 sqrt(n)), at most n: the usual rule of thumb for the list count (Johnson, Douze & Jegou 2019)."""
    import math
    r = math.isqrt(16 * n)
    return min(n, r + (r * r < 16 * n))


def ivf_check(n: int, lists, iterations, seed) -> Tuple[int, int, int]:
    """(lists, iterations, seed) as ints, or ValueError: 1 <= lists <= n, iterations >= 0, 0 <= seed < 2^64."""
    lists, iterations, seed = int(lists), int(iterations), int(seed)
    if not 1 <= lists <= n:
        raise ValueError(f"lists must be in [1, {n:,}] (the reference rows), not {lists}")
    if iterations < 0:
        raise ValueError(f"iterations must be >= 0, not {iterations}")
    if not 0 <= seed < 1 << 64:
        raise ValueError(f"seed must be in [0, 2^64), not {seed}")
    return lists, iterations, seed


def ivf_nprobe(nprobe, lists: int) -> int:
    nprobe = int(nprobe)
    if not 1 <= nprobe <= min(IVF_MAX_PROBE, lists):
        raise ValueError(f"nprobe must be in [1, {min(IVF_MAX_PROBE, lists)}] (at most 64 and the index's {lists:,} lists), "
                         f"not {nprobe}")
    return nprobe


def ivf_training_rows(n: int, lists: int, seed: int, device):
    """The training rows, int64 cuda [min(n, 256 lists)]: rows in the order of (mix32(key ^ row), row), key = synth._keys(seed)[0]."""
    import torch as t
    from .synth import _keys, _mix32
    r = t.arange(n, dtype=t.int64, device=device)
    h = _mix32((r & 0xFFFFFFFF) ^ _keys(seed)[0])
    return t.sort(h, stable=True).indices[: min(n, IVF_TRAIN_PER_LIST * lists)]


def ivf_normalize(rows):
    """rows / their fp64 norm, rounded to fp32 (gnm_ivf_normalize): float32 cuda [n, 512]."""
    import torch as t
    x = _neighbours_args(t, rows, "rows")
    out = t.empty_like(x)
    lib = load_library()
    with t.cuda.device(x.device):
        _check(lib, lib.gnm_ivf_normalize(x.data_ptr(), x.shape[0], out.data_ptr(), _stream(t, x.device)))
    return out


def ivf_assign(rows, centroids):
    """Each row's k = 1 centroid under s, the row as the query: (similarity float32 [n], list int64 [n]), cuda.  The queries
    are searched NEIGHBOURS_CHUNK rows per call; each row's result does not depend on the others."""
    import torch as t
    x = _neighbours_args(t, rows, "rows")
    sims, lists = [], []
    for a in range(0, x.shape[0], NEIGHBOURS_CHUNK):
        s, i = embedding_neighbours(x[a:a + NEIGHBOURS_CHUNK], centroids, 1)
        sims.append(s[:, 0]); lists.append(i[:, 0])
    if not sims:
        return t.empty(0, dtype=t.float32, device=x.device), t.empty(0, dtype=t.int64, device=x.device)
    return t.cat(sims), t.cat(lists)


def ivf_layout(assign, lists: int):
    """(rows int64 [n], offsets int64 [lists + 1]): the row indices stably sorted by their list."""
    import torch as t
    order = t.sort(assign, stable=True).indices
    offsets = t.zeros(lists + 1, dtype=t.int64, device=assign.device)
    offsets[1:] = t.cumsum(t.bincount(assign, minlength=lists), 0)
    return order, offsets


def ivf_centroids(xhat, assign, lists: int):
    """The normalised sums of each list's normalised rows, summed in row order after a stable sort by list (gnm_ivf_centroids):
    float32 cuda [lists, 512]; an empty list gives the zero row."""
    import torch as t
    order, offsets = ivf_layout(assign, lists)
    xs = xhat.index_select(0, order).contiguous()
    off32 = offsets.to(t.int32)
    sums = t.empty((lists, EMBED), dtype=t.float32, device=xhat.device)
    cent = t.empty_like(sums)
    lib = load_library()
    with t.cuda.device(xhat.device):
        _check(lib, lib.gnm_ivf_centroids(xs.data_ptr(), off32.data_ptr(), lists, sums.data_ptr(), cent.data_ptr(),
                                          _stream(t, xhat.device)))
    return cent


def ivf_reseed(centroids, xhat, train, best, assign):
    """Empty lists, in ascending order, each take the normalised training row not yet taken with the lowest best similarity
    (ties: the lowest row).  train: the training rows' indices; best, assign: their k = 1 search.  Returns (centroids, the
    reseeded lists int64)."""
    import torch as t
    lists = centroids.shape[0]
    empty = t.nonzero(t.bincount(assign, minlength=lists) == 0).flatten()
    if empty.numel() == 0:
        return centroids, empty
    by_row = t.sort(train, stable=True).indices
    order = by_row[t.sort(best[by_row], stable=True).indices]
    out = centroids.clone()
    out[empty] = xhat[order[: empty.numel()]]
    return out, empty


def ivf_build(rows, lists: int, iterations: int = 20, seed: int = 0) -> IvfIndex:
    """Spherical k-means of rows (float32 cuda [n, 512]) into `lists` lists, and the layout of every row (include/gnm.h,
    "Embedding index").  The same rows, lists, iterations and seed give a bitwise identical index."""
    import torch as t
    x = _neighbours_args(t, rows, "rows")
    lists, iterations, seed = ivf_check(x.shape[0], lists, iterations, seed)
    train = ivf_training_rows(x.shape[0], lists, seed, x.device)
    xhat = ivf_normalize(x.index_select(0, train).contiguous())
    cent = xhat[:lists].clone()
    for _ in range(iterations):
        best, assign = ivf_assign(xhat, cent)
        cent = ivf_centroids(xhat, assign, lists)
        cent, _ = ivf_reseed(cent, xhat, train, best, assign)
    _, assign = ivf_assign(x, cent)
    order, offsets = ivf_layout(assign, lists)
    return IvfIndex(cent, order, offsets)


def ivf_chunks(offsets, l_begin: int, l_end: int, max_rows: int = NEIGHBOURS_CHUNK):
    """The reference chunks of lists [l_begin, l_end) for gnm_ivf_search: (l0, l1, a, b) = lists l0 .. l1 - 1, index rows
    [a, b); consecutive whole lists up to max_rows rows, a longer list alone in pieces of max_rows rows."""
    off = [int(v) for v in offsets]
    out, l = [], l_begin
    while l < l_end:
        if off[l + 1] - off[l] > max_rows:
            out += [(l, l + 1, a, min(a + max_rows, off[l + 1])) for a in range(off[l], off[l + 1], max_rows)]
            l += 1
            continue
        e = l + 1
        while e < l_end and off[e + 1] - off[l] <= max_rows:
            e += 1
        out.append((l, e, off[l], off[e]))
        l = e
    return out


def ivf_probes(query, centroids, nprobe: int):
    """Each query's nprobe nearest centroids under the total order: int32 cuda [nq, nprobe] (embedding_neighbours, NEIGHBOURS_CHUNK
    queries per call, so its workspace does not grow with the queries; each query's result does not depend on the others)."""
    import torch as t
    out = t.empty((query.shape[0], nprobe), dtype=t.int32, device=query.device)
    for a in range(0, query.shape[0], NEIGHBOURS_CHUNK):
        out[a:a + NEIGHBOURS_CHUNK] = embedding_neighbours(query[a:a + NEIGHBOURS_CHUNK], centroids, nprobe)[1]
    return out


def ivf_check_probes(probes, nq: int, nprobe: int, lists: int):
    """ValueError unless probes is an integer cuda tensor [nq, nprobe] of list ids in [0, lists), distinct within each row."""
    import torch as t
    if tuple(probes.shape) != (nq, nprobe) or probes.dtype not in (t.int32, t.int64):
        raise ValueError(f"probes must be integers [{nq}, {nprobe}], not {probes.dtype} {list(probes.shape)}")
    if nq and nprobe and (int(probes.min()) < 0 or int(probes.max()) >= lists):
        raise ValueError(f"probes must be list ids in [0, {lists})")
    if nq and nprobe > 1 and bool((t.diff(t.sort(probes, 1).values, dim=1) == 0).any()):
        raise ValueError("probes must be distinct within each row")
    return probes.to(t.int32)


def ivf_search(query, reference, index: IvfIndex, k: int, nprobe: int, *, ref_index0: int = 0,
               self_index0: Optional[int] = None, lists: Optional[Tuple[int, int]] = None, probes=None,
               reference_shard: bool = False):
    """The k nearest rows of every query among the rows of its nprobe nearest lists (gnm_ivf_search), shaped and ordered like
    embedding_neighbours: (sim float32 [nq, k], idx int64 [nq, k]), cuda, padded with (-inf, -1).  reference None: all-vs-all
    over the query rows (self_index0 defaults to ref_index0).  Indices are ref_index0 + reference row.  lists=(l0, l1) searches
    only those lists of the probes (a rank's share); reference_shard: `reference` then holds only the rows of those lists, in
    list order (index.rows[offsets[l0]:offsets[l1]]).  probes: precomputed ivf_probes, checked.  At nprobe = L the result is
    bitwise embedding_neighbours.

    Each reference chunk (ivf_chunks) is prepared once (gnm_ivf_prepare); its live pairs, the (query, list) pairs whose list
    lies in the chunk, go to gnm_ivf_search in query ranges of at most about IVF_QUERY_BYTES of workspace."""
    import torch as t
    k = _neighbours_k(k)
    q = _neighbours_args(t, query, "query")
    ref = q if reference is None else _neighbours_args(t, reference, "reference")
    self0 = (ref_index0 if reference is None else -1) if self_index0 is None else int(self_index0)
    L = index.centroids.shape[0]
    nprobe = ivf_nprobe(nprobe, L)
    dev = q.device
    nq = q.shape[0]
    off = index.offsets.cpu().numpy().astype(np.int64)
    l0_, l1_ = (0, L) if lists is None else (int(lists[0]), int(lists[1]))
    if not 0 <= l0_ <= l1_ <= L:
        raise ValueError(f"lists must be a range inside [0, {L}], not {lists}")
    base = int(off[l0_]) if reference_shard else 0
    want = int(off[l1_] - off[l0_]) if reference_shard else index.rows.shape[0]
    if ref.shape[0] != want:
        raise ValueError(f"the index holds {want:,} rows here, the reference {ref.shape[0]:,}")
    probes = ivf_probes(q, index.centroids.to(dev), nprobe) if probes is None else ivf_check_probes(probes.to(dev), nq, nprobe, L)
    rows = index.rows.to(dev)
    sim = t.full((nq, k), float("-inf"), dtype=t.float32, device=dev)
    idx = t.full((nq, k), -1, dtype=t.int64, device=dev)
    s_out, i_out = t.empty_like(sim), t.empty_like(idx)
    lib = load_library()
    work = t.empty(0, dtype=t.uint8, device=dev)
    halves = t.empty(0, dtype=t.float32, device=dev)
    with t.cuda.device(dev):
        stream = _stream(t, dev)
        for l0, l1, a, b in ivf_chunks(off, l0_, l1_, IVF_REF_ROWS):
            lp = probes.to(t.int64) - l0
            live = (lp >= 0) & (lp < l1 - l0)
            cum = t.cumsum(live.sum(1), 0)
            total = int(cum[-1]) if nq else 0
            if total == 0 or b == a:
                continue
            ridx = rows[a:b]
            r = ref[a - base:b - base] if reference_shard else ref.index_select(0, ridx).contiguous()
            if halves.numel() < 2 * (b - a) * EMBED:
                halves = t.empty(2 * (b - a) * EMBED, dtype=t.float32, device=dev)
            hi, lo = halves[: (b - a) * EMBED], halves[(b - a) * EMBED: 2 * (b - a) * EMBED]
            _check(lib, lib.gnm_ivf_prepare(r.data_ptr(), b - a, hi.data_ptr(), lo.data_ptr(), stream))
            gidx = (ridx + int(ref_index0)).contiguous()
            h_off = np.ascontiguousarray(np.clip(off[l0:l1 + 1], a, b) - a, dtype=np.int64)
            qi, ji = t.nonzero(live, as_tuple=True)                                # query-major: pairs in query order
            pq, pl = qi.to(t.int32), lp[qi, ji].to(t.int32)
            # pairs per call: a range of whole queries of at most pc + nprobe pairs
            pc = max(total, nprobe)                               # >= nprobe: every range holds a whole query
            while pc > nprobe and lib.gnm_ivf_search_workspace_bytes(pc + nprobe, b - a, _ptr(h_off), l1 - l0, k) > IVF_QUERY_BYTES:
                pc = max(nprobe, (pc + 1) // 2)
            cuts = t.searchsorted(cum, t.arange(pc, total, pc, device=dev), right=True).tolist()
            bounds = [0] + cuts + [nq]
            pstart = [0] + cum[t.tensor(bounds[1:], device=dev) - 1].tolist()
            for c in range(len(bounds) - 1):
                qa, qb, pa, pb = bounds[c], bounds[c + 1], int(pstart[c]), int(pstart[c + 1])
                if pb == pa:
                    continue
                need = int(lib.gnm_ivf_search_workspace_bytes(pb - pa, b - a, _ptr(h_off), l1 - l0, k))
                if need == 0:
                    _check(lib, 1)
                if need > work.numel():
                    work = t.empty(need, dtype=t.uint8, device=dev)
                cq = (pq[pa:pb] - qa).contiguous()
                cl = pl[pa:pb].contiguous()
                _check(lib, lib.gnm_ivf_search(q[qa:qb].data_ptr(), qb - qa, cq.data_ptr(), cl.data_ptr(), pb - pa, hi.data_ptr(),
                                               lo.data_ptr(), b - a, _ptr(h_off), l1 - l0, gidx.data_ptr(),
                                               self0 + qa if self0 >= 0 else -1, k, s_out.data_ptr(), i_out.data_ptr(),
                                               work.data_ptr(), need, stream))
                _check(lib, lib.gnm_neighbours_merge(sim[qa:qb].data_ptr(), idx[qa:qb].data_ptr(), s_out.data_ptr(),
                                                     i_out.data_ptr(), qb - qa, k, stream))
    return sim, idx


CLUSTER_MAX_BLOCK = 8192         # rows per gnm_cluster_block call: a threshold mask of 8 MB
CLUSTER_SLOT_BYTES = 2 * EMBED * 4 + 8   # per representative slot: its TF32 halves and its global row index


def cluster_threshold(min_similarity) -> float:
    """The clustering threshold rounded once to fp32 (as a Python float); ValueError outside (0, 1]."""
    t = float(np.float32(min_similarity))
    if not 0.0 < t <= 1.0:
        raise ValueError(f"min_similarity must be in (0, 1], not {min_similarity}")
    return t


def cluster_block(rows, covered, min_similarity):
    """One block step of greedy clustering (gnm_cluster_block, include/gnm.h).

    rows float32 cuda [n, 512], n <= CLUSTER_MAX_BLOCK: the block's rows in file order; covered uint8 cuda [n]: nonzero where an
    earlier block's representative has similarity >= min_similarity with the row (embedding_neighbours at k = 1, the row as the
    query).  Returns the block's new representatives as block-local row indices, int64 cuda, ascending: row j is one iff it is not
    covered and s(j, i) < min_similarity for every new representative i < j, each comparison bitwise that of the search's
    similarity.  Waits for the device to read the count."""
    import torch as t
    x = _neighbours_args(t, rows, "rows")
    n = x.shape[0]
    if n > CLUSTER_MAX_BLOCK:
        raise ValueError(f"a block holds at most {CLUSTER_MAX_BLOCK} rows, not {n}")
    assert covered.dtype == t.uint8 and covered.shape == (n,) and covered.device == x.device, \
        "covered: uint8 tensor [n] on the rows' device expected"
    thr = cluster_threshold(min_similarity)
    cov = covered.contiguous()
    lib = load_library()
    with t.cuda.device(x.device):
        need = int(lib.gnm_cluster_block_workspace_bytes(n))
        if need == 0 and n:
            _check(lib, 1)
        work = t.empty(need, dtype=t.uint8, device=x.device)
        reps = t.empty(max(n, 1), dtype=t.int32, device=x.device)
        count = t.empty(1, dtype=t.int32, device=x.device)
        _check(lib, lib.gnm_cluster_block(x.data_ptr(), n, cov.data_ptr(), thr, reps.data_ptr(), count.data_ptr(),
                                          work.data_ptr(), need, t.cuda.current_stream(x.device).cuda_stream))
        m = int(count.item())
    return reps[:m].long()


def cluster_block_probed(rows, covered, min_similarity, probes, home):
    """cluster_block, comparing row j only with the block's representatives i whose home list is one of j's probes
    (gnm_cluster_block_probed): probes int32 cuda [n, nprobe] (the block rows' ivf_probes), home int32 cuda [n] (the list the
    index places each block row in)."""
    import torch as t
    x = _neighbours_args(t, rows, "rows")
    n = x.shape[0]
    if n > CLUSTER_MAX_BLOCK:
        raise ValueError(f"a block holds at most {CLUSTER_MAX_BLOCK} rows, not {n}")
    assert covered.dtype == t.uint8 and covered.shape == (n,) and covered.device == x.device, \
        "covered: uint8 tensor [n] on the rows' device expected"
    assert probes.dtype == t.int32 and probes.dim() == 2 and probes.shape[0] == n and probes.device == x.device, \
        "probes: int32 tensor [n, nprobe] on the rows' device expected"
    assert home.dtype == t.int32 and home.shape == (n,) and home.device == x.device, "home: int32 tensor [n] expected"
    thr = cluster_threshold(min_similarity)
    cov, pr, hm = covered.contiguous(), probes.contiguous(), home.contiguous()
    lib = load_library()
    with t.cuda.device(x.device):
        need = int(lib.gnm_cluster_block_workspace_bytes(n))
        if need == 0 and n:
            _check(lib, 1)
        work = t.empty(need, dtype=t.uint8, device=x.device)
        reps = t.empty(max(n, 1), dtype=t.int32, device=x.device)
        count = t.empty(1, dtype=t.int32, device=x.device)
        _check(lib, lib.gnm_cluster_block_probed(x.data_ptr(), n, cov.data_ptr(), thr, pr.data_ptr(), pr.shape[1], hm.data_ptr(),
                                                 reps.data_ptr(), count.data_ptr(), work.data_ptr(), need,
                                                 _stream(t, x.device)))
        m = int(count.item())
    return reps[:m].long()


class ClusterSlots(NamedTuple):
    """The slots of the representatives of lists [l0, l0 + m) of an index (gnm_ivf_search_ranges, include/gnm.h): list l0 + j owns
    slots [offsets[j], offsets[j + 1]) and holds the representatives in slots [offsets[j], end[j]), in ascending row order."""
    l0: int
    offsets: np.ndarray       # host int64 [m + 1] from 0: the capacities, the index's list sizes
    end: "object"             # cuda int64 [m]
    hi: "object"              # cuda float32 [slots, 512]: the representatives' TF32 halves (gnm_ivf_prepare)
    lo: "object"
    index: "object"           # cuda int64 [slots]: their global rows


def cluster_slots(offsets, l0: int, l1: int, device) -> ClusterSlots:
    """Empty slots for the representatives of lists [l0, l1) of an index with these offsets (int64 [L + 1])."""
    import torch as t
    off = np.asarray(offsets, np.int64)[l0:l1 + 1]
    off = np.ascontiguousarray(off - off[0])
    cap = int(off[-1])
    return ClusterSlots(int(l0), off, t.from_numpy(off[:-1].copy()).to(device),
                        t.empty((cap, EMBED), dtype=t.float32, device=device), t.empty((cap, EMBED), dtype=t.float32, device=device),
                        t.empty(cap, dtype=t.int64, device=device))


def cluster_slots_counts(slots: ClusterSlots):
    """The representatives each list holds: int64 cuda [m]."""
    import torch as t
    return slots.end - t.from_numpy(slots.offsets[:-1]).to(slots.end.device)


def cluster_slots_append(slots: ClusterSlots, rows, gidx, home) -> None:
    """Append new representatives: rows float32 cuda [r, 512] with global rows gidx (int64 [r], ascending, after every row the
    slots hold) and home lists home (int [r]); those of other lists are skipped.  Only the new slots are written."""
    import torch as t
    m = slots.end.shape[0]
    j = home.to(t.int64) - slots.l0
    own = t.nonzero((j >= 0) & (j < m)).flatten()
    if own.numel() == 0:
        return
    j = j[own]
    order = t.sort(j, stable=True).indices
    js = j[order]
    rank = t.arange(js.numel(), device=js.device) - t.searchsorted(js, js)
    pos = slots.end[js] + rank
    x = _neighbours_args(t, rows.index_select(0, own[order]), "rows")
    hi, lo = t.empty_like(x), t.empty_like(x)
    lib = load_library()
    with t.cuda.device(x.device):
        _check(lib, lib.gnm_ivf_prepare(x.data_ptr(), x.shape[0], hi.data_ptr(), lo.data_ptr(), _stream(t, x.device)))
    slots.hi.index_copy_(0, pos, hi)
    slots.lo.index_copy_(0, pos, lo)
    slots.index.index_copy_(0, pos, gidx[own[order]])
    slots.end.add_(t.bincount(j, minlength=m))


def cluster_slots_search(slots: ClusterSlots, query, probes):
    """Each query's nearest representative among those of its probed lists that these slots hold (gnm_ivf_search_ranges at
    k = 1): (sim float32 [nq, 1], idx int64 [nq, 1] global rows), cuda, (-inf, -1) where there is none.  probes: int32 cuda
    [nq, nprobe]; lists outside the slots' are skipped.  The queries go in ranges of at most about IVF_QUERY_BYTES of workspace,
    sized from the capacities, so no call waits for the device."""
    import torch as t
    q = _neighbours_args(t, query, "query")
    nq, nprobe = probes.shape
    dev = q.device
    m = slots.end.shape[0]
    sim = t.full((nq, 1), float("-inf"), dtype=t.float32, device=dev)
    idx = t.full((nq, 1), -1, dtype=t.int64, device=dev)
    if nq == 0 or slots.offsets[-1] == 0:
        return sim, idx
    lib = load_library()
    off = slots.offsets
    ws = lambda pairs: int(lib.gnm_ivf_search_ranges_workspace_bytes(pairs, int(off[-1]), _ptr(off), m, 1))
    qc = nq
    while qc > 1 and ws(qc * nprobe) > IVF_QUERY_BYTES:
        qc = (qc + 1) // 2
    need = ws(min(qc, nq) * nprobe)
    if need == 0:
        _check(lib, 1)
    work = t.empty(need, dtype=t.uint8, device=dev)
    pl_all = (probes.to(t.int32) - slots.l0).contiguous()
    with t.cuda.device(dev):
        stream = _stream(t, dev)
        for a in range(0, nq, qc):
            b = min(nq, a + qc)
            pq = t.arange(b - a, dtype=t.int32, device=dev).repeat_interleave(nprobe)
            pl = pl_all[a:b].reshape(-1)
            _check(lib, lib.gnm_ivf_search_ranges(q[a:b].data_ptr(), b - a, pq.data_ptr(), pl.data_ptr(), pq.numel(),
                                                  slots.hi.data_ptr(), slots.lo.data_ptr(), int(off[-1]), _ptr(off),
                                                  slots.end.data_ptr(), m, slots.index.data_ptr(), 1, sim[a:b].data_ptr(),
                                                  idx[a:b].data_ptr(), work.data_ptr(), need, stream))
    return sim, idx


MAP_A = 1.57694346               # 1 / (1 + a x^2b) least-squares fitted to umap-learn's curve at min_dist = 0.1, spread = 1
MAP_B = 0.89506088


def map_default_epochs(n: int) -> int:
    """umap-learn's default: 500 layout epochs for at most 10,000 rows, else 200."""
    return 500 if n <= 10000 else 200


def map_check(n: int, k, epochs, seed) -> Tuple[int, int, int]:
    """(k, epochs, seed) as ints, or ValueError: 1 <= k <= 64, k < n, epochs >= 1 (None: map_default_epochs), 0 <= seed < 2^64."""
    k = int(k)
    if not 1 <= k <= NEIGHBOURS_MAX_K:
        raise ValueError(f"k must be in [1, {NEIGHBOURS_MAX_K}], not {k}")
    if k >= n:
        raise ValueError(f"k must be smaller than the number of sequences ({n:,}), not {k}")
    epochs = map_default_epochs(n) if epochs is None else int(epochs)
    if epochs < 1:
        raise ValueError(f"epochs must be >= 1, not {epochs}")
    seed = int(seed)
    if not 0 <= seed < 1 << 64:
        raise ValueError(f"seed must be in [0, 2^64), not {seed}")
    return k, epochs, seed


class MapMembership(NamedTuple):
    """Result of map_membership (cuda tensors, fp64; gnm_map_membership)."""
    mean_d: "object"          # [1]
    rho: "object"             # [n]
    sigma: "object"           # [n]
    w: "object"               # [n, k] directed memberships
    union: "object"           # [n, k] fuzzy union at the entry that emits the pair, -1 elsewhere


class MapGraph(NamedTuple):
    """The layout graph (cuda tensors): both directions of every kept edge, each row sorted by column."""
    row_ptr: "object"         # int64 [n + 1]
    col: "object"             # int32 [nnz]
    weight: "object"          # float64 [nnz]
    eps: "object"             # float64 [nnz]: epochs per sample, max w / w


def _stream(t, dev):
    return t.cuda.current_stream(dev).cuda_stream


def map_membership(sim, idx) -> MapMembership:
    """Step 2 of the map: memberships and their fuzzy union from the all-vs-all lists of embedding_neighbours (sim float32
    cuda [n, k], idx int64 cuda [n, k])."""
    import torch as t
    assert sim.dtype == t.float32 and idx.dtype == t.int64 and sim.is_cuda and sim.shape == idx.shape and sim.dim() == 2
    n, k = sim.shape
    sim, idx = sim.contiguous(), idx.contiguous()
    f64 = dict(dtype=t.float64, device=sim.device)
    out = MapMembership(t.empty(1, **f64), t.empty(n, **f64), t.empty(n, **f64), t.empty((n, k), **f64), t.empty((n, k), **f64))
    lib = load_library()
    with t.cuda.device(sim.device):
        _check(lib, lib.gnm_map_membership(sim.data_ptr(), idx.data_ptr(), n, k, *(a.data_ptr() for a in out),
                                           _stream(t, sim.device)))
    return out


def map_graph(union, idx, epochs: int) -> MapGraph:
    """Step 3: drop union weights below max w / epochs, as umap-learn does, and store both directions of the rest as CSR rows
    sorted by column, with the epochs per sample.  Integer bookkeeping with torch's stable sort and cumsum, on the device."""
    import torch as t
    n, k = union.shape
    u = union.reshape(-1)
    max_w = u.max()
    e = t.nonzero(u >= max_w / epochs).flatten()
    i, j, w = e // k, idx.reshape(-1)[e], u[e]
    rows, cols, ws = t.cat([i, j]), t.cat([j, i]), t.cat([w, w])
    order = t.sort(rows * n + cols, stable=True).indices
    rows, cols, ws = rows[order], cols[order], ws[order]
    row_ptr = t.zeros(n + 1, dtype=t.int64, device=union.device)
    row_ptr[1:] = t.cumsum(t.bincount(rows, minlength=n), 0)
    return MapGraph(row_ptr, cols.to(t.int32).contiguous(), ws.contiguous(), (max_w / ws).contiguous())


def map_pca(rows):
    """Step 4a: (xhat float32 [n, 512], center float64 [512], S float64 [512, 512], V float64 [2, 512]) of rows (float32 cuda
    [n, 512]): the fp64-normalised rows, their mean and covariance, and its top-2 eigenvectors (gnm_map_pca)."""
    import torch as t
    x = _neighbours_args(t, rows, "rows")
    n = x.shape[0]
    lib = load_library()
    dev = x.device
    xhat = t.empty_like(x)
    center = t.empty(EMBED, dtype=t.float64, device=dev)
    S = t.empty((EMBED, EMBED), dtype=t.float64, device=dev)
    V = t.empty((2, EMBED), dtype=t.float64, device=dev)
    with t.cuda.device(dev):
        need = int(lib.gnm_map_pca_workspace_bytes(n))
        if need == 0:
            _check(lib, 1)
        work = t.empty(need, dtype=t.uint8, device=dev)
        _check(lib, lib.gnm_map_pca(x.data_ptr(), n, xhat.data_ptr(), center.data_ptr(), S.data_ptr(), V.data_ptr(),
                                    work.data_ptr(), need, _stream(t, dev)))
    return xhat, center, S, V


def map_init(xhat, center, V, seed: int, *, projection: bool = False):
    """Step 4b: the initial layout float32 cuda [n, 2] (gnm_map_init).  projection=True also returns the fp64 projections
    [n, 2] it was scaled from."""
    import torch as t
    n = xhat.shape[0]
    dev = xhat.device
    lib = load_library()
    Y = t.empty((n, 2), dtype=t.float32, device=dev)
    with t.cuda.device(dev):
        need = int(lib.gnm_map_init_workspace_bytes(n))
        if need == 0:
            _check(lib, 1)
        work = t.empty(need, dtype=t.uint8, device=dev)
        _check(lib, lib.gnm_map_init(xhat.contiguous().data_ptr(), n, center.contiguous().data_ptr(), V.contiguous().data_ptr(),
                                     int(seed), Y.data_ptr(), work.data_ptr(), need, _stream(t, dev)))
        proj = work[: n * 16].view(t.float64).reshape(n, 2).clone() if projection else None
    return (Y, proj) if projection else Y


def map_epochs(graph: MapGraph, Y, epochs: int, seed: int, e_begin: int = 0, e_end: Optional[int] = None):
    """Step 5: layout epochs e_begin .. e_end - 1 (default: all) of `epochs` from Y (float32 cuda [n, 2]); returns a new tensor
    (gnm_map_epochs)."""
    import torch as t
    n = Y.shape[0]
    e_end = epochs if e_end is None else int(e_end)
    out = Y.contiguous().clone()
    tmp = t.empty_like(out)
    lib = load_library()
    with t.cuda.device(Y.device):
        _check(lib, lib.gnm_map_epochs(graph.row_ptr.data_ptr(), graph.col.data_ptr(), graph.eps.data_ptr(), n, int(epochs),
                                       int(e_begin), e_end, int(seed), out.data_ptr(), tmp.data_ptr(), _stream(t, Y.device)))
    return out


def map_layout(rows, sim, idx, epochs: int, seed: int):
    """Steps 2-5 from the rows and their all-vs-all neighbour lists: the map, float32 cuda [n, 2]."""
    m = map_membership(sim, idx)
    graph = map_graph(m.union, idx, epochs)
    xhat, center, _, V = map_pca(rows)
    Y = map_init(xhat, center, V, seed)
    return map_epochs(graph, Y, epochs, seed)


def embedding_map(rows, k: int = 15, epochs: Optional[int] = None, seed: int = 0):
    """A 2-D UMAP layout of rows (float32 cuda [n, 512]) on one GPU: the all-vs-all k-nearest-neighbour lists
    (embedding_neighbours), then map_layout.  Returns float32 cuda [n, 2].  DESIGN.md, "Embedding map"."""
    import torch as t
    x = _neighbours_args(t, rows, "rows")
    k, epochs, seed = map_check(x.shape[0], k, epochs, seed)
    sim, idx = embedding_neighbours(x, None, k)
    return map_layout(x, sim, idx, epochs, seed)


def both_strands(forward, reverse):
    """A contig's strand-averaged scores or embedding: (forward + reverse) * 0.5 in fp32, for float32 numpy arrays or torch
    tensors of the same shape (the per-contig outputs of the forward and the reverse strand).  fp32 addition commutes, so a
    contig and its reverse complement get bitwise the same result."""
    if isinstance(forward, np.ndarray):
        f, r = np.asarray(forward, np.float32), np.asarray(reverse, np.float32)
        return (f + r) * np.float32(0.5)
    return (forward + reverse) * 0.5


class WindowScores(NamedTuple):
    """Result of Classifier.window_scores and Head.window_scores (cuda tensors)."""
    probs: "object"           # float32 [W, 3] (chromosome, plasmid, virus); Head.window_scores: [W, C]
    contig: "object"          # int32 [W], index of the window's contig
    start: "object"           # int64 [W], first byte in the contig (0-based, before stripping n/N)
    length: "object"          # int32 [W], bytes of sequence (1..6000; the rest of the window is 'N' padding)
    offsets: "object"         # int32 [n_contigs + 1], CSR: the windows of contig c are [offsets[c], offsets[c+1])


class WindowRegions(NamedTuple):
    """Result of window_regions (cuda tensors); R regions in window order."""
    posterior: "object"          # float32 [W, C], forward-backward posterior of every class at every window
    state: "object"              # int32 [W], the Viterbi path
    region_contig: "object"      # int32 [R]
    region_start: "object"       # int64 [R], 0-based, in the contig's bytes as given (before stripping n/N)
    region_end: "object"         # int64 [R], exclusive
    region_class: "object"       # int32 [R]
    region_windows: "object"     # int32 [R]
    region_posterior: "object"   # float32 [R], mean posterior of the region's class over its windows
    region_scores: "object"      # float32 [R, C], mean window score of every class


REGIONS_MIN_LENGTH = 12000       # mean region length L >= 2 * 6000, so the switch rate s / L is at most 0.5 at every stride
REGIONS_WORK_BYTES = 1 << 30     # workspace per gnm_window_regions call; a call takes whole sequences (at least one)


def regions_mean_length(mean_region_length) -> float:
    """L as a float; ValueError below REGIONS_MIN_LENGTH or not finite."""
    L = float(mean_region_length)
    if not (np.isfinite(L) and L >= REGIONS_MIN_LENGTH):
        raise ValueError(f"mean_region_length must be a finite number >= {REGIONS_MIN_LENGTH}, not {mean_region_length}")
    return L


def window_regions(ws: "WindowScores", stride: int, mean_region_length, *, work_bytes: int = REGIONS_WORK_BYTES) -> "WindowRegions":
    """Class regions along each sequence from its window-score profile (gnm_window_regions, include/gnm.h; DESIGN.md, "Window
    regions"): the Viterbi path and forward-backward posteriors of a C-state HMM over the windows, and the maximal runs of the
    path as regions.

    ws: Classifier.window_scores or Head.window_scores output as it is (C = ws.probs.shape[1], 2..32); stride: the stride it
    was computed at (1..6000); mean_region_length: L >= 12000 bases.  The windows are checked on the device first (finite
    scores; within a sequence, starts increasing by positive multiples of the stride) and decoded in calls of whole sequences
    whose workspace fits work_bytes (a longer sequence gets a call of its own).  A sequence's results depend only on its own
    windows, so they are bitwise the same whatever the chunking or the other sequences."""
    import torch as t
    stride = int(stride)
    if not 1 <= stride <= WINDOW:
        raise ValueError(f"stride must be in [1, {WINDOW}], not {stride}")
    L = regions_mean_length(mean_region_length)
    probs, contig, start, length, offsets = ws
    if probs.dim() != 2 or not 2 <= probs.shape[1] <= 32:
        raise ValueError(f"scores must be [W, C] with 2 <= C <= 32, not {list(probs.shape)}")
    W, C_ = probs.shape
    dev = probs.device
    assert probs.is_cuda and probs.dtype == t.float32, "probs: float32 cuda tensor expected"
    assert contig.shape == (W,) and start.shape == (W,) and length.shape == (W,), "contig, start, length: [W] expected"
    probs = probs.contiguous()
    contig = contig.to(device=dev, dtype=t.int32).contiguous()
    start = start.to(device=dev, dtype=t.int64).contiguous()
    length = length.to(device=dev, dtype=t.int32).contiguous()
    offsets = offsets.to(device=dev, dtype=t.int32).contiguous()
    offs = offsets.cpu().numpy().astype(np.int64)
    if offs.ndim != 1 or offs.size < 1 or offs[0] != 0 or offs[-1] != W or (np.diff(offs) < 0).any():
        raise ValueError(f"offsets must be a non-decreasing CSR from 0 to {W}")
    if W:
        same = contig[1:] == contig[:-1]
        d = start[1:] - start[:-1]
        bad = t.stack([~t.isfinite(probs).all(), (same & ((d <= 0) | (d % stride != 0))).any(), (length < 1).any(),
                       (contig != t.repeat_interleave(t.arange(offs.size - 1, dtype=t.int32, device=dev),
                                                      offsets[1:] - offsets[:-1], output_size=W)).any()]).cpu().numpy()
        for flag, msg in zip(bad, ("scores are not all finite",
                                   f"window starts do not increase by positive multiples of the stride {stride} within a sequence",
                                   "a window length is < 1", "contig does not match offsets")):
            if flag:
                raise ValueError(msg)
    posterior = t.empty((W, C_), dtype=t.float32, device=dev)
    state = t.empty(W, dtype=t.int32, device=dev)
    first = t.zeros(W, dtype=t.uint8, device=dev)
    r_start = t.empty(W, dtype=t.int64, device=dev)
    r_end = t.empty(W, dtype=t.int64, device=dev)
    r_windows = t.empty(W, dtype=t.int32, device=dev)
    r_post = t.empty(W, dtype=t.float32, device=dev)
    r_scores = t.empty((W, C_), dtype=t.float32, device=dev)
    lib = load_library()
    max_windows = max(1, (int(work_bytes) - 768) // (8 * C_ + 6))      # gnm_window_regions_workspace_bytes, include/gnm.h
    with t.cuda.device(dev):
        stream = t.cuda.current_stream(dev).cuda_stream
        work = t.empty(0, dtype=t.uint8, device=dev)
        n_seqs, a = offs.size - 1, 0
        while a < n_seqs:
            # the longest run of whole sequences from a whose windows fit, at least one sequence
            b = max(a + 1, int(np.searchsorted(offs, offs[a] + max_windows, side="right")) - 1)
            b = min(b, n_seqs)
            w0, nw = int(offs[a]), int(offs[b] - offs[a])
            if nw:
                need = int(lib.gnm_window_regions_workspace_bytes(nw, C_))
                if need == 0:
                    _check(lib, 1)
                if need > work.numel():
                    work = t.empty(need, dtype=t.uint8, device=dev)
                _check(lib, lib.gnm_window_regions(
                    probs[w0:].data_ptr(), nw, C_, offsets[a:].data_ptr(), b - a, start[w0:].data_ptr(),
                    length[w0:].data_ptr(), stride, L, posterior[w0:].data_ptr(), state[w0:].data_ptr(), first[w0:].data_ptr(),
                    r_start[w0:].data_ptr(), r_end[w0:].data_ptr(), r_windows[w0:].data_ptr(), r_post[w0:].data_ptr(),
                    r_scores[w0:].data_ptr(), work.data_ptr(), work.numel(), stream))
            a = b
    rows = t.nonzero(first).flatten()
    return WindowRegions(posterior, state, contig[rows], r_start[rows], r_end[rows], state[rows], r_windows[rows], r_post[rows],
                         r_scores[rows])


class Attributions(NamedTuple):
    """Result of Classifier.attribute_contigs (cuda tensors); the windows are those of window_scores at stride 6000."""
    probs: "object"           # float32 [W, 3]
    contig: "object"          # int32 [W]
    start: "object"           # int64 [W], first byte in the contig (0-based, before stripping n/N)
    length: "object"          # int32 [W]
    offsets: "object"         # int32 [n_contigs + 1], CSR
    attr: "object"            # float32 [W, 5997]: d log p_target / d one-hot token, token t = bases t .. t+3 of the window
    logp: "object" = None     # integrated gradients only: float32 [W, 2], log p_target(window), log p_target(baseline)
                              # (novelty: D_target(window), D_target(baseline))
    head_probs: "object" = None   # Head.attribute_contigs / integrated_gradients_contigs: float32 [W, C], the head's scores
                                  # (novelty: the window's distances to every class)
    target: "object" = None   # Head.attribute_novelty_contigs / integrated_gradients_novelty_contigs: int32 [W], each window's
                              # target, its sequence's nearest class


CLASSES = ("chromosome", "plasmid", "virus")
ATTR_MAX_BATCH = 256             # windows per attribution chunk (attribution context, ~21 MB per window)
IG_BASELINES = ("zero", "N")     # GNM_IG_BASELINE_ZERO, GNM_IG_BASELINE_N
IG_STEPS = 64                    # default integrated-gradients steps: the smallest m of the fp64 convergence study with every
                                 # completeness gap below 1 on the unsharpened weights (profiles/integrated_gradients_h100.md)


def ig_baseline_index(baseline) -> int:
    """"zero" / "N" (or 0 / 1) -> GNM_IG_BASELINE_*."""
    if isinstance(baseline, str):
        if baseline not in IG_BASELINES:
            raise ValueError(f"baseline must be one of {IG_BASELINES}, not {baseline!r}")
        return IG_BASELINES.index(baseline)
    b = int(baseline)
    if b not in (0, 1):
        raise ValueError(f"baseline must be 0 (zero) or 1 (N), not {b}")
    return b


def class_index(target) -> int:
    """0 / 1 / 2 or "chromosome" / "plasmid" / "virus" -> class index."""
    if isinstance(target, str):
        if target not in CLASSES:
            raise ValueError(f"target must be one of {CLASSES}, not {target!r}")
        return CLASSES.index(target)
    t = int(target)
    if t not in (0, 1, 2):
        raise ValueError(f"target must be 0, 1 or 2, not {t}")
    return t


class Classifier:
    """
    The IGLOO1D classifier on one H100.

    weights : dict from genomad_b200.weights.load_weights() (short names -> numpy arrays in Keras layouts)
    device  : CUDA device index
    max_batch : windows per internal step (workspace ~10 MB per window)
    """

    def __init__(self, weights: Optional[Dict[str, np.ndarray]] = None, device: int = 0, max_batch: int = 1024):
        import torch
        if not torch.cuda.is_available():
            raise GnmError("no CUDA device visible: genomad_b200 runs on H100 (sm_90a) only, there is no CPU fallback")
        self._torch = torch
        self.lib = load_library()
        self.device = int(device)
        self.max_batch = int(max_batch)
        if weights is None:
            weights = _weights.load_weights()
        self._w = {k: np.ascontiguousarray(v) for k, v in weights.items()}   # keep host arrays alive during create
        cw = _weights.to_c_struct(self._w, _Weights, _IglooW, _BnW)
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):
            rc = self.lib.gnm_create(self.device, C.byref(cw), self.max_batch, C.byref(self._h))
        if rc != 0:
            msg = self.lib.gnm_last_error().decode(errors="replace")
            if self._h:
                self.lib.gnm_destroy(self._h)
                self._h = C.c_void_p()
            raise GnmError(msg)

    # ------------------------------------------------------------------ lifecycle
    def close(self):
        if getattr(self, "_attr", None):
            self.lib.gnm_attr_destroy(self._attr)
            self._attr = None
        if getattr(self, "_h", None):
            self.lib.gnm_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ helpers
    def _stream(self) -> int:
        return self._torch.cuda.current_stream(self.device).cuda_stream

    def _dev(self):
        return self._torch.device("cuda", self.device)

    def set_option(self, name: str, value: int):
        _check(self.lib, self.lib.gnm_set_option(self._h, name.encode(), int(value)))

    def get_option(self, name: str) -> int:
        v = C.c_int()
        _check(self.lib, self.lib.gnm_get_option(self._h, name.encode(), C.byref(v)))
        return v.value

    @property
    def kernel_launches(self) -> int:
        return int(self.lib.gnm_kernel_launches(self._h))

    # ------------------------------------------------------------------ device-tensor API
    def encode(self, ascii_windows):
        """uint8 cuda tensor [n, 6000] -> uint16 tokens [n, 5997] (torch.uint16)."""
        t = self._torch
        a = ascii_windows.contiguous()
        assert a.dtype == t.uint8 and a.dim() == 2 and a.shape[1] == WINDOW and a.is_cuda
        out = t.empty((a.shape[0], TOKENS), dtype=t.uint16, device=a.device)
        _check(self.lib, self.lib.gnm_encode(self._h, a.data_ptr(), a.shape[0], out.data_ptr(), self._stream()))
        return out

    def predict_ascii(self, ascii_windows, out=None):
        """uint8 cuda tensor [n, 6000] -> float32 probabilities [n, 3] (chromosome, plasmid, virus)."""
        t = self._torch
        a = ascii_windows.contiguous()
        assert a.dtype == t.uint8 and a.dim() == 2 and a.shape[1] == WINDOW and a.is_cuda
        if out is None:
            out = t.empty((a.shape[0], 3), dtype=t.float32, device=a.device)
        _check(self.lib, self.lib.gnm_forward_ascii(self._h, a.data_ptr(), a.shape[0], out.data_ptr(), self._stream()))
        return out

    def predict_tokens(self, tokens, out=None):
        """uint16 cuda tensor [n, 5997] -> float32 probabilities [n, 3]; the analogue of nn_model.predict(batch).  Any uint16 is
        valid: as in tf.one_hot(x, 257), a token above 256 contributes nothing."""
        t = self._torch
        k = tokens.contiguous()
        assert k.dtype == t.uint16 and k.dim() == 2 and k.shape[1] == TOKENS and k.is_cuda
        if out is None:
            out = t.empty((k.shape[0], 3), dtype=t.float32, device=k.device)
        _check(self.lib, self.lib.gnm_forward_tokens(self._h, k.data_ptr(), k.shape[0], out.data_ptr(), self._stream()))
        return out

    def segment_mean(self, probs, offsets):
        """probs float32 cuda [W,3], offsets int32 cuda [n_contigs+1] -> float32 [n_contigs,3]."""
        t = self._torch
        assert probs.dtype == t.float32 and offsets.dtype == t.int32 and probs.is_cuda and offsets.is_cuda
        n = offsets.numel() - 1
        out = t.empty((n, 3), dtype=t.float32, device=probs.device)
        _check(self.lib, self.lib.gnm_segment_mean(self._h, probs.contiguous().data_ptr(), offsets.contiguous().data_ptr(),
                                                   n, out.data_ptr(), self._stream()))
        return out

    def segment_sum(self, probs, offsets):
        """-> float32 [n_contigs,4] = (sum p0, sum p1, sum p2, window count): the cross-GPU partial."""
        t = self._torch
        n = offsets.numel() - 1
        out = t.empty((n, 4), dtype=t.float32, device=probs.device)
        _check(self.lib, self.lib.gnm_segment_sum(self._h, probs.contiguous().data_ptr(), offsets.contiguous().data_ptr(),
                                                  n, out.data_ptr(), self._stream()))
        return out

    # ------------------------------------------------------------------ encoder embeddings
    def _embed_out(self, n: int, device):
        t = self._torch
        return (t.empty((n, 3), dtype=t.float32, device=device), t.empty((n, EMBED), dtype=t.float32, device=device))

    def embed_tokens(self, tokens):
        """uint16 cuda [n, 5997] -> (probabilities float32 [n, 3], encoder embeddings float32 [n, 512]) (gnm_embed_tokens)."""
        t = self._torch
        k = tokens.contiguous()
        assert k.dtype == t.uint16 and k.dim() == 2 and k.shape[1] == TOKENS and k.is_cuda
        probs, emb = self._embed_out(k.shape[0], k.device)
        _check(self.lib, self.lib.gnm_embed_tokens(self._h, k.data_ptr(), k.shape[0], probs.data_ptr(), emb.data_ptr(),
                                                   self._stream()))
        return probs, emb

    def embed_ascii(self, ascii_windows):
        """uint8 cuda [n, 6000] -> (probabilities [n, 3], embeddings [n, 512]), both float32 on the device (gnm_embed_ascii)."""
        t = self._torch
        a = ascii_windows.contiguous()
        assert a.dtype == t.uint8 and a.dim() == 2 and a.shape[1] == WINDOW and a.is_cuda
        probs, emb = self._embed_out(a.shape[0], a.device)
        _check(self.lib, self.lib.gnm_embed_ascii(self._h, a.data_ptr(), a.shape[0], probs.data_ptr(), emb.data_ptr(),
                                                  self._stream()))
        return probs, emb

    def embed_windows(self, seq_u8, win_start, win_len, reverse: bool = False):
        """Windows straight from the sequence buffer (see predict_windows) -> (probabilities [W, 3], embeddings [W, 512])."""
        t = self._torch
        start, length = win_start.contiguous(), win_len.contiguous()
        assert start.dtype == t.int64 and length.dtype == t.int32 and start.numel() == length.numel()
        probs, emb = self._embed_out(start.numel(), seq_u8.device)
        fn = self.lib.gnm_embed_windows_rc if reverse else self.lib.gnm_embed_windows
        _check(self.lib, fn(self._h, seq_u8.data_ptr(), start.data_ptr(), length.data_ptr(), start.numel(), probs.data_ptr(),
                            emb.data_ptr(), self._stream()))
        return probs, emb

    def embed_host_into(self, ascii_ptr: int, n: int, probs_ptr: int, d_embed_ptr: int):
        """Raw-pointer gnm_embed_host: host windows -> host probabilities (probs_ptr may be 0) + device embeddings [n, 512]."""
        with self._torch.cuda.device(self.device):
            _check(self.lib, self.lib.gnm_embed_host(self._h, ascii_ptr, n, probs_ptr or None, d_embed_ptr))

    def segment_sum_rows(self, rows, offsets, carry=None):
        """rows float32 cuda [R, 512], offsets int32 cuda [k + 1] (offsets[0] = 0) -> (sums float32 [k, 512], carry [512]).
        Plain fp32 running sums in row order; `carry` (a previous call's) seeds segment 0 and the returned carry is the running
        sum of segment k-1, so chained calls over consecutive row blocks give the bits of one call."""
        t = self._torch
        assert rows.dtype == t.float32 and offsets.dtype == t.int32 and rows.is_cuda and offsets.is_cuda
        assert rows.dim() == 2 and rows.shape[1] == EMBED
        rows, offs = rows.contiguous(), offsets.contiguous()
        k = offs.numel() - 1
        sums = t.empty((k, EMBED), dtype=t.float32, device=rows.device)
        if carry is not None:
            assert carry.dtype == t.float32 and carry.numel() == EMBED and carry.is_cuda
            carry = carry.contiguous()
        out_carry = t.zeros(EMBED, dtype=t.float32, device=rows.device) if carry is None else carry.clone()
        if k == 0:
            return sums, out_carry
        rows_ptr = rows.data_ptr() if rows.numel() else sums.data_ptr()      # no rows: any aligned buffer, nothing reads it
        _check(self.lib, self.lib.gnm_segment_sum_rows(self._h, rows_ptr, offs.data_ptr(), k,
                                                       carry.data_ptr() if carry is not None else None, sums.data_ptr(),
                                                       out_carry.data_ptr(), self._stream()))
        return sums, out_carry

    # ------------------------------------------------------------------ contigs in memory -> windows on the device
    def contig_buffers(self, seqs):
        """Contigs -> (uint8 cuda [total_bytes], int64 cuda [n_contigs + 1] offsets), one host-to-device copy each.
        `seqs` is a list of str / bytes (str is UTF-8 encoded, i.e. the bytes the FASTA reader would see) or a
        (uint8 tensor or array, int64 offsets) pair on the host or on CUDA."""
        t = self._torch
        dev = self._dev()
        if isinstance(seqs, tuple) and len(seqs) == 2 and not isinstance(seqs[0], (str, bytes, bytearray)):
            seq = t.as_tensor(seqs[0]).to(device=dev, dtype=t.uint8).reshape(-1)
            offs = t.as_tensor(seqs[1]).to(device=dev, dtype=t.int64).reshape(-1)
        else:
            parts = [s.encode() if isinstance(s, str) else bytes(s) for s in seqs]
            offs_h = np.zeros(len(parts) + 1, dtype=np.int64)
            np.cumsum([len(p) for p in parts], out=offs_h[1:])
            seq = t.from_numpy(np.frombuffer(b"".join(parts), dtype=np.uint8).copy()).to(dev)
            offs = t.from_numpy(offs_h).to(dev)
        if seq.numel() == 0:
            seq = t.zeros(16, dtype=t.uint8, device=dev)          # all contigs empty: the library still wants a buffer
        return seq.contiguous(), offs.contiguous()

    def contig_windows(self, seq_u8, seq_offsets_i64, single_window: bool = False, stride: int = WINDOW,
                       reverse: bool = False):
        """Plan the windows of contigs on the device: uint8 cuda [total_bytes] + int64 cuda offsets [n_contigs + 1] ->
        (win_start int64 [W] absolute byte offsets, win_len int32 [W], win_offsets int32 [n_contigs + 1]).
        stride 6000: the reference's windows (gnm_contig_windows); any other stride in [1, 6000]: a window every `stride` nt of
        the whole contig (gnm_contig_windows_stride; not with single_window).  reverse: the same windows of each contig's
        reverse complement (gnm_contig_windows_rc); start / length then name each window's forward segment, laid from the
        stripped end."""
        t = self._torch
        assert seq_u8.dtype == t.uint8 and seq_offsets_i64.dtype == t.int64 and seq_u8.is_cuda and seq_offsets_i64.is_cuda
        stride = int(stride)
        if not 1 <= stride <= WINDOW:
            raise ValueError(f"stride must be in [1, {WINDOW}], not {stride}")
        if single_window and stride != WINDOW:
            raise ValueError("single_window plans the reference's windows only (stride 6000)")
        seq, offs = seq_u8.contiguous(), seq_offsets_i64.contiguous()
        n = offs.numel() - 1
        assert n >= 0
        cap = n + seq.numel() // stride                                   # always enough (gnm.h)
        start = t.empty(cap, dtype=t.int64, device=seq.device)
        length = t.empty(cap, dtype=t.int32, device=seq.device)
        woff = t.empty(n + 1, dtype=t.int32, device=seq.device)
        nw = C.c_int64()
        if reverse:
            rc = self.lib.gnm_contig_windows_rc(self._h, seq.data_ptr(), offs.data_ptr(), n, int(bool(single_window)), stride,
                                                start.data_ptr(), length.data_ptr(), cap, woff.data_ptr(), C.byref(nw),
                                                self._stream())
        elif stride == WINDOW:
            rc = self.lib.gnm_contig_windows(self._h, seq.data_ptr(), offs.data_ptr(), n, int(bool(single_window)),
                                             start.data_ptr(), length.data_ptr(), cap, woff.data_ptr(), C.byref(nw),
                                             self._stream())
        else:
            rc = self.lib.gnm_contig_windows_stride(self._h, seq.data_ptr(), offs.data_ptr(), n, stride, start.data_ptr(),
                                                    length.data_ptr(), cap, woff.data_ptr(), C.byref(nw), self._stream())
        _check(self.lib, rc)
        return start[:nw.value], length[:nw.value], woff

    def gather_windows(self, seq_u8, win_start, win_len, reverse: bool = False):
        """Kept windows -> uint8 cuda [W, 6000], upper-cased and N-padded (gnm_gather_windows).  reverse: each window's
        segment reverse-complemented first (gnm_gather_windows_rc, for the windows of contig_windows(..., reverse=True))."""
        t = self._torch
        start, length = win_start.contiguous(), win_len.contiguous()
        assert start.dtype == t.int64 and length.dtype == t.int32 and start.numel() == length.numel()
        out = t.empty((start.numel(), WINDOW), dtype=t.uint8, device=seq_u8.device)
        fn = self.lib.gnm_gather_windows_rc if reverse else self.lib.gnm_gather_windows
        _check(self.lib, fn(self._h, seq_u8.data_ptr(), start.data_ptr(), length.data_ptr(), start.numel(), out.data_ptr(),
                            self._stream()))
        return out

    def predict_windows(self, seq_u8, win_start, win_len, out=None, reverse: bool = False):
        """Per-window probabilities float32 [W, 3] straight from the sequence buffer (gnm_forward_windows; reverse:
        gnm_forward_windows_rc, the reverse-complement gather of gather_windows(..., reverse=True))."""
        t = self._torch
        start, length = win_start.contiguous(), win_len.contiguous()
        assert start.dtype == t.int64 and length.dtype == t.int32 and start.numel() == length.numel()
        if out is None:
            out = t.empty((start.numel(), 3), dtype=t.float32, device=seq_u8.device)
        fn = self.lib.gnm_forward_windows_rc if reverse else self.lib.gnm_forward_windows
        _check(self.lib, fn(self._h, seq_u8.data_ptr(), start.data_ptr(), length.data_ptr(), start.numel(), out.data_ptr(),
                            self._stream()))
        return out

    def classify_contigs(self, seqs, single_window: bool = False, return_window_probs: bool = False,
                         return_embeddings: bool = False, strand: str = "forward"):
        """Contigs in, one score triple per contig out -- what the reference module computes per contig
        (nn_classification.py:65-75, 316-320), with windowing on the GPU.

        seqs: list of str / bytes, or a (uint8 tensor, int64 offsets) pair on the host or on CUDA (see contig_buffers).
        Returns cuda tensors (means float32 [n_contigs, 3], window counts int32 [n_contigs]), then, if asked, the per-window
        probabilities float32 [W, 3], then, if asked, the per-contig mean encoder embeddings float32 [n_contigs, 512]
        (segment_sum_rows / count in fp32).  A contig that is empty after stripping n/N has count 0, mean (0, 0, 0) and a zero
        embedding; the reference drops such contigs, so drop those rows to mirror its outputs.

        strand "reverse" scores each contig's reverse complement instead (the reference's Sequence.rc(), windowed as the
        reference windows any contig): bitwise the forward call on the reverse-complemented contigs.  both_strands() combines
        the two calls' outputs."""
        t = self._torch
        if strand not in ("forward", "reverse"):
            raise ValueError(f"strand must be 'forward' or 'reverse', not {strand!r}")
        rev = strand == "reverse"
        seq, offs = self.contig_buffers(seqs)
        start, length, woff = self.contig_windows(seq, offs, single_window, reverse=rev)
        if return_embeddings:
            probs, emb = self.embed_windows(seq, start, length, reverse=rev)
        else:
            probs = self.predict_windows(seq, start, length, reverse=rev)
        if probs.numel():
            means = self.segment_mean(probs, woff)
        else:                 # no contig has a window (an empty probs tensor has no buffer to hand to gnm_segment_mean)
            means = t.zeros((woff.numel() - 1, 3), dtype=t.float32, device=seq.device)
        counts = woff[1:] - woff[:-1]
        out = (means, counts, probs) if return_window_probs else (means, counts)
        if return_embeddings:
            sums, _ = self.segment_sum_rows(emb, woff)
            out = out + (sums / counts.clamp(min=1).to(t.float32)[:, None],)
        return out

    def window_scores(self, seqs, stride: int = WINDOW) -> "WindowScores":
        """Class scores of every window of every contig, with the window's place in its contig: the per-window probabilities
        the reference averages away (nn_classification.py:316-320), and at stride < 6000 a window every `stride` nt
        (overlapping windows, each classified by the unchanged model) for a finer profile along the contig.

        seqs: as for classify_contigs.  Returns cuda tensors WindowScores(probs float32 [W, 3], contig int32 [W],
        start int64 [W] (0-based, in the contig's bytes as given, i.e. before stripping n/N), length int32 [W] (bytes of
        sequence, padding excluded), offsets int32 [n_contigs + 1] (CSR: the windows of contig c)).  At stride 6000 these are
        the windows, and bitwise the probabilities, of classify_contigs(..., return_window_probs=True)."""
        t = self._torch
        seq, offs = self.contig_buffers(seqs)
        start, length, woff = self.contig_windows(seq, offs, stride=stride)
        n = woff.numel() - 1
        counts = (woff[1:] - woff[:-1]).to(t.int64)
        contig = t.repeat_interleave(t.arange(n, dtype=t.int32, device=seq.device), counts)
        probs = (self.predict_windows(seq, start, length) if start.numel()
                 else t.zeros((0, 3), dtype=t.float32, device=seq.device))
        rel = start - offs[:-1].index_select(0, contig.to(t.int64)) if start.numel() else start
        return WindowScores(probs, contig, rel, length, woff)

    # ------------------------------------------------------------------ attributions
    def _attr_ctx(self, max_batch: Optional[int] = None):
        """The attribution workspace, created on first use (ATTR_MAX_BATCH windows per chunk, capped at the handle's max_batch)."""
        if getattr(self, "_attr", None):
            return self._attr
        mb = min(int(max_batch or ATTR_MAX_BATCH), self.max_batch)
        ctx = C.c_void_p()
        with self._torch.cuda.device(self.device):
            rc = self.lib.gnm_attr_create(self._h, mb, C.byref(ctx))
        if rc != 0:
            msg = self.lib.gnm_last_error().decode(errors="replace")
            if ctx:
                self.lib.gnm_attr_destroy(ctx)
            raise GnmError(msg)
        self._attr = ctx
        self.attr_max_batch = mb
        return ctx

    def attribute_ascii(self, ascii_windows, target):
        """uint8 cuda [n, 6000], target class (0 / 1 / 2 or its name) -> (probabilities float32 [n, 3], attributions float32
        [n, 5997]): attr[i, t] = d log p_target / d x[t, tok[t]] for the one-hot tokens x of window i (gnm_attribute_ascii).
        The probabilities are bitwise those of predict_ascii."""
        t = self._torch
        a = ascii_windows.contiguous()
        assert a.dtype == t.uint8 and a.dim() == 2 and a.shape[1] == WINDOW and a.is_cuda
        c = class_index(target)
        probs = t.empty((a.shape[0], 3), dtype=t.float32, device=a.device)
        attr = t.empty((a.shape[0], TOKENS), dtype=t.float32, device=a.device)
        if a.shape[0]:
            _check(self.lib, self.lib.gnm_attribute_ascii(self._h, self._attr_ctx(), a.data_ptr(), a.shape[0], c,
                                                          probs.data_ptr(), attr.data_ptr(), self._stream()))
        return probs, attr

    def attribute_windows(self, seq_u8, win_start, win_len, target):
        """Planned windows of a sequence buffer (see predict_windows) -> (probabilities [W, 3], attributions [W, 5997])."""
        t = self._torch
        start, length = win_start.contiguous(), win_len.contiguous()
        assert start.dtype == t.int64 and length.dtype == t.int32 and start.numel() == length.numel()
        c = class_index(target)
        n = start.numel()
        probs = t.empty((n, 3), dtype=t.float32, device=seq_u8.device)
        attr = t.empty((n, TOKENS), dtype=t.float32, device=seq_u8.device)
        if n:
            _check(self.lib, self.lib.gnm_attribute_windows(self._h, self._attr_ctx(), seq_u8.data_ptr(), start.data_ptr(),
                                                            length.data_ptr(), n, c, probs.data_ptr(), attr.data_ptr(),
                                                            self._stream()))
        return probs, attr

    def attribute_contigs(self, seqs, target, single_window: bool = False) -> "Attributions":
        """Attributions of the reference's windows of every contig (the windows whose mean is the contig score), with their
        place in the contig.  seqs: as for classify_contigs.  Token t of a window covers its bases t .. t+3; sum or spread the
        values over those bases for a per-base track."""
        t = self._torch
        seq, offs = self.contig_buffers(seqs)
        start, length, woff = self.contig_windows(seq, offs, single_window)
        n = woff.numel() - 1
        counts = (woff[1:] - woff[:-1]).to(t.int64)
        contig = t.repeat_interleave(t.arange(n, dtype=t.int32, device=seq.device), counts)
        probs, attr = self.attribute_windows(seq, start, length, target)
        rel = start - offs[:-1].index_select(0, contig.to(t.int64)) if start.numel() else start
        return Attributions(probs, contig, rel, length, woff, attr)

    def _ig_args(self, steps, baseline):
        steps = int(steps)
        if steps < 1:
            raise ValueError(f"steps must be >= 1, not {steps}")
        return steps, ig_baseline_index(baseline)

    def integrated_gradients_ascii(self, ascii_windows, target, steps: int = IG_STEPS, baseline="zero"):
        """uint8 cuda [n, 6000], target class -> (probabilities float32 [n, 3], logp float32 [n, 2], attributions float32
        [n, 5997]) by integrated gradients (gnm_attribute_ig_ascii): attr[i, t] = (1/m) sum_k g_k[t, tok[t]] (baseline "zero",
        all-zero one-hot rows) or (1/m) sum_k (g_k[t, tok[t]] - g_k[t, 0]) (baseline "N", the all-N window), g_k the input
        gradient of log p_target at x' + (k + 1/2)/m (x - x'), m = steps.  The attributions add up to about
        logp[:, 0] - logp[:, 1] = log p_target(x) - log p_target(x').  The probabilities are bitwise those of predict_ascii.
        steps is capped by the attribution context's max_batch (ATTR_MAX_BATCH)."""
        t = self._torch
        a = ascii_windows.contiguous()
        assert a.dtype == t.uint8 and a.dim() == 2 and a.shape[1] == WINDOW and a.is_cuda
        c = class_index(target)
        m, b = self._ig_args(steps, baseline)
        n = a.shape[0]
        probs = t.empty((n, 3), dtype=t.float32, device=a.device)
        logp = t.empty((n, 2), dtype=t.float32, device=a.device)
        attr = t.empty((n, TOKENS), dtype=t.float32, device=a.device)
        if n:
            _check(self.lib, self.lib.gnm_attribute_ig_ascii(self._h, self._attr_ctx(), a.data_ptr(), n, c, m, b, probs.data_ptr(),
                                                             logp.data_ptr(), attr.data_ptr(), self._stream()))
        return probs, logp, attr

    def integrated_gradients_windows(self, seq_u8, win_start, win_len, target, steps: int = IG_STEPS, baseline="zero"):
        """Planned windows of a sequence buffer (see predict_windows) -> (probabilities [W, 3], logp [W, 2], attributions
        [W, 5997]) by integrated gradients (see integrated_gradients_ascii)."""
        t = self._torch
        start, length = win_start.contiguous(), win_len.contiguous()
        assert start.dtype == t.int64 and length.dtype == t.int32 and start.numel() == length.numel()
        c = class_index(target)
        m, b = self._ig_args(steps, baseline)
        n = start.numel()
        probs = t.empty((n, 3), dtype=t.float32, device=seq_u8.device)
        logp = t.empty((n, 2), dtype=t.float32, device=seq_u8.device)
        attr = t.empty((n, TOKENS), dtype=t.float32, device=seq_u8.device)
        if n:
            _check(self.lib, self.lib.gnm_attribute_ig_windows(self._h, self._attr_ctx(), seq_u8.data_ptr(), start.data_ptr(),
                                                               length.data_ptr(), n, c, m, b, probs.data_ptr(), logp.data_ptr(),
                                                               attr.data_ptr(), self._stream()))
        return probs, logp, attr

    def integrated_gradients_contigs(self, seqs, target, steps: int = IG_STEPS, baseline="zero",
                                     single_window: bool = False) -> "Attributions":
        """attribute_contigs by integrated gradients: the same windows and record, attr the IG attributions and logp
        float32 [W, 2] = (log p_target(window), log p_target(baseline))."""
        t = self._torch
        seq, offs = self.contig_buffers(seqs)
        start, length, woff = self.contig_windows(seq, offs, single_window)
        n = woff.numel() - 1
        counts = (woff[1:] - woff[:-1]).to(t.int64)
        contig = t.repeat_interleave(t.arange(n, dtype=t.int32, device=seq.device), counts)
        probs, logp, attr = self.integrated_gradients_windows(seq, start, length, target, steps, baseline)
        rel = start - offs[:-1].index_select(0, contig.to(t.int64)) if start.numel() else start
        return Attributions(probs, contig, rel, length, woff, attr, logp)

    # ------------------------------------------------------------------ host-buffer API
    def classify_host(self, ascii_windows: np.ndarray) -> np.ndarray:
        """numpy uint8 [n, 6000] (host) -> numpy float32 [n, 3]; copies overlap compute inside the library."""
        a = np.ascontiguousarray(ascii_windows, dtype=np.uint8)
        assert a.ndim == 2 and a.shape[1] == WINDOW
        out = np.empty((a.shape[0], 3), dtype=np.float32)
        with self._torch.cuda.device(self.device):
            _check(self.lib, self.lib.gnm_classify_host(self._h, _ptr(a), a.shape[0], _ptr(out)))
        return out

    def classify_host_into(self, ascii_ptr: int, n: int, out_ptr: int):
        """Raw-pointer variant (pinned torch tensors): no numpy conversion on the timed path."""
        with self._torch.cuda.device(self.device):
            _check(self.lib, self.lib.gnm_classify_host(self._h, ascii_ptr, n, out_ptr))

    def check_status(self):
        """Synchronise the current stream and raise GnmError if a step reported a device-side failure
        (mbarrier time-out, activation range overflow -- see gnm_check_status in include/gnm.h)."""
        _check(self.lib, self.lib.gnm_check_status(self._h, self._stream()))

    # ------------------------------------------------------------------ introspection
    def stage_times(self) -> List[Tuple[str, float]]:
        cap = 16384
        names = (C.c_char_p * cap)()
        ms = (C.c_float * cap)()
        cnt = C.c_int(cap)
        _check(self.lib, self.lib.gnm_stage_times(self._h, names, ms, C.byref(cnt)))
        return [(names[i].decode(), float(ms[i])) for i in range(cnt.value)]

    def debug_fetch(self, which: str, n: int):
        t = self._torch
        shapes = {"buf0": (n, TOKENS, 128), "buf1": (n, TOKENS, 128), "q0": (n, 749, 128), "q1": (n, 749, 128),
                  "mpi0": (n, 2100), "mpi1": (n, 2100), "h0": (n, 256), "h1": (n, 512), "h2": (n, 512), "logits": (n, 752),
                  "conv_dbg": (self.get_option("num_sms"), 16), "routeq0": (n, 749, 128), "routeq1": (n, 749, 128),
                  "route0": (n, 749, 128), "route1": (n, 749, 128), "attr_y1": (n, TOKENS, 128), "attr_g_out": (n, 256),
                  "attr_s_w": (n,), "attr_s2": (n,), "attr_gz3": (n, TOKENS, 128), "attr_gz2": (n, TOKENS, 128),
                  "attr_gy1": (n, TOKENS, 128), "attr_gz1": (n, TOKENS, 128), "attr_g_h1": (n, EMBED)}
        dtype = t.uint8 if which in ("route0", "route1") else t.float32
        out = t.empty(shapes[which], dtype=dtype, device=self._dev())
        _check(self.lib, self.lib.gnm_debug_fetch(self._h, which.encode(), n, out.data_ptr(), self._stream()))
        return out


# ------------------------------------------------------------------------------------------------ classifier heads
def head_param_count(C: int) -> int:
    """Floats of a head's flat parameter buffer: W1, b1, gamma, beta, W2, b2 (gnm_head_train_read)."""
    return EMBED * EMBED + 3 * EMBED + EMBED * C + C


class NoveltyFit(NamedTuple):
    """A fitted novelty model (gnm_novelty_fit, include/gnm.h): center [512], whitening P [512, 512] (lower triangular),
    means [C, 512] (whitened class means m_c), all float64; the smallest Cholesky pivot; and, with stats=True, the class means
    mu_c [C, 512] and the scatter S [512, 512] (None otherwise)."""
    center: np.ndarray
    whitening: np.ndarray
    means: np.ndarray
    min_pivot: float
    class_means: Optional[np.ndarray] = None
    scatter: Optional[np.ndarray] = None


def novelty_fit(clf: "Classifier", X, rows, labels, n_classes: int, stats: bool = False) -> NoveltyFit:
    """Fit the novelty model on rows `rows` (int64 cuda [N]) of X (float32 cuda [n_rows, 512]) with labels (int32 cuda
    [n_rows], the label of each row of X), on clf's device.  GnmError on an empty class, no within-class variation or a
    non-positive pivot."""
    t = clf._torch
    assert X.dtype == t.float32 and X.dim() == 2 and X.shape[1] == EMBED and X.is_cuda and X.is_contiguous()
    assert rows.dtype == t.int64 and labels.dtype == t.int32 and labels.numel() == X.shape[0]
    C_ = int(n_classes)
    n = int(rows.numel())
    need = int(clf.lib.gnm_novelty_fit_workspace_bytes(max(n, 1), C_))
    if need == 0:
        raise GnmError(clf.lib.gnm_last_error().decode(errors="replace"))
    work = t.empty(need + 256, dtype=t.uint8, device=X.device)
    base = (-work.data_ptr()) % 256
    center, whitening, means = np.empty(EMBED), np.empty((EMBED, EMBED)), np.empty((C_, EMBED))
    mu = np.empty((C_, EMBED)) if stats else None
    S = np.empty((EMBED, EMBED)) if stats else None
    piv = C.c_double()
    with t.cuda.device(clf.device):
        _check(clf.lib, clf.lib.gnm_novelty_fit(clf._h, X.data_ptr(), X.shape[0], rows.contiguous().data_ptr(), n,
                                                labels.contiguous().data_ptr(), C_, _ptr(center), _ptr(whitening),
                                                _ptr(means), C.byref(piv), _ptr(mu) if stats else None,
                                                _ptr(S) if stats else None, work.data_ptr() + base, need, clf._stream()))
    return NoveltyFit(center, whitening, means, piv.value, mu, S)


def novelty_scores(dist, counts, calibration):
    """Per-sequence novelty from the per-contig mean window distances dist (float32 [n, C]), the window counts [n] and the
    head's sorted calibration values (float32): (novelty float32 [n] = min_c dist, nearest_class int32 [n] = the argmin,
    lowest index on ties, p_value float64 [n] = (1 + #{v in calibration : v >= novelty}) / (1 + |calibration|)).  A sequence
    without a window, or whose distances are not all finite, gets novelty NaN, nearest_class -1 and p NaN."""
    dist = np.asarray(dist, dtype=np.float32)
    counts = np.asarray(counts).reshape(-1)
    cal = np.asarray(calibration, dtype=np.float32).reshape(-1)
    n = len(counts)
    assert dist.ndim == 2 and len(dist) == n
    has = (counts > 0) & np.isfinite(dist).all(1)
    nov = np.full(n, np.nan, np.float32)
    nearest = np.full(n, -1, np.int32)
    p = np.full(n, np.nan, np.float64)
    if has.any():
        d = dist[has]
        nearest[has] = d.argmin(1)
        nov[has] = d.min(1)
        ge = len(cal) - np.searchsorted(cal, nov[has], side="left")
        p[has] = (1.0 + ge) / (1.0 + len(cal))
    return nov, nearest, p


class Head:
    """A C-class head (weights.HeadFile, or a dict with arrays / class_names) on a Classifier's device and workspace: encoder
    embeddings -> class probabilities (gnm_head_forward), per-contig means and sums (gnm_head_segment_*).  Follows the
    classifier's conv_impl; the shipped head at C = 3 gives bitwise the classifier's own probabilities."""

    def __init__(self, clf: "Classifier", head):
        self.clf, self.lib = clf, clf.lib
        self.class_names = tuple(head.class_names)
        self._a = {k: np.ascontiguousarray(head.arrays[k], dtype=np.float32) for k in _weights.HEAD_KEYS}
        self.n_classes = int(self._a["d2b"].shape[0])
        hw = _weights.head_c_struct(self._a, _HeadW, _BnW)
        self._hd = C.c_void_p()
        with clf._torch.cuda.device(clf.device):
            rc = self.lib.gnm_head_create(clf._h, C.byref(hw), C.byref(self._hd))
        if rc != 0:
            msg = self.lib.gnm_last_error().decode(errors="replace")
            self.close()
            raise GnmError(msg)
        self.calibration = None
        nov = getattr(head, "novelty", None)
        if nov is not None:
            self.set_novelty(nov["novelty_center"], nov["novelty_whitening"], nov["novelty_means"], nov["novelty_calibration"])

    @property
    def has_novelty(self) -> bool:
        return getattr(self, "_nv", None) is not None

    def set_novelty(self, center, whitening, means, calibration=None):
        """Attach a novelty model (float64 center [512], whitening [512, 512] lower triangular, whitened means [C, 512];
        gnm_head_set_novelty) and, when given, its sorted float32 calibration values."""
        self._nv = tuple(np.ascontiguousarray(a, dtype=np.float64) for a in (center, whitening, means))
        assert self._nv[0].shape == (EMBED,) and self._nv[1].shape == (EMBED, EMBED) and self._nv[2].shape == (self.n_classes, EMBED)
        with self.clf._torch.cuda.device(self.clf.device):
            _check(self.lib, self.lib.gnm_head_set_novelty(self.clf._h, self._hd, *(_ptr(a) for a in self._nv)))
        self.calibration = None if calibration is None else np.asarray(calibration, dtype=np.float32)

    def novelty(self, embeddings, out=None):
        """float32 cuda [n, 512] -> float32 [n, C]: each row's whitened squared distance to every class mean / 512
        (gnm_head_novelty), into `out` when given."""
        t = self.clf._torch
        x = embeddings.contiguous()
        assert x.dtype == t.float32 and x.dim() == 2 and x.shape[1] == EMBED and x.is_cuda
        if out is None:
            out = t.empty((x.shape[0], self.n_classes), dtype=t.float32, device=x.device)
        assert out.shape == (x.shape[0], self.n_classes) and out.is_contiguous() and out.dtype == t.float32
        if x.shape[0]:
            _check(self.lib, self.lib.gnm_head_novelty(self.clf._h, self._hd, x.data_ptr(), x.shape[0], out.data_ptr(),
                                                       self.clf._stream()))
        return out

    def novelty_contigs(self, seqs, single_window: bool = False):
        """Contigs in, cuda tensors (per-contig mean window distances float32 [n_contigs, C], window counts int32
        [n_contigs]) out: the windows of classify_contigs (forward strand), embedded, scored by novelty and averaged by
        segment_mean.  novelty_scores turns them into (novelty, nearest_class, p_value)."""
        clf, t = self.clf, self.clf._torch
        seq, offs = clf.contig_buffers(seqs)
        start, length, woff = clf.contig_windows(seq, offs, single_window)
        if start.numel():
            dist = self.novelty(clf.embed_windows(seq, start, length)[1])
        else:
            dist = t.zeros((0, self.n_classes), dtype=t.float32, device=seq.device)
        return self.segment_mean(dist, woff), woff[1:] - woff[:-1]

    def close(self):
        if getattr(self, "_hd", None):
            self.lib.gnm_head_destroy(self._hd)
            self._hd = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def predict(self, embeddings, out=None):
        """float32 cuda [n, 512] -> float32 [n, C] probabilities (into `out` when given)."""
        t = self.clf._torch
        x = embeddings.contiguous()
        assert x.dtype == t.float32 and x.dim() == 2 and x.shape[1] == EMBED and x.is_cuda
        if out is None:
            out = t.empty((x.shape[0], self.n_classes), dtype=t.float32, device=x.device)
        assert out.shape == (x.shape[0], self.n_classes) and out.is_contiguous() and out.dtype == t.float32
        if x.shape[0]:
            _check(self.lib, self.lib.gnm_head_forward(self.clf._h, self._hd, x.data_ptr(), x.shape[0], out.data_ptr(),
                                                       self.clf._stream()))
        return out

    # ------------------------------------------------------------------ contigs in memory
    def classify_contigs(self, seqs, single_window: bool = False, strand: str = "forward"):
        """Classifier.classify_contigs for the head's classes: contigs in, cuda tensors (means float32 [n_contigs, C], window
        counts int32 [n_contigs]) out.  The windows are planned on the device (Classifier.contig_windows), embedded
        (Classifier.embed_windows), scored by predict and averaged per contig by segment_mean; a contig without a window has
        count 0 and mean 0.  strand "reverse" scores each contig's reverse complement: bitwise the forward call on the
        reverse-complemented contigs, and both_strands() combines the two calls' means."""
        clf = self.clf
        if strand not in ("forward", "reverse"):
            raise ValueError(f"strand must be 'forward' or 'reverse', not {strand!r}")
        rev = strand == "reverse"
        seq, offs = clf.contig_buffers(seqs)
        start, length, woff = clf.contig_windows(seq, offs, single_window, reverse=rev)
        probs = self._window_probs(seq, start, length, rev)
        return self.segment_mean(probs, woff), woff[1:] - woff[:-1]

    def window_scores(self, seqs, stride: int = WINDOW) -> "WindowScores":
        """Classifier.window_scores for the head's classes: WindowScores with probs float32 [W, C], the head's scores of every
        window (a window every `stride` nt), and the same contig, start, length and offsets as Classifier.window_scores."""
        clf, t = self.clf, self.clf._torch
        seq, offs = clf.contig_buffers(seqs)
        start, length, woff = clf.contig_windows(seq, offs, stride=stride)
        n = woff.numel() - 1
        counts = (woff[1:] - woff[:-1]).to(t.int64)
        contig = t.repeat_interleave(t.arange(n, dtype=t.int32, device=seq.device), counts)
        probs = self._window_probs(seq, start, length, False)
        rel = start - offs[:-1].index_select(0, contig.to(t.int64)) if start.numel() else start
        return WindowScores(probs, contig, rel, length, woff)

    def _window_probs(self, seq, start, length, reverse):
        t = self.clf._torch
        if not start.numel():
            return t.zeros((0, self.n_classes), dtype=t.float32, device=seq.device)
        return self.predict(self.clf.embed_windows(seq, start, length, reverse=reverse)[1])

    # ------------------------------------------------------------------ attributions of the head's classes
    def class_index(self, target) -> int:
        """An index in [0, C) or one of class_names -> class index."""
        if isinstance(target, str):
            if target not in self.class_names:
                raise ValueError(f"target must be one of the head's classes {self.class_names}, not {target!r}")
            return self.class_names.index(target)
        t = int(target)
        if not 0 <= t < self.n_classes:
            raise ValueError(f"target must be in [0, {self.n_classes}), not {t}")
        return t

    def _attr_out(self, n, device, ig):
        t = self.clf._torch
        probs = t.empty((n, 3), dtype=t.float32, device=device)
        head_probs = t.empty((n, self.n_classes), dtype=t.float32, device=device)
        logp = t.empty((n, 2), dtype=t.float32, device=device) if ig else None
        attr = t.empty((n, TOKENS), dtype=t.float32, device=device)
        return probs, head_probs, logp, attr

    def attribute_ascii(self, ascii_windows, target):
        """uint8 cuda [n, 6000], a class of the head (index or name) -> (probabilities float32 [n, 3], head probabilities
        [n, C], attributions [n, 5997]): attr[i, t] = d log p_target / d x[t, tok[t]] for the head's p (gnm_attribute_head_ascii),
        through the classifier's attribution context.  The probabilities are bitwise those of Classifier.predict_ascii, the head
        probabilities those of predict(embed_ascii(...))."""
        clf = self.clf
        a = ascii_windows.contiguous()
        assert a.dtype == clf._torch.uint8 and a.dim() == 2 and a.shape[1] == WINDOW and a.is_cuda
        c = self.class_index(target)
        probs, head_probs, _, attr = self._attr_out(a.shape[0], a.device, False)
        if a.shape[0]:
            _check(self.lib, self.lib.gnm_attribute_head_ascii(clf._h, clf._attr_ctx(), self._hd, a.data_ptr(), a.shape[0], c,
                                                               probs.data_ptr(), head_probs.data_ptr(), attr.data_ptr(),
                                                               clf._stream()))
        return probs, head_probs, attr

    def attribute_windows(self, seq_u8, win_start, win_len, target):
        """Planned windows of a sequence buffer (see Classifier.predict_windows) -> (probabilities [W, 3], head probabilities
        [W, C], attributions [W, 5997])."""
        clf, t = self.clf, self.clf._torch
        start, length = win_start.contiguous(), win_len.contiguous()
        assert start.dtype == t.int64 and length.dtype == t.int32 and start.numel() == length.numel()
        c = self.class_index(target)
        n = start.numel()
        probs, head_probs, _, attr = self._attr_out(n, seq_u8.device, False)
        if n:
            _check(self.lib, self.lib.gnm_attribute_head_windows(clf._h, clf._attr_ctx(), self._hd, seq_u8.data_ptr(),
                                                                 start.data_ptr(), length.data_ptr(), n, c, probs.data_ptr(),
                                                                 head_probs.data_ptr(), attr.data_ptr(), clf._stream()))
        return probs, head_probs, attr

    def _contig_record(self, seqs, single_window, attr_fn):
        clf, t = self.clf, self.clf._torch
        seq, offs = clf.contig_buffers(seqs)
        start, length, woff = clf.contig_windows(seq, offs, single_window)
        n = woff.numel() - 1
        counts = (woff[1:] - woff[:-1]).to(t.int64)
        contig = t.repeat_interleave(t.arange(n, dtype=t.int32, device=seq.device), counts)
        out = attr_fn(seq, start, length)
        rel = start - offs[:-1].index_select(0, contig.to(t.int64)) if start.numel() else start
        probs, head_probs, attr = out[0], out[1], out[-1]
        logp = out[2] if len(out) == 4 else None
        return Attributions(probs, contig, rel, length, woff, attr, logp, head_probs)

    def attribute_contigs(self, seqs, target, single_window: bool = False) -> "Attributions":
        """Classifier.attribute_contigs for a class of the head: the same windows and record, with head_probs [W, C]."""
        return self._contig_record(seqs, single_window, lambda s, b, l: self.attribute_windows(s, b, l, target))

    def integrated_gradients_ascii(self, ascii_windows, target, steps: int = IG_STEPS, baseline="zero"):
        """uint8 cuda [n, 6000], a class of the head -> (probabilities [n, 3], head probabilities [n, C], logp [n, 2],
        attributions [n, 5997]) by integrated gradients of the head's log p_target (gnm_attribute_head_ig_ascii; the rule of
        Classifier.integrated_gradients_ascii)."""
        clf = self.clf
        a = ascii_windows.contiguous()
        assert a.dtype == clf._torch.uint8 and a.dim() == 2 and a.shape[1] == WINDOW and a.is_cuda
        c = self.class_index(target)
        m, b = clf._ig_args(steps, baseline)
        n = a.shape[0]
        probs, head_probs, logp, attr = self._attr_out(n, a.device, True)
        if n:
            _check(self.lib, self.lib.gnm_attribute_head_ig_ascii(clf._h, clf._attr_ctx(), self._hd, a.data_ptr(), n, c, m, b,
                                                                  probs.data_ptr(), head_probs.data_ptr(), logp.data_ptr(),
                                                                  attr.data_ptr(), clf._stream()))
        return probs, head_probs, logp, attr

    def integrated_gradients_windows(self, seq_u8, win_start, win_len, target, steps: int = IG_STEPS, baseline="zero"):
        """Planned windows of a sequence buffer -> (probabilities [W, 3], head probabilities [W, C], logp [W, 2], attributions
        [W, 5997]) by integrated gradients (see integrated_gradients_ascii)."""
        clf, t = self.clf, self.clf._torch
        start, length = win_start.contiguous(), win_len.contiguous()
        assert start.dtype == t.int64 and length.dtype == t.int32 and start.numel() == length.numel()
        c = self.class_index(target)
        m, b = clf._ig_args(steps, baseline)
        n = start.numel()
        probs, head_probs, logp, attr = self._attr_out(n, seq_u8.device, True)
        if n:
            _check(self.lib, self.lib.gnm_attribute_head_ig_windows(clf._h, clf._attr_ctx(), self._hd, seq_u8.data_ptr(),
                                                                    start.data_ptr(), length.data_ptr(), n, c, m, b,
                                                                    probs.data_ptr(), head_probs.data_ptr(), logp.data_ptr(),
                                                                    attr.data_ptr(), clf._stream()))
        return probs, head_probs, logp, attr

    def integrated_gradients_contigs(self, seqs, target, steps: int = IG_STEPS, baseline="zero",
                                     single_window: bool = False) -> "Attributions":
        """attribute_contigs by integrated gradients, with logp [W, 2] of the head's class."""
        return self._contig_record(seqs, single_window,
                                   lambda s, b, l: self.integrated_gradients_windows(s, b, l, target, steps, baseline))

    # ------------------------------------------------------------------ attributions of the novelty distance
    def novelty_targets(self, target, n: int) -> np.ndarray:
        """A class of the head (index or name) or an int array [n] of classes -> host int32 [n], each entry checked."""
        if isinstance(target, (str, int, np.integer)):
            return np.full(n, self.class_index(target), np.int32)
        tg = target.cpu().numpy() if hasattr(target, "cpu") else np.asarray(target)
        if tg.shape != (n,) or tg.dtype.kind not in "iu":
            raise ValueError(f"target must be a class of the head or an integer array of {n} classes, not {tg.dtype} {tg.shape}")
        bad = np.flatnonzero((tg < 0) | (tg >= self.n_classes))
        if bad.size:
            raise ValueError(f"target[{bad[0]}] = {tg[bad[0]]} is not a class of the head, in [0, {self.n_classes})")
        return np.ascontiguousarray(tg, dtype=np.int32)

    def _novelty_out(self, n, device, ig):
        t = self.clf._torch
        probs = t.empty((n, 3), dtype=t.float32, device=device)
        dist = t.empty((n, self.n_classes), dtype=t.float32, device=device)
        dist_target = t.empty((n, 2), dtype=t.float32, device=device) if ig else None
        attr = t.empty((n, TOKENS), dtype=t.float32, device=device)
        return probs, dist, dist_target, attr

    def attribute_novelty_ascii(self, ascii_windows, target):
        """uint8 cuda [n, 6000], target class(es) (a class of the head, or an int array [n]) -> (probabilities float32 [n, 3],
        distances [n, C], attributions [n, 5997]): attr[i, t] = d D_c / d x[t, tok[t]] for window i's whitened distance D_c to
        its target class c (gnm_attribute_novelty_ascii).  The probabilities are bitwise those of Classifier.predict_ascii, the
        distances those of novelty(embed_ascii(...))."""
        clf = self.clf
        a = ascii_windows.contiguous()
        assert a.dtype == clf._torch.uint8 and a.dim() == 2 and a.shape[1] == WINDOW and a.is_cuda
        n = a.shape[0]
        tg = self.novelty_targets(target, n)
        probs, dist, _, attr = self._novelty_out(n, a.device, False)
        if n:
            _check(self.lib, self.lib.gnm_attribute_novelty_ascii(clf._h, clf._attr_ctx(), self._hd, a.data_ptr(), n, _ptr(tg),
                                                                  probs.data_ptr(), dist.data_ptr(), attr.data_ptr(),
                                                                  clf._stream()))
        return probs, dist, attr

    def attribute_novelty_windows(self, seq_u8, win_start, win_len, target):
        """Planned windows of a sequence buffer -> (probabilities [W, 3], distances [W, C], attributions [W, 5997])."""
        clf, t = self.clf, self.clf._torch
        start, length = win_start.contiguous(), win_len.contiguous()
        assert start.dtype == t.int64 and length.dtype == t.int32 and start.numel() == length.numel()
        n = start.numel()
        tg = self.novelty_targets(target, n)
        probs, dist, _, attr = self._novelty_out(n, seq_u8.device, False)
        if n:
            _check(self.lib, self.lib.gnm_attribute_novelty_windows(clf._h, clf._attr_ctx(), self._hd, seq_u8.data_ptr(),
                                                                    start.data_ptr(), length.data_ptr(), n, _ptr(tg),
                                                                    probs.data_ptr(), dist.data_ptr(), attr.data_ptr(),
                                                                    clf._stream()))
        return probs, dist, attr

    def integrated_gradients_novelty_ascii(self, ascii_windows, target, steps: int = IG_STEPS, baseline="zero"):
        """uint8 cuda [n, 6000], target class(es) -> (probabilities [n, 3], distances [n, C], dist_target [n, 2] = (D_c(x),
        D_c(x')), attributions [n, 5997]) by integrated gradients of D_c (gnm_attribute_novelty_ig_ascii; the rule of
        Classifier.integrated_gradients_ascii).  The attributions add up to about D_c(x) - D_c(x')."""
        clf = self.clf
        a = ascii_windows.contiguous()
        assert a.dtype == clf._torch.uint8 and a.dim() == 2 and a.shape[1] == WINDOW and a.is_cuda
        n = a.shape[0]
        tg = self.novelty_targets(target, n)
        m, b = clf._ig_args(steps, baseline)
        probs, dist, dist_target, attr = self._novelty_out(n, a.device, True)
        if n:
            _check(self.lib, self.lib.gnm_attribute_novelty_ig_ascii(clf._h, clf._attr_ctx(), self._hd, a.data_ptr(), n, _ptr(tg),
                                                                     m, b, probs.data_ptr(), dist.data_ptr(),
                                                                     dist_target.data_ptr(), attr.data_ptr(), clf._stream()))
        return probs, dist, dist_target, attr

    def integrated_gradients_novelty_windows(self, seq_u8, win_start, win_len, target, steps: int = IG_STEPS,
                                             baseline="zero"):
        """Planned windows of a sequence buffer -> (probabilities [W, 3], distances [W, C], dist_target [W, 2], attributions
        [W, 5997]) by integrated gradients of D_c (see integrated_gradients_novelty_ascii)."""
        clf, t = self.clf, self.clf._torch
        start, length = win_start.contiguous(), win_len.contiguous()
        assert start.dtype == t.int64 and length.dtype == t.int32 and start.numel() == length.numel()
        n = start.numel()
        tg = self.novelty_targets(target, n)
        m, b = clf._ig_args(steps, baseline)
        probs, dist, dist_target, attr = self._novelty_out(n, seq_u8.device, True)
        if n:
            _check(self.lib, self.lib.gnm_attribute_novelty_ig_windows(clf._h, clf._attr_ctx(), self._hd, seq_u8.data_ptr(),
                                                                       start.data_ptr(), length.data_ptr(), n, _ptr(tg), m, b,
                                                                       probs.data_ptr(), dist.data_ptr(),
                                                                       dist_target.data_ptr(), attr.data_ptr(), clf._stream()))
        return probs, dist, dist_target, attr

    def nearest_window_targets(self, seqs, single_window: bool = False, names=None) -> np.ndarray:
        """int32 [W]: each window of the contig pass gets its sequence's nearest class (novelty_contigs + novelty_scores).  A
        sequence with windows but no nearest class (a distance that is not finite) is refused, named from `names` if given."""
        if not self.has_novelty:
            raise GnmError("the head has no novelty model (train-head --novelty)")
        dist, counts = self.novelty_contigs(seqs, single_window)
        counts = counts.cpu().numpy()
        cal = self.calibration if self.calibration is not None else np.zeros(0, np.float32)
        _, nearest, _ = novelty_scores(dist.cpu().numpy(), counts, cal)
        bad = np.flatnonzero((nearest < 0) & (counts > 0))
        if bad.size:
            i = int(bad[0])
            who = names[i] if names is not None else f"sequence {i}"
            raise GnmError(f"{who}: its window distances are not finite, so it has no nearest class to attribute")
        return np.repeat(nearest, counts).astype(np.int32)

    def _novelty_record(self, seqs, single_window, attr_fn, names=None):
        clf, t = self.clf, self.clf._torch
        target = self.nearest_window_targets(seqs, single_window, names)
        seq, offs = clf.contig_buffers(seqs)
        start, length, woff = clf.contig_windows(seq, offs, single_window)
        n = woff.numel() - 1
        counts = (woff[1:] - woff[:-1]).to(t.int64)
        contig = t.repeat_interleave(t.arange(n, dtype=t.int32, device=seq.device), counts)
        out = attr_fn(seq, start, length, target)
        rel = start - offs[:-1].index_select(0, contig.to(t.int64)) if start.numel() else start
        dist_target = out[2] if len(out) == 4 else None
        return Attributions(out[0], contig, rel, length, woff, out[-1], dist_target, out[1],
                            t.from_numpy(target).to(seq.device))

    def attribute_novelty_contigs(self, seqs, single_window: bool = False, names=None) -> "Attributions":
        """Attributions of every window of the contig pass to its distance to its sequence's nearest class (the class the
        novelty file reports), with head_probs the windows' distances [W, C] and target their class [W].  A sequence with
        windows but no nearest class is refused, by its name in `names` when given."""
        return self._novelty_record(seqs, single_window, self.attribute_novelty_windows, names)

    def integrated_gradients_novelty_contigs(self, seqs, steps: int = IG_STEPS, baseline="zero",
                                             single_window: bool = False, names=None) -> "Attributions":
        """attribute_novelty_contigs by integrated gradients, with logp [W, 2] = (D_c(window), D_c(baseline))."""
        return self._novelty_record(seqs, single_window,
                                    lambda s, b, l, tg: self.integrated_gradients_novelty_windows(s, b, l, tg, steps, baseline),
                                    names)

    def _segment(self, fn, probs, offsets, width):
        t = self.clf._torch
        assert probs.dtype == t.float32 and offsets.dtype == t.int32 and probs.is_cuda and offsets.is_cuda
        C_ = probs.shape[1]
        n = offsets.numel() - 1
        out = t.zeros((n, width(C_)), dtype=t.float32, device=probs.device)
        if n and probs.numel():
            _check(self.lib, fn(self.clf._h, probs.contiguous().data_ptr(), C_, offsets.contiguous().data_ptr(), n,
                                out.data_ptr(), self.clf._stream()))
        return out

    def segment_mean(self, probs, offsets):
        """probs float32 cuda [W, C], offsets int32 cuda [n + 1] -> float32 [n, C]: fp32 running mean in window order."""
        return self._segment(self.lib.gnm_head_segment_mean, probs, offsets, lambda c: c)

    def segment_sum(self, probs, offsets):
        """-> float32 [n, C + 1] = (sums, window count): the cross-GPU partial."""
        return self._segment(self.lib.gnm_head_segment_sum, probs, offsets, lambda c: c + 1)


class HeadTrainer:
    """Training of a C-class head on cached embeddings (gnm_head_train_*; semantics in include/gnm.h).  `init` maps the
    short names of weights.HEAD_KEYS to the initial arrays (weights.initial_head)."""

    def __init__(self, init: Dict[str, np.ndarray], device: int = 0, max_batch: int = 1024, seed: int = 0,
                 learning_rate: float = 1e-3):
        import torch
        self._torch = torch
        self.lib = load_library()
        self.device, self.max_batch = int(device), int(max_batch)
        self._a = {k: np.ascontiguousarray(init[k], dtype=np.float32) for k in _weights.HEAD_KEYS}
        self.n_classes = int(self._a["d2b"].shape[0])
        hw = _weights.head_c_struct(self._a, _HeadW, _BnW)
        self._tr = C.c_void_p()
        with torch.cuda.device(self.device):
            rc = self.lib.gnm_head_train_create(self.device, C.byref(hw), self.max_batch, int(seed) & 0xFFFFFFFFFFFFFFFF,
                                                float(learning_rate), C.byref(self._tr))
        if rc != 0:
            msg = self.lib.gnm_last_error().decode(errors="replace")
            self.close()
            raise GnmError(msg)

    def close(self):
        if getattr(self, "_tr", None):
            self.lib.gnm_head_train_destroy(self._tr)
            self._tr = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self) -> int:
        return self._torch.cuda.current_stream(self.device).cuda_stream

    def step(self, X, idx, labels, class_weights, loss=None):
        """One step on rows idx (int64 cuda [B]) of X (float32 cuda [N, 512]); labels int32 cuda [N]; class_weights float32
        cuda [C].  Returns the batch loss, float32 cuda [1] (`loss` when given).  Asynchronous: an index outside [0, N) or a
        label outside [0, C) is caught on the device, and the next step or weights() raises GnmError."""
        t = self._torch
        assert X.dtype == t.float32 and X.dim() == 2 and X.shape[1] == EMBED and X.is_contiguous()
        assert idx.dtype == t.int64 and labels.dtype == t.int32 and class_weights.dtype == t.float32
        assert class_weights.numel() == self.n_classes and labels.numel() == X.shape[0]
        if loss is None:
            loss = t.empty(1, dtype=t.float32, device=X.device)
        with t.cuda.device(self.device):
            _check(self.lib, self.lib.gnm_head_train_step(self._tr, X.data_ptr(), X.shape[0], idx.contiguous().data_ptr(),
                                                          labels.contiguous().data_ptr(), class_weights.contiguous().data_ptr(),
                                                          idx.numel(), loss.data_ptr(), self._stream()))
        self._last_b = idx.numel()
        return loss

    def weights(self) -> Dict[str, np.ndarray]:
        """The current parameters and moving statistics as arrays for weights.save_head (waits for the device)."""
        C_ = self.n_classes
        flat = np.empty(head_param_count(C_), np.float32)
        mm, mv = np.empty(EMBED, np.float32), np.empty(EMBED, np.float32)
        step = C.c_longlong()
        with self._torch.cuda.device(self.device):
            _check(self.lib, self.lib.gnm_head_train_read(self._tr, _ptr(flat), _ptr(mm), _ptr(mv), C.byref(step),
                                                          self._stream()))
        self.steps = step.value
        return {**_unflatten_head(flat, C_), "bn1m": mm, "bn1v": mv}

    def fetch(self, which: str):
        """Test hook: the last step's "grad", "adam_m" or "adam_v" (dicts by short name: the gradients, the Adam moments after
        the step), "mask" (uint8 [B, 512]) or "batch_stats" (float32 [3, 512]: mu, 1 / sqrt(var + 1e-3), var)."""
        flat = which in ("grad", "adam_m", "adam_v")
        if flat:
            out = np.empty(head_param_count(self.n_classes), np.float32)
        elif which == "mask":
            out = np.empty((getattr(self, "_last_b", 0), EMBED), np.uint8)
        else:
            out = np.empty((3, EMBED), np.float32)
        with self._torch.cuda.device(self.device):
            _check(self.lib, self.lib.gnm_head_train_fetch(self._tr, which.encode(), _ptr(out), self._stream()))
        return _unflatten_head(out, self.n_classes) if flat else out


def _unflatten_head(flat: np.ndarray, C_: int) -> Dict[str, np.ndarray]:
    E = EMBED
    parts, o = {}, 0
    for k, shape in (("d1w", (E, E)), ("d1b", (E,)), ("bn1g", (E,)), ("bn1b", (E,)), ("d2w", (E, C_)), ("d2b", (C_,))):
        n = int(np.prod(shape))
        parts[k] = flat[o: o + n].reshape(shape).copy()
        o += n
    return parts
