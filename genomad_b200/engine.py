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
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import weights as _weights

_PKG = Path(__file__).resolve().parent
_LIB_PATH = Path(os.environ["GENOMAD_B200_LIB"]) if os.environ.get("GENOMAD_B200_LIB") else _PKG / "libgnm.so"   # dev: A/B two builds
_lib = None

WINDOW = 6000
TOKENS = 5997


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
    "gnm_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int]),
    "gnm_get_option": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_int)]),
    "gnm_kernel_launches": (C.c_longlong, [C.c_void_p]),
    "gnm_stage_times": (C.c_int, [C.c_void_p, C.POINTER(C.c_char_p), C.POINTER(C.c_float), C.POINTER(C.c_int)]),
    "gnm_debug_fetch": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int, C.c_void_p, C.c_void_p]),
    "gnm_pack_patches": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.POINTER(C.c_int), C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.c_void_p]),
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
        """uint16 cuda tensor [n, 5997] -> float32 probabilities [n, 3]; the analogue of nn_model.predict(batch)."""
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
                  "mpi0": (n, 2100), "mpi1": (n, 2100), "h0": (n, 256), "logits": (n, 752),
                  "conv_dbg": (self.get_option("num_sms"), 16)}
        out = t.empty(shapes[which], dtype=t.float32, device=self._dev())
        _check(self.lib, self.lib.gnm_debug_fetch(self._h, which.encode(), n, out.data_ptr(), self._stream()))
        return out
