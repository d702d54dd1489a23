"""
Host-side FASTA reading, windowing and window-matrix construction for nn-classification.

Mirrors the behaviour (not the code) of the reference's ``genomad/sequence.py:96-167`` and the
window rules of ``genomad/modules/nn_classification.py:65-72``; the quirks that are pinned by golden
vectors made with the real reference code (tests/golden/encoder_golden.json):

  * files are read in text mode with universal newlines: ``\\r\\n`` and ``\\r`` end a line like ``\\n``;
  * everything before the first line that starts with ``>`` is ignored;
  * a record's name is the first whitespace-delimited token of its header line;
  * leading/trailing ``n``/``N`` of the whole contig are stripped; records that are then empty are dropped;
  * windows are consecutive 6000-nt slices; the last slice is kept only if it has >= 2500 nt, except
    that the first window is always kept; ``--single-window`` keeps only the first;
  * a window other than the first is skipped if it contains more than 4000 upper-case ``N`` in the
    RAW text (lower-case ``n`` does not count) -- nn_classification.py:70-71;
  * windows are upper-cased and right-padded with ``N`` to 6000 bytes (nn_classification.py:72).

Unlike the reference (a Python generator of ``Sequence`` objects feeding a per-window numba call), the
production path (``ParsedFasta`` / ``encode_fasta``) is native code in libgnm.so (csrc/fasta.cpp): a
multi-threaded INDEX pass over the mmap'ed file (O(records) state, no copy), after which any block of the global
window list is exported straight from the file text into pinned uint8 [n, 6000] chunks that are shipped to the
GPU as they are -- tokenisation happens on the device (csrc/encode.cuh).  gzip input is inflated natively into
memory (BGZF files block-parallel on all reader threads); bz2 / xz / zstd go through Python's bindings.  ``iter_fasta`` / ``window_spans`` /
``encode_fasta_py`` are the readable pure-Python statement of the same rules; the tests hold the native code
to them and both to golden vectors made with the real reference.

Score profiles (``--write-window-scores --window-stride s``) use the same rules with a window every s nt instead of
every 6000 (``profile_spans``; ``ParsedFasta.windows(s)`` is the native list, ``gnm_contig_windows_stride`` the device
one).
"""
from __future__ import annotations

import bz2
import gzip
import lzma
from dataclasses import dataclass
from pathlib import Path
from typing import Iterator, List, Optional, Tuple

import numpy as np

WINDOW = 6000
MIN_TAIL = 2500
MAX_N = 4000


class Compression:
    bzip2, gzip, xz, zstd, uncompressed = "bzip2", "gzip", "xz", "zstd", "uncompressed"


def is_compressed(path) -> str:
    """Magic-number sniffing, same formats as reference utils.py:126-152."""
    with open(path, "rb") as fh:
        sig = fh.read(8)
    if sig[:2] == b"\x1f\x8b":
        return Compression.gzip
    if sig[:3] == b"BZh":
        return Compression.bzip2
    if sig[:7] == b"\xfd7zXZ\x00\x00":
        return Compression.xz
    if sig[:4] == b"\x28\xb5\x2f\xfd":
        return Compression.zstd
    return Compression.uncompressed


def read_bytes(path) -> bytes:
    kind = is_compressed(path)
    if kind == Compression.gzip:
        with gzip.open(path, "rb") as fh:
            return fh.read()
    if kind == Compression.bzip2:
        with bz2.open(path, "rb") as fh:
            return fh.read()
    if kind == Compression.xz:
        with lzma.open(path, "rb") as fh:
            return fh.read()
    if kind == Compression.zstd:
        try:
            from compression import zstd  # Python >= 3.14, as in the reference
        except ImportError as e:  # pragma: no cover
            raise RuntimeError("zstd-compressed input needs Python >= 3.14") from e
        with zstd.open(path, "rb") as fh:
            return fh.read()
    with open(path, "rb") as fh:
        return fh.read()


def iter_fasta(path, strip_n: bool = True) -> Iterator[Tuple[str, bytes]]:
    """Yield (header, sequence bytes) for every record that is non-empty after stripping."""
    data = read_bytes(path)
    if b"\r" in data:                       # universal newlines
        data = data.replace(b"\r\n", b"\n").replace(b"\r", b"\n")
    chunks = (b"\n" + data).split(b"\n>")
    for rec in chunks[1:]:                  # chunks[0] is whatever precedes the first header line
        header, _, body = rec.partition(b"\n")
        seq = body.replace(b"\n", b"")
        if strip_n:
            seq = seq.strip(b"nN")
        if seq:
            yield header.decode("utf-8", errors="replace"), seq


def accession(header: str) -> str:
    parts = header.split()
    if not parts:
        raise ValueError("FASTA record with an empty header line")
    return parts[0]


def check_fasta(path) -> bool:
    """False if the file has no record or two records share an identifier (reference sequence.py:124-131).
    Note: like the reference, this pass does NOT strip Ns (only truly empty records are dropped)."""
    names = [accession(h) for h, _ in iter_fasta(path, strip_n=False)]
    return bool(names) and len(names) == len(set(names))


def window_spans(length: int, single_window: bool = False) -> List[Tuple[int, int]]:
    """[start, end) of every candidate window of a contig of `length` nt (before the N rule)."""
    spans = []
    win = 0
    while win * WINDOW < length:
        s, e = win * WINDOW, min((win + 1) * WINDOW, length)
        if e - s < MIN_TAIL:
            if win == 0:
                spans.append((s, e))
            break
        spans.append((s, e))
        win += 1
        if single_window and win == 1:
            break
    return spans


_RC_TABLE = bytes.maketrans(b"ACTGNactgn", b"TGACNtgacn")


def reverse_complement(seq: bytes) -> bytes:
    """The reference's Sequence.rc() (sequence.py:41-43) on bytes: ACTGNactgn -> TGACNtgacn, every other byte (IUPAC codes,
    U / u, anything else) unchanged, then reversed."""
    return bytes(seq).translate(_RC_TABLE)[::-1]


def rc_spans(length: int, stride: int = WINDOW, single_window: bool = False) -> List[Tuple[int, int]]:
    """[start, end) in forward coordinates of every candidate window of the reverse complement of a stripped contig of
    `length` nt, before the N rule: candidate k of rc(S) is rc(S)[k * stride, k * stride + len_k), which is the forward
    segment [length - k * stride - len_k, length - k * stride)."""
    spans = profile_spans(length, stride)[:1] if single_window else profile_spans(length, stride)
    return [(length - e, length - s) for s, e in spans]


def profile_spans(length: int, stride: int) -> List[Tuple[int, int]]:
    """[start, end) of every candidate window of a stripped contig of `length` nt at window stride `stride` (1..6000), before
    the N rule: candidate k starts at k * stride and is min(6000, length - k * stride) long; the first is always a candidate,
    any other one only if it has >= 2500 nt.  There are 1 + max(0, (length - 2500) // stride) of them, and at stride 6000
    they are window_spans(length)."""
    if not 1 <= stride <= WINDOW:
        raise ValueError(f"window stride must be in [1, {WINDOW}], not {stride}")
    spans = []
    k = 0
    while k * stride < length:
        s, e = k * stride, min(k * stride + WINDOW, length)
        if k > 0 and e - s < MIN_TAIL:
            break
        spans.append((s, e))
        k += 1
    return spans


@dataclass
class EncodedFasta:
    names: np.ndarray        # [n_contigs] str    -- order of appearance (== rows of the outputs)
    contig_ids: np.ndarray   # [n_windows] int64  -- sorted, one per kept window
    offsets: np.ndarray      # [n_contigs + 1] int32 -- window range of each contig
    windows: np.ndarray      # [n_windows, 6000] uint8 -- upper-cased, N-padded ASCII


def encode_fasta_py(path, single_window: bool = False, out: Optional[np.ndarray] = None) -> EncodedFasta:
    """Pure-Python statement of encode_fasta (specification / cross-check for the native reader)."""
    names: List[str] = []
    ids: List[int] = []
    pieces: List[bytes] = []
    for cid, (header, seq) in enumerate(iter_fasta(path, strip_n=True)):
        names.append(accession(header))
        for wn, (s, e) in enumerate(window_spans(len(seq), single_window)):
            raw = seq[s:e]
            if wn > 0 and raw.count(b"N") > MAX_N:
                continue
            up = raw.upper()
            pieces.append(up if len(up) == WINDOW else up.ljust(WINDOW, b"N"))
            ids.append(cid)
    n = len(pieces)
    if out is not None:
        assert out.dtype == np.uint8 and out.shape[0] >= n and out.shape[1] == WINDOW
        win = out[:n]
        if n:
            win.reshape(-1)[:] = np.frombuffer(b"".join(pieces), dtype=np.uint8)
    else:
        win = (np.frombuffer(b"".join(pieces), dtype=np.uint8).reshape(n, WINDOW) if n
               else np.zeros((0, WINDOW), np.uint8))
    cid_arr = np.asarray(ids, dtype=np.int64)
    counts = np.bincount(cid_arr, minlength=len(names)) if n else np.zeros(len(names), np.int64)
    offsets = np.zeros(len(names) + 1, dtype=np.int32)
    np.cumsum(counts, out=offsets[1:])
    return EncodedFasta(np.array(names), cid_arr, offsets, win)


class ParsedFasta:
    """
    One native pass over a FASTA file (libgnm.so, csrc/fasta.cpp): answers check_fasta() and produces the window
    matrix without re-reading the file.  The analogue of check_fasta + generate_data()
    (reference sequence.py:124-131, nn_classification.py:54-82; the TFRecord round trip is gone).
    """

    def __init__(self, path, single_window: bool = False, threads: Optional[int] = None):
        import ctypes as C
        import os
        from . import engine
        self._lib = engine.load_library()
        avail = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
        self._threads = max(1, min(int(threads), avail, 32)) if threads else min(32, avail)    # --threads is honoured (32 saturate the reader)
        self._h = C.c_void_p()
        kind = is_compressed(path)
        if kind == Compression.uncompressed:
            self._text = None                               # mmap inside the library: the file is never copied
            rc = self._lib.gnm_fasta_open(str(path).encode(), int(bool(single_window)), self._threads, C.byref(self._h))
        elif kind == Compression.gzip:
            self._text = None                               # inflated natively (BGZF: block-parallel), owned by the library
            rc = self._lib.gnm_fasta_open_gz(str(path).encode(), int(bool(single_window)), self._threads, C.byref(self._h))
        else:
            self._text = read_bytes(path)                   # decompressed text, kept alive: the index points into it
            buf = self._text
            rc = self._lib.gnm_fasta_parse(C.cast(C.c_char_p(buf), C.c_void_p), len(buf), int(bool(single_window)),
                                           self._threads, C.byref(self._h))
        if rc != 0:
            raise RuntimeError(self._lib.gnm_fasta_last_error().decode())
        nrec, dup, nc, nw, hb = C.c_int64(), C.c_int(), C.c_int64(), C.c_int64(), C.c_int64()
        self._lib.gnm_fasta_info(self._h, C.byref(nrec), C.byref(dup), C.byref(nc), C.byref(nw), C.byref(hb))
        self.n_records, self.has_duplicate_ids = nrec.value, bool(dup.value)
        self.n_contigs, self.n_windows, self._header_bytes = nc.value, nw.value, hb.value

    def check(self) -> bool:
        """reference check_fasta(): at least one record and no repeated identifier."""
        return self.n_records > 0 and not self.has_duplicate_ids

    def encode(self, out: Optional[np.ndarray] = None) -> EncodedFasta:
        import ctypes as C
        n, nc = self.n_windows, self.n_contigs
        if out is not None:
            assert out.dtype == np.uint8 and out.shape[0] >= n and out.shape[1] == WINDOW and out.flags.c_contiguous
            win = out[:n]
        else:
            win = np.empty((n, WINDOW), dtype=np.uint8)
        offsets = np.zeros(nc + 1, dtype=np.int32)
        headers = C.create_string_buffer(max(1, self._header_bytes))
        rc = self._lib.gnm_fasta_export(self._h, win.ctypes.data if n else None, offsets.ctypes.data, headers, self._threads)
        if rc != 0:
            raise RuntimeError(self._lib.gnm_fasta_last_error().decode())
        lines = headers.raw[: self._header_bytes].decode("utf-8", errors="replace").split("\n")[:nc]
        names = np.array([accession(h) for h in lines]) if nc else np.array([], dtype="<U1")
        ids = np.repeat(np.arange(nc, dtype=np.int64), np.diff(offsets))
        return EncodedFasta(names, ids, offsets, win)

    def index(self) -> EncodedFasta:
        """Names, contig ids and offsets only (windows=None): what the driver needs before streaming the windows."""
        import ctypes as C
        nc = self.n_contigs
        offsets = np.zeros(nc + 1, dtype=np.int32)
        headers = C.create_string_buffer(max(1, self._header_bytes))
        rc = self._lib.gnm_fasta_export(self._h, None, offsets.ctypes.data, headers, self._threads)
        if rc != 0:
            raise RuntimeError(self._lib.gnm_fasta_last_error().decode())
        lines = headers.raw[: self._header_bytes].decode("utf-8", errors="replace").split("\n")[:nc]
        names = np.array([accession(h) for h in lines]) if nc else np.array([], dtype="<U1")
        ids = np.repeat(np.arange(nc, dtype=np.int64), np.diff(offsets))
        return EncodedFasta(names, ids, offsets, None)

    def export_windows(self, first: int, count: int, out: np.ndarray) -> np.ndarray:
        """Windows [first, first+count) of the global list -> out[:count] (uint8 [*, 6000], e.g. a pinned chunk)."""
        assert out.dtype == np.uint8 and out.shape[1] == WINDOW and out.shape[0] >= count and out.flags.c_contiguous
        if count:
            rc = self._lib.gnm_fasta_export_windows(self._h, int(first), int(count), out.ctypes.data, self._threads)
            if rc != 0:
                raise RuntimeError(self._lib.gnm_fasta_last_error().decode())
        return out[:count]

    def release_before(self, upto: int) -> None:
        """mmap mode: drop the file pages that precede global window `upto` from the resident set."""
        self._lib.gnm_fasta_release_before(self._h, int(upto))

    def spans(self) -> Tuple[np.ndarray, np.ndarray]:
        """Start (0-based, in the record's sequence before stripping) int64 and length (padding excluded) int32 of every window
        of the list export_windows() serves."""
        starts = np.empty(self.n_windows, dtype=np.int64)
        lengths = np.empty(self.n_windows, dtype=np.int32)
        if self.n_windows:
            rc = self._lib.gnm_fasta_spans(self._h, starts.ctypes.data, lengths.ctypes.data)
            if rc != 0:
                raise RuntimeError(self._lib.gnm_fasta_last_error().decode())
        return starts, lengths

    def windows(self, stride: int = WINDOW, single_window: bool = False, reverse: bool = False) -> "WindowList":
        """The window list at `stride` (1..6000) over this index (native, records on the reader threads).  At stride 6000 with
        this file's single_window it is the list export_windows() serves.  reverse: the same list made from every record's
        reverse complement (reverse_complement()); its export is reverse-complemented, its spans name forward segments."""
        return WindowList(self, stride, single_window, reverse)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.gnm_fasta_free(self._h)
            self._h = None
        self._text = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class WindowList:
    """
    Windows every `stride` nt of every kept record of a ParsedFasta (gnm_fasta_windows_*), or of every kept record's reverse
    complement (reverse=True): what the module streams for a score profile or for the reverse strand.  Same interface as ParsedFasta for the classifier's chunk loop (n_windows, export_windows,
    release_before), plus spans(): the CSR offsets per contig and each window's start (0-based, in the record's sequence
    before stripping) and length (padding excluded).  The ParsedFasta must stay open while the list is used.
    """

    def __init__(self, parsed: ParsedFasta, stride: int, single_window: bool = False, reverse: bool = False):
        import ctypes as C
        self._parsed, self._lib, self._threads = parsed, parsed._lib, parsed._threads
        self.stride = int(stride)
        self.reverse = bool(reverse)
        self._h = C.c_void_p()
        plan = self._lib.gnm_fasta_windows_plan_rc if self.reverse else self._lib.gnm_fasta_windows_plan
        rc = plan(parsed._h, self.stride, int(bool(single_window)), self._threads, C.byref(self._h))
        if rc != 0:
            raise RuntimeError(self._lib.gnm_fasta_last_error().decode())
        nc, nw = C.c_int64(), C.c_int64()
        self._lib.gnm_fasta_windows_info(self._h, C.byref(nc), C.byref(nw))
        self.n_contigs, self.n_windows = nc.value, nw.value

    def spans(self) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """(offsets int32 [n_contigs + 1], starts int64 [n_windows], lengths int32 [n_windows])."""
        offsets = np.zeros(self.n_contigs + 1, dtype=np.int32)
        starts = np.empty(self.n_windows, dtype=np.int64)
        lengths = np.empty(self.n_windows, dtype=np.int32)
        rc = self._lib.gnm_fasta_windows_spans(self._h, offsets.ctypes.data, starts.ctypes.data if self.n_windows else None,
                                               lengths.ctypes.data if self.n_windows else None)
        if rc != 0:
            raise RuntimeError(self._lib.gnm_fasta_last_error().decode())
        return offsets, starts, lengths

    def export_windows(self, first: int, count: int, out: np.ndarray) -> np.ndarray:
        """Windows [first, first+count) of this list -> out[:count] (uint8 [*, 6000])."""
        assert out.dtype == np.uint8 and out.shape[1] == WINDOW and out.shape[0] >= count and out.flags.c_contiguous
        if count:
            rc = self._lib.gnm_fasta_windows_export(self._h, int(first), int(count), out.ctypes.data, self._threads)
            if rc != 0:
                raise RuntimeError(self._lib.gnm_fasta_last_error().decode())
        return out[:count]

    def release_before(self, upto: int) -> None:
        self._lib.gnm_fasta_windows_release_before(self._h, int(upto))

    def close(self):
        if getattr(self, "_h", None):
            self._lib.gnm_fasta_windows_free(self._h)
            self._h = None
        self._parsed = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def encode_fasta(path, single_window: bool = False, out: Optional[np.ndarray] = None,
                 threads: Optional[int] = None) -> EncodedFasta:
    """FASTA -> dense window matrix (native)."""
    p = ParsedFasta(path, single_window, threads)
    try:
        return p.encode(out)
    finally:
        p.close()
