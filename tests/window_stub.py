"""
A CPU stand-in for the GPU classifier behind nn_classification's real chunk loop (_classify_parsed): per-window probabilities
that are a deterministic function of the window's bytes, gnm_segment_mean's fp32 running mean, and host buffers that need no
CUDA.  Used by the window-score tests, in one process and under gloo.
"""
import ctypes as C

import numpy as np
import torch

WINDOW = 6000


def stub_probs(win: np.ndarray) -> np.ndarray:
    """uint8 [m, 6000] -> float32 [m, 3], a function of every byte and its position."""
    x = (win.astype(np.float64) * np.cos(np.arange(WINDOW) * 0.001)).sum(1)
    return np.stack([np.sin(x) ** 2, np.cos(x) ** 2 / 3, 2 * np.cos(x) ** 2 / 3], 1).astype(np.float32)


def running_mean(probs: np.ndarray, offsets: np.ndarray) -> np.ndarray:
    """gnm_segment_mean: per contig, an fp32 running sum in window order divided by the count (zeros for no window)."""
    out = np.zeros((len(offsets) - 1, probs.shape[1]), np.float32)
    for c in range(len(offsets) - 1):
        a, b = int(offsets[c]), int(offsets[c + 1])
        if b > a:
            s = np.zeros(probs.shape[1], np.float32)
            for i in range(a, b):
                s = (s + probs[i]).astype(np.float32)
            out[c] = s / np.float32(b - a)
    return out


class StubClassifier:
    device = 0
    max_batch = 16

    def __init__(self):
        self.seen = []                  # every window handed to the classifier, in call order

    def classify_host_into(self, ascii_ptr: int, n: int, out_ptr: int):
        win = np.ctypeslib.as_array((C.c_uint8 * (n * WINDOW)).from_address(ascii_ptr)).reshape(n, WINDOW).copy()
        self.seen.append(win)
        out = np.ctypeslib.as_array((C.c_float * (n * 3)).from_address(out_ptr)).reshape(n, 3)
        out[:] = stub_probs(win)

    def segment_mean(self, probs, offsets):
        return torch.from_numpy(running_mean(probs.numpy(), offsets.numpy()))

    def windows_seen(self) -> np.ndarray:
        return np.concatenate(self.seen) if self.seen else np.zeros((0, WINDOW), np.uint8)


def install(setattr_, module, clf: StubClassifier) -> None:
    """Route module's classifier and host buffers to the stub (setattr_ is monkeypatch.setattr or plain setattr)."""
    setattr_(module, "_make_classifier", lambda batch_size, device: clf)
    setattr_(module, "_device", lambda c: torch.device("cpu"))
    setattr_(module, "_pinned_probs", lambda n: torch.empty((n, 3), dtype=torch.float32))

    def chunk(n):
        t = torch.empty((n, WINDOW), dtype=torch.uint8)
        return t, t.numpy()
    setattr_(module, "_pinned_chunk", chunk)
