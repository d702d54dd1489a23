"""
CPU stand-ins for the classifier-head objects behind the real module code (nn_classification --head, train-head): a head whose
probabilities are a deterministic function of each embedding row, with gnm_head_segment_*'s fp32 running sums, and a trainer
that records every step it is given.  Used with tests/window_stub.py's classifier, in one process and under gloo.
"""
import numpy as np
import torch

import window_stub as WS
from genomad_b200 import weights as W


def stub_head_probs(emb: np.ndarray, C: int) -> np.ndarray:
    """float32 [n, 512] -> float32 [n, C]: a softmax of a fixed projection of the row."""
    proj = np.cos(np.arange(512 * C, dtype=np.float64).reshape(512, C) * 0.37)
    z = emb.astype(np.float64) @ proj * 0.05
    z -= z.max(1, keepdims=True)
    e = np.exp(z)
    return (e / e.sum(1, keepdims=True)).astype(np.float32)


def running_sum(probs: np.ndarray, offsets: np.ndarray) -> np.ndarray:
    """gnm_head_segment_sum: per contig, fp32 running sums in window order, then the window count."""
    C = probs.shape[1]
    out = np.zeros((len(offsets) - 1, C + 1), np.float32)
    for c in range(len(offsets) - 1):
        a, b = int(offsets[c]), int(offsets[c + 1])
        s = np.zeros(C, np.float32)
        for i in range(a, b):
            s = (s + probs[i]).astype(np.float32)
        out[c, :C], out[c, C] = s, b - a
    return out


class StubHead:
    def __init__(self, clf, head_file):
        self.class_names = tuple(head_file.class_names)
        self.n_classes = len(self.class_names)

    def predict(self, embeddings, out=None):
        p = torch.from_numpy(stub_head_probs(embeddings.numpy(), self.n_classes))
        if out is None:
            return p
        out.copy_(p)
        return out

    def segment_mean(self, probs, offsets):
        return torch.from_numpy(WS.running_mean(probs.numpy(), offsets.numpy()))

    def segment_sum(self, probs, offsets):
        return torch.from_numpy(running_sum(probs.numpy(), offsets.numpy()))

    def close(self):
        pass


class StubTrainer:
    """Records (X, idx, labels of the rows) of every step; the parameters stay the initial ones."""

    def __init__(self, init, device, max_batch, seed, learning_rate):
        self.init, self.max_batch, self.seed = init, max_batch, seed
        self.steps = []

    def step(self, X, idx, labels, class_weights, loss=None):
        assert idx.numel() <= self.max_batch
        self.X, self.cw = X, class_weights.clone()
        self.steps.append((idx.clone().numpy(), labels[idx].clone().numpy()))
        if loss is not None:
            loss.fill_(0.5)
        return loss

    def weights(self):
        return {k: v.copy() for k, v in self.init.items()}

    def close(self):
        pass


def write_head(path, C: int, seed: int, names=None, weights=None):
    """A C-class head file for the shipped encoder (or for `weights`)."""
    w = weights if weights is not None else W.load_weights()
    W.save_head(path, W.initial_head(C, seed), names or tuple(f"k{i}" for i in range(C)), w)
    return path
