"""
Weight loading for the IGLOO1D classifier.

The reference loads ``genomad/data/nn_classifier.h5`` with Keras' legacy-H5 loader, which maps
weights to layers BY ORDER (reference genomad/modules/nn_classification.py:309-310,
genomad/_paths.py:20-22).  This module reads either that very file (through genomad_b200.h5lite,
no h5py) or the flat ``.npz`` exported from it by tools/export_weights.py, checks every shape, and
returns a dict of numpy arrays in Keras layouts keyed by short names.

Layer order in the file (root attr ``layer_names`` / group ``model`` attr ``weight_names``):
  conv1d, conv1d_1, conv1d_2, igloo1d_kernel, igloo1d_kernel_1, dense, batch_normalization,
  then dense_1, batch_normalization_1, dense_2 -- i.e. creation order in igloo.py:45-82 / model.py:28-44,
  so igloo1d_kernel sits on conv #1's output and igloo1d_kernel_1 on conv #3's.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import re
from pathlib import Path
from typing import Dict, NamedTuple, Optional, Tuple

import numpy as np

DEFAULT_NPZ = Path(__file__).resolve().parent / "data" / "nn_classifier.npz"

_ENC = "/model/"
KEYS = {
    "c1w": (_ENC + "conv1d/kernel:0", (6, 257, 128)), "c1b": (_ENC + "conv1d/bias:0", (128,)),
    "c2w": (_ENC + "conv1d_1/kernel:0", (6, 128, 128)), "c2b": (_ENC + "conv1d_1/bias:0", (128,)),
    "c3w": (_ENC + "conv1d_2/kernel:0", (6, 128, 128)), "c3b": (_ENC + "conv1d_2/bias:0", (128,)),
    "d0w": (_ENC + "dense/kernel:0", (256, 512)), "d0b": (_ENC + "dense/bias:0", (512,)),
    "bn0g": (_ENC + "batch_normalization/gamma:0", (512,)), "bn0b": (_ENC + "batch_normalization/beta:0", (512,)),
    "bn0m": (_ENC + "batch_normalization/moving_mean:0", (512,)),
    "bn0v": (_ENC + "batch_normalization/moving_variance:0", (512,)),
    "d1w": ("/dense_1/dense_1/kernel:0", (512, 512)), "d1b": ("/dense_1/dense_1/bias:0", (512,)),
    "bn1g": ("/batch_normalization_1/batch_normalization_1/gamma:0", (512,)),
    "bn1b": ("/batch_normalization_1/batch_normalization_1/beta:0", (512,)),
    "bn1m": ("/batch_normalization_1/batch_normalization_1/moving_mean:0", (512,)),
    "bn1v": ("/batch_normalization_1/batch_normalization_1/moving_variance:0", (512,)),
    "d2w": ("/dense_2/dense_2/kernel:0", (512, 3)), "d2b": ("/dense_2/dense_2/bias:0", (3,)),
}
for _s, _g in ((0, "igloo1d_kernel"), (1, "igloo1d_kernel_1")):
    KEYS[f"ig{_s}_w_mult"] = (f"{_ENC}{_g}/w_mult:0", (1, 2100, 4, 128))
    KEYS[f"ig{_s}_w_summer"] = (f"{_ENC}{_g}/w_summer:0", (1, 512, 1))
    KEYS[f"ig{_s}_w_bias"] = (f"{_ENC}{_g}/w_bias:0", (1, 2100))
    KEYS[f"ig{_s}_w_qk"] = (f"{_ENC}{_g}/w_qk:0", (2100, 749))
    KEYS[f"ig{_s}_w_v"] = (f"{_ENC}{_g}/w_v:0", (1, 128, 128))
    KEYS[f"ig{_s}_random_patches"] = (f"{_ENC}{_g}/random_patches:0", (2100, 4, 1))

EXPECTED_ORDER = ["conv1d", "conv1d_1", "conv1d_2", "igloo1d_kernel", "igloo1d_kernel_1", "dense",
                  "batch_normalization"]


def _validate(raw: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    out = {}
    for short, (path, shape) in KEYS.items():
        if path not in raw:
            raise KeyError(f"weight {path} missing")
        a = np.asarray(raw[path])
        if tuple(a.shape) != shape:
            raise ValueError(f"{path}: shape {a.shape}, expected {shape}")
        want = np.int32 if short.endswith("random_patches") else np.float32
        if a.dtype != want:
            raise ValueError(f"{path}: dtype {a.dtype}, expected {np.dtype(want)}")
        out[short] = np.ascontiguousarray(a)
    for s in (0, 1):
        p = out[f"ig{s}_random_patches"]
        if p.min() < 0 or p.max() >= 5997:
            raise ValueError("patch index out of range")
    return out


def load_weights(path=None) -> Dict[str, np.ndarray]:
    """Load from ``.npz`` (default: the copy shipped in genomad_b200/data) or from a Keras legacy ``.h5``."""
    p = Path(path) if path else DEFAULT_NPZ
    if p.suffix == ".npz":
        z = np.load(p)
        raw = {k: z[k] for k in z.files if k.startswith("/")}
        order = [str(x) for x in z["__weight_order__"]] if "__weight_order__" in z.files else None
    else:
        from .h5lite import H5File
        f = H5File(p)
        raw = dict(f.datasets)
        order = list(f.attrs["/"].get("layer_names") or []) + ["|"] + list(f.attrs.get("/model", {}).get("weight_names") or [])
    if order:
        enc = order[order.index("|") + 1:] if "|" in order else []
        seen = []
        for name in enc:
            layer = name.split("/")[0]
            if layer not in seen:
                seen.append(layer)
        if seen and seen != EXPECTED_ORDER:
            raise ValueError(f"unexpected encoder layer order {seen}; weights are matched to layers by order")
    return _validate(raw)


def to_c_struct(w: Dict[str, np.ndarray], Weights, IglooW, BnW):
    """Fill the ctypes mirror of ``gnm_weights`` (include/gnm.h) with host pointers into ``w``."""
    def ptr(k):
        return w[k].ctypes.data_as(C.c_void_p)
    cw = Weights()
    cw.conv1_kernel, cw.conv1_bias = ptr("c1w"), ptr("c1b")
    cw.conv2_kernel, cw.conv2_bias = ptr("c2w"), ptr("c2b")
    cw.conv3_kernel, cw.conv3_bias = ptr("c3w"), ptr("c3b")
    for s in (0, 1):
        g = IglooW()
        g.w_mult, g.w_summer, g.w_bias = ptr(f"ig{s}_w_mult"), ptr(f"ig{s}_w_summer"), ptr(f"ig{s}_w_bias")
        g.w_qk, g.w_v, g.patches = ptr(f"ig{s}_w_qk"), ptr(f"ig{s}_w_v"), ptr(f"ig{s}_random_patches")
        cw.igloo[s] = g
    cw.dense0_kernel, cw.dense0_bias = ptr("d0w"), ptr("d0b")
    cw.bn0 = BnW(ptr("bn0g"), ptr("bn0b"), ptr("bn0m"), ptr("bn0v"))
    cw.dense1_kernel, cw.dense1_bias = ptr("d1w"), ptr("d1b")
    cw.bn1 = BnW(ptr("bn1g"), ptr("bn1b"), ptr("bn1m"), ptr("bn1v"))
    cw.dense2_kernel, cw.dense2_bias = ptr("d2w"), ptr("d2b")
    return cw


# ------------------------------------------------------------------------------------------------ classifier heads
# A head file (.npz) holds the layers the reference trains on the frozen encoder (create_classifier, model.py:34-45) under the
# shipped file's names and layouts, with C classes instead of 3, plus `class_names` (C strings) and `encoder_sha256` (the
# encoder it was trained on).  INTEGRATION.md, "Head files".
HEAD_KEYS = ("d1w", "d1b", "bn1g", "bn1b", "bn1m", "bn1v", "d2w", "d2b")
HEAD_MIN_CLASSES, HEAD_MAX_CLASSES = 2, 32
SHIPPED_CLASSES = ("chromosome", "plasmid", "virus")
_CLASS_NAME = re.compile(r"[A-Za-z0-9_.-]+")


# A head file may also carry a novelty model (train-head --novelty; DESIGN.md, "Head novelty"): all four keys or none.
NOVELTY_KEYS = ("novelty_center", "novelty_whitening", "novelty_means", "novelty_calibration")


class HeadFile(NamedTuple):
    arrays: Dict[str, np.ndarray]   # short names of HEAD_KEYS -> float32 arrays; d2w [512, C], d2b [C]
    class_names: Tuple[str, ...]
    encoder_sha256: str
    novelty: Optional[Dict[str, np.ndarray]] = None   # NOVELTY_KEYS -> arrays (check_novelty), or None


def encoder_sha256(weights: Dict[str, np.ndarray]) -> str:
    """sha256 over the encoder arrays (every KEYS entry that is not a head layer), in KEYS order, as raw little-endian bytes."""
    h = hashlib.sha256()
    for short in KEYS:
        if short in HEAD_KEYS:
            continue
        a = np.asarray(weights[short])
        h.update(np.ascontiguousarray(a, dtype=a.dtype.newbyteorder("<")).tobytes())
    return h.hexdigest()


def check_class_names(names) -> Tuple[str, ...]:
    """C unique names matching [A-Za-z0-9_.-]+ with 2 <= C <= 32 (ValueError otherwise)."""
    names = tuple(str(x) for x in names)
    if not HEAD_MIN_CLASSES <= len(names) <= HEAD_MAX_CLASSES:
        raise ValueError(f"class_names: {len(names)} classes, a head has {HEAD_MIN_CLASSES} to {HEAD_MAX_CLASSES}")
    bad = [x for x in names if not _CLASS_NAME.fullmatch(x)]
    if bad:
        raise ValueError(f"class_names: {bad[0]!r} does not match [A-Za-z0-9_.-]+")
    dup = sorted({x for x in names if names.count(x) > 1})
    if dup:
        raise ValueError(f"class_names: {dup[0]!r} appears more than once")
    return names


def _check_head_arrays(arrays, C: int) -> Dict[str, np.ndarray]:
    out = {}
    for short in HEAD_KEYS:
        path, shape = KEYS[short]
        if short == "d2w":
            shape = (512, C)
        elif short == "d2b":
            shape = (C,)
        if short not in arrays:
            raise ValueError(f"{path} missing")
        a = np.asarray(arrays[short])
        if a.dtype != np.float32:
            raise ValueError(f"{path}: dtype {a.dtype}, expected float32")
        if tuple(a.shape) != shape:
            raise ValueError(f"{path}: shape {a.shape}, expected {shape}")
        if not np.isfinite(a).all():
            raise ValueError(f"{path}: not all finite")
        if short == "bn1v" and not (a + np.float32(1e-3) > 0).all():
            # inference folds 1 / sqrt(var + 1e-3) into the BN scale: NaN or infinite otherwise
            raise ValueError(f"{path}: moving variance + 1e-3 must be > 0 (unit {int(np.flatnonzero(~(a + np.float32(1e-3) > 0))[0])})")
        out[short] = np.ascontiguousarray(a)
    return out


def check_novelty(novelty, C: int) -> Dict[str, np.ndarray]:
    """The four novelty arrays, checked (ValueError naming the key): novelty_center float64 [512], novelty_whitening float64
    [512, 512] lower triangular with a positive diagonal, novelty_means float64 [C, 512] (the whitened class means),
    novelty_calibration float32 [n >= 1] sorted ascending; all finite."""
    missing = [k for k in NOVELTY_KEYS if k not in novelty]
    if missing:
        raise ValueError(f"{missing[0]} missing: a novelty model needs all of {', '.join(NOVELTY_KEYS)}")
    want = {"novelty_center": (np.float64, (512,)), "novelty_whitening": (np.float64, (512, 512)),
            "novelty_means": (np.float64, (C, 512)), "novelty_calibration": (np.float32, None)}
    out = {}
    for key in NOVELTY_KEYS:
        a = np.asarray(novelty[key])
        dtype, shape = want[key]
        if a.dtype != dtype:
            raise ValueError(f"{key}: dtype {a.dtype}, expected {np.dtype(dtype)}")
        if shape is not None and tuple(a.shape) != shape:
            raise ValueError(f"{key}: shape {a.shape}, expected {shape}")
        if shape is None and (a.ndim != 1 or a.size < 1):
            raise ValueError(f"{key}: shape {a.shape}, expected [n] with n >= 1")
        if not np.isfinite(a).all():
            raise ValueError(f"{key}: not all finite")
        out[key] = np.ascontiguousarray(a)
    w = out["novelty_whitening"]
    if np.triu(w, 1).any():
        raise ValueError("novelty_whitening: not lower triangular")
    if not (np.diagonal(w) > 0).all():
        raise ValueError(f"novelty_whitening: diagonal not positive at {int(np.flatnonzero(~(np.diagonal(w) > 0))[0])}")
    if (np.diff(out["novelty_calibration"]) < 0).any():
        raise ValueError("novelty_calibration: not sorted ascending")
    return out


def load_head(path, weights: Dict[str, np.ndarray]) -> HeadFile:
    """Read and validate a head file against the encoder `weights` (load_weights()); ValueError naming the offending key."""
    with np.load(Path(path), allow_pickle=False) as z:
        files = set(z.files)
        for key in ("class_names", "encoder_sha256"):
            if key not in files:
                raise ValueError(f"{key} missing")
        names = z["class_names"]
        if names.ndim != 1 or names.dtype.kind != "U":
            raise ValueError(f"class_names: expected a 1-D array of strings, not {names.dtype} {names.shape}")
        names = check_class_names(names.tolist())
        sha = z["encoder_sha256"]
        if sha.dtype.kind != "U" or sha.ndim != 0:
            raise ValueError("encoder_sha256: expected one string")
        sha = str(sha)
        arrays = _check_head_arrays({s: z[KEYS[s][0]] for s in HEAD_KEYS if KEYS[s][0] in files}, len(names))
        novelty = None
        if any(k in files for k in NOVELTY_KEYS):
            novelty = check_novelty({k: z[k] for k in NOVELTY_KEYS if k in files}, len(names))
    if sha != encoder_sha256(weights):
        raise ValueError("encoder_sha256: the head was trained on another encoder than the one loaded")
    return HeadFile(arrays, names, sha, novelty)


def save_head(path, arrays: Dict[str, np.ndarray], class_names, weights: Dict[str, np.ndarray], novelty=None) -> None:
    """Write a head file, with the novelty model's four keys after the others when `novelty` is given.  The zip members carry
    a fixed timestamp, so equal heads give byte-identical files."""
    import zipfile
    names = check_class_names(class_names)
    arrays = _check_head_arrays(arrays, len(names))
    members = [(KEYS[s][0], arrays[s]) for s in HEAD_KEYS]
    members += [("class_names", np.array(names, dtype=f"<U{max(len(x) for x in names)}")),
                ("encoder_sha256", np.array(encoder_sha256(weights)))]
    if novelty is not None:
        novelty = check_novelty(novelty, len(names))
        members += [(k, novelty[k]) for k in NOVELTY_KEYS]
    with zipfile.ZipFile(Path(path), "w", compression=zipfile.ZIP_STORED) as zf:
        for name, a in members:
            with zf.open(zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), "w", force_zip64=True) as f:
                np.lib.format.write_array(f, np.asarray(a), allow_pickle=False)


def shipped_head(weights: Dict[str, np.ndarray]) -> HeadFile:
    """The shipped classifier's own head (chromosome, plasmid, virus) as a head: the reference point of the head path."""
    return HeadFile({s: np.ascontiguousarray(weights[s], dtype=np.float32) for s in HEAD_KEYS}, SHIPPED_CLASSES,
                    encoder_sha256(weights))


def initial_head(C: int, seed: int) -> Dict[str, np.ndarray]:
    """Keras defaults for a new head, drawn with numpy.random.default_rng(seed): Glorot-uniform dense_1 then dense_2 kernels,
    zero biases, gamma 1, beta 0, moving mean 0, moving variance 1."""
    rng = np.random.default_rng(seed)

    def glorot(fan_in, fan_out):
        lim = np.sqrt(6.0 / (fan_in + fan_out))
        return rng.uniform(-lim, lim, (fan_in, fan_out)).astype(np.float32)
    d1w = glorot(512, 512)
    d2w = glorot(512, C)
    z, o = np.zeros(512, np.float32), np.ones(512, np.float32)
    return {"d1w": d1w, "d1b": z.copy(), "bn1g": o.copy(), "bn1b": z.copy(), "bn1m": z.copy(), "bn1v": o.copy(),
            "d2w": d2w, "d2b": np.zeros(C, np.float32)}


def head_c_struct(arrays: Dict[str, np.ndarray], HeadW, BnW):
    """Fill the ctypes mirror of ``gnm_head_weights`` (include/gnm.h) with host pointers into ``arrays``."""
    def ptr(k):
        return arrays[k].ctypes.data_as(C.c_void_p)
    hw = HeadW()
    hw.n_classes = int(arrays["d2b"].shape[0])
    hw.dense1_kernel, hw.dense1_bias = ptr("d1w"), ptr("d1b")
    hw.bn1 = BnW(ptr("bn1g"), ptr("bn1b"), ptr("bn1m"), ptr("bn1v"))
    hw.dense2_kernel, hw.dense2_bias = ptr("d2w"), ptr("d2b")
    return hw
