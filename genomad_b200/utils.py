"""
Small host utilities of the nn-classification module: console + log file, md5, execution-info JSON,
restart comparison, find-proviruses detection.  Behavioural mirror of the helpers the reference module
uses (reference genomad/utils.py:42-123, 216-297); written against the standard library only.
"""
from __future__ import annotations

import hashlib
import json
import os
import re
import sys
from datetime import datetime, timezone
from pathlib import Path
from typing import Iterable, Optional

from ._paths import NNOutputs

_MARKUP = re.compile(r"\[/?[a-zA-Z#][^\[\]]*\]")


def _plain(msg: str) -> str:
    """Drop rich-style markup such as [green]...[/green] (the reference logs through rich)."""
    return _MARKUP.sub("", msg)


class HybridConsole:
    """
    Timestamped messages to stdout (silent when verbose=False) AND to an append-mode log file that is
    deleted when the console is created; errors go to stderr and the log (reference utils.py:42-123).
    """

    def __init__(self, output_file: Optional[Path] = None, verbose: bool = True):
        self.output_file = Path(output_file) if output_file else None
        self.verbose = verbose
        if self.output_file and self.output_file.exists():
            self.output_file.unlink()

    @staticmethod
    def _stamp() -> str:
        return datetime.now().strftime("[%X]")

    def _write_file(self, line: str) -> None:
        if self.output_file is None:
            return
        with open(self.output_file, "a") as fout:
            fout.write(line + "\n")

    def print(self, msg: str = "") -> None:
        text = _plain(msg)
        if self.verbose:
            print(text, flush=True)
        self._write_file(text)

    def log(self, msg: str, **_ignored) -> None:
        line = f"{self._stamp()} {_plain(msg)}"
        if self.verbose:
            print(line, flush=True)
        self._write_file(line)

    warning = log

    def error(self, msg: str) -> None:
        line = f"{self._stamp()} {_plain(msg)}"
        print(line, file=sys.stderr, flush=True)
        self._write_file(line)


_MD5_CACHE: dict = {}
_MD5_PENDING: dict = {}


def _md5_key(path):
    st = os.stat(path)
    return (str(Path(path).resolve()), st.st_size, st.st_mtime_ns)


def start_md5(path) -> None:
    """Begin hashing `path` on a helper thread (hashlib releases the GIL); get_md5() joins it."""
    import threading
    key = _md5_key(path)
    if key in _MD5_CACHE or key in _MD5_PENDING:
        return
    box = {}
    t = threading.Thread(target=lambda: box.setdefault("v", _md5_uncached(path)), daemon=True)
    t.start()
    _MD5_PENDING[key] = (t, box)


def get_md5(path, size: int = 1 << 20) -> str:
    """md5 of a file; memoised on (path, size, mtime) -- the reference re-hashes the input up to three times per run."""
    key = _md5_key(path)
    if key in _MD5_CACHE:
        return _MD5_CACHE[key]
    if key in _MD5_PENDING:
        t, box = _MD5_PENDING.pop(key)
        t.join()
        _MD5_CACHE[key] = digest = box["v"]
        return digest
    _MD5_CACHE[key] = digest = _md5_uncached(path, size)
    return digest


def _md5_uncached(path, size: int = 1 << 20) -> str:
    m = hashlib.md5()
    with open(path, "rb") as fin:
        while True:
            b = fin.read(size)
            if not b:
                break
            m.update(b)
    return m.hexdigest()


def get_n_available_cpus() -> int:
    try:
        return len(os.sched_getaffinity(0))
    except (AttributeError, OSError):
        return os.cpu_count() or 1


def write_execution_info(module_name: str, input_file: Path, parameters: dict, output_file: Path) -> None:
    """Same JSON keys as the reference (utils.py:238-254); aggregated-classification cross-checks input_md5."""
    info = {
        "module": module_name,
        "input": Path(input_file).name,
        "input_md5": get_md5(input_file),
        "start_time": datetime.now(timezone.utc).astimezone().isoformat(),
        "parameters": parameters,
    }
    with open(output_file, "w") as fout:
        fout.write(json.dumps(info, indent=4) + "\n")


def get_execution_info(path: Path):
    with open(path) as fin:
        info = json.load(fin)
    return info["input_md5"], info["module"], info["parameters"]


def compare_executions(input_file: Path, parameters: dict, execution_info_file: Path) -> bool:
    prev_md5, _, prev_params = get_execution_info(execution_info_file)
    return parameters == prev_params and get_md5(input_file) == prev_md5


def check_provirus_execution(prefix: str, input_file: Path, output_dir: Path) -> bool:
    """True iff find-proviruses ran on this very input and reported >= 1 provirus (utils.py:280-297)."""
    out = NNOutputs(prefix, Path(output_dir))
    if not out.find_proviruses_execution_info.exists():
        return False
    prev_md5, *_ = get_execution_info(out.find_proviruses_execution_info)
    if get_md5(input_file) != prev_md5:
        return False
    required = [out.find_proviruses_output, out.find_proviruses_nucleotide_output,
                out.find_proviruses_proteins_output, out.find_proviruses_genes_output]
    if not all(p.exists() for p in required):
        return False
    with open(out.find_proviruses_output) as fin:
        next(fin, None)
        return any(True for _ in fin)


def display_header(console: HybridConsole, version: str, module_name: str, description: str, output_dir: Path,
                   files: Iterable[Path], descriptions: Iterable[str]) -> None:
    console.print(f"Executing geNomad {module_name} (H100 build v{version}). {description}")
    console.print("Outputs:")
    console.print(f"  {output_dir}")
    for f, d in zip(files, descriptions):
        console.print(f"    {Path(f).name} ({d})")
