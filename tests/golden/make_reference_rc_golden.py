#!/usr/bin/env python
"""
Golden vectors for the reverse strand: the reference's own read_fasta(strip_n=True), Sequence.rc(), seq_windows(6000, 2500), N
rule and ljust (genomad/sequence.py, genomad/modules/nn_classification.py:65-72), imported by path and run unmodified on
adversarial records, with and without --single-window.

    python tests/golden/make_reference_rc_golden.py     # needs the reference checkout; seconds -> reference_rc_golden.npz

The records: lower case, IUPAC codes in both cases, U / u, n / N runs at both ends; windows the N rule drops on one strand only
(and 'n' runs it must not count); lengths 1, 2499 / 2500 / 2501, 6000, 8499 / 8500 / 8501, 12,000 and longer; an all-N and an
empty record (dropped); CRLF line ends and irregular line lengths.  Stored: the FASTA text, and per mode (suffix "" or "_single")
the kept records' names, the CSR window offsets, the reverse windows' rows exactly as the reference builds them (rc, then
seq_windows, N rule, upper(), ljust to 6000 with N), and each window's forward segment (start 0-based in the record before
stripping, length), checked here against those rows.
"""
import importlib.util
import sys
import types
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
REF = Path("/root/reference/genomad")


def load_reference_sequence():
    pkg = types.ModuleType("genomad")
    pkg.__path__ = [str(REF)]
    sys.modules["genomad"] = pkg

    def load(name):
        spec = importlib.util.spec_from_file_location(f"genomad.{name}", REF / f"{name}.py")
        mod = importlib.util.module_from_spec(spec)
        sys.modules[f"genomad.{name}"] = mod
        spec.loader.exec_module(mod)
        setattr(pkg, name, mod)
        return mod
    load("utils")
    return load("sequence")


def records():
    """[(header, sequence str, line widths or None, crlf)]"""
    rng = np.random.default_rng(41)

    def rnd(n, alphabet="ACGT"):
        return "".join(np.array(list(alphabet))[rng.integers(0, len(alphabet), n)])
    out = []

    def add(name, s, widths=None, crlf=False):
        out.append((name, s, widths, crlf))
    mixed = rnd(8500, "ACGTacgtRYKMSWBDHVNrykmswbdhvnUuXx-*")
    add("mixed_case_iupac desc", mixed)
    add("len1", "a")
    for n in (2499, 2500, 2501, 6000, 8499, 8500, 8501, 12000, 12001, 14500):
        add(f"len{n}", rnd(n, "ACGTacgt"))
    add("n_runs_both_ends", "nnNNnN" + rnd(9000, "ACGTNacgtn") + "NnnNNN")
    s = list(rnd(12500))                                         # forward windows [0,6000) [6000,12000); reverse [6500,12500) [500,6500)
    s[6000:10500] = "N" * 4500
    add("n_rule_forward_only", "".join(s))
    s = list(rnd(12500))
    s[1000:5600] = "N" * 4600
    add("n_rule_reverse_only", "".join(s))
    s = list(rnd(12500))
    s[1000:5600] = "n" * 4600                                    # lower-case n: not counted
    add("n_rule_lowercase_n", "".join(s))
    s = list(rnd(31000, "ACGTacgt"))
    s[9000:13100] = "N" * 4100                                   # reverse window [13000,19000) keeps it, [7000,13000) drops
    s[20000:24300] = "N" * 4300
    add("long_many_windows", "".join(s), widths=[70, 61, 80, 3, 120])
    add("all_n", "NNNNnnnnNNNN")
    add("empty", "")
    add("crlf_irregular", rnd(17000, "ACGTNacgtnRYry"), widths=[59, 60, 1, 77, 200], crlf=True)
    add("crlf_regular", rnd(9100, "ACGTacgt"), widths=[60], crlf=True)
    add("n_edge_after_strip", "NN" + rnd(2499) + "N" * 3000 + rnd(4000) + "nn")
    return out


def fasta_text(recs) -> bytes:
    parts = []
    for name, s, widths, crlf in recs:
        eol = "\r\n" if crlf else "\n"
        lines, i, k = [], 0, 0
        w = widths or [60]
        while i < len(s):
            lines.append(s[i: i + w[k % len(w)]])
            i += w[k % len(w)]
            k += 1
        parts.append(f">{name}{eol}" + "".join(l + eol for l in lines))
    return "".join(parts).encode()


def main():
    seqmod = load_reference_sequence()
    recs = records()
    text = fasta_text(recs)
    raw = {name.split()[0]: s for name, s, _, _ in recs}
    path = HERE / "_rc_golden_input.fna"
    path.write_bytes(text)
    out = {"fasta": np.frombuffer(text, np.uint8)}
    try:
        for single, suffix in ((False, ""), (True, "_single")):
            names, offsets, rows, starts, lengths = [], [0], [], [], []
            for seq in seqmod.read_fasta(path, strip_n=True):
                names.append(seq.accession)
                rc = seq.rc()
                src = raw[seq.accession]
                lead = len(src) - len(src.lstrip("nN"))
                L = len(seq.seq)
                for k, win in enumerate(seqmod.seq_windows(rc, 6_000, 2_500, max_windows=1 if single else None)):
                    if k > 0 and win.count("N") > 4_000:
                        continue
                    row = win.seq_ascii.ljust(6_000, b"N")
                    n = min(6000, L - k * 6000)
                    a = L - k * 6000 - n                             # the forward segment of candidate k
                    assert len(win) == n and win.seq == seq.seq[a: a + n].translate(
                        str.maketrans("ACTGNactgn", "TGACNtgacn"))[::-1]
                    rows.append(np.frombuffer(row, np.uint8))
                    starts.append(lead + a)
                    lengths.append(n)
                offsets.append(len(rows))
            out["names" + suffix] = np.array(names)
            out["offsets" + suffix] = np.array(offsets, np.int32)
            out["windows" + suffix] = np.stack(rows)
            out["starts" + suffix] = np.array(starts, np.int64)
            out["lengths" + suffix] = np.array(lengths, np.int32)
    finally:
        path.unlink()
    dst = HERE / "reference_rc_golden.npz"
    np.savez_compressed(dst, **out)
    print(f"wrote {dst}: {len(out['names'])} records, {len(out['windows'])} / {len(out['windows_single'])} reverse windows")


if __name__ == "__main__":
    main()
