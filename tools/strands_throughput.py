"""
Cost of the reverse strand on one H100 (a study, not part of bench.py), on the seeded contig set of tools/contig_throughput.py:

  gather   gnm_gather_windows_rc against gnm_gather_windows, one max_batch step each, CUDA events     ms per step
  steps    gnm_forward_windows_rc against gnm_forward_windows on all windows of each strand            windows/s
  module   nn-classification on the contigs as a FASTA file, without and with --both-strands, alternated  s
  export   the native reader's export of the reverse list against the forward list, on the reader threads   windows/s

The reverse probabilities are checked bitwise against gnm_forward_ascii on gnm_gather_windows_rc's rows.

    python tools/strands_throughput.py [--contigs 10000] [--seed 0] [--rounds 2] [--max-batch 1024] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from contig_throughput import card, make_contigs  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--contigs", type=int, default=10000)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--max-batch", type=int, default=1024)
    ap.add_argument("--out", type=str, default="")
    a = ap.parse_args()

    import torch
    from genomad_b200 import engine, nn_classification, sequence
    if not torch.cuda.is_available():
        raise SystemExit("needs an H100")
    seq_h, offs_h = make_contigs(a.contigs, a.seed)
    clf = engine.Classifier(None, device=0, max_batch=a.max_batch)
    lib = clf.lib
    seq = torch.from_numpy(seq_h).cuda()
    offs = torch.from_numpy(offs_h).cuda()
    out = {"card": card(), "contigs": a.contigs, "seed": a.seed, "gbp": round(seq_h.size / 1e9, 4), "max_batch": a.max_batch}

    # ---- gather: one step of each strand, 50 launches over different windows
    stage = torch.empty((a.max_batch, engine.WINDOW), dtype=torch.uint8, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for rev in (False, True):
        start, length, _ = clf.contig_windows(seq, offs, reverse=rev)
        n_win = start.numel()
        m = min(a.max_batch, n_win)
        fn = lib.gnm_gather_windows_rc if rev else lib.gnm_gather_windows
        for rep in range(2):                                               # the first round warms up
            ev[0].record()
            for i in range(50):
                k = (i * m) % max(1, n_win - m + 1)
                engine._check(lib, fn(clf._h, seq.data_ptr(), start[k:].data_ptr(), length[k:].data_ptr(), m,
                                      stage.data_ptr(), clf._stream()))
            ev[1].record(); torch.cuda.synchronize()
        key = "reverse" if rev else "forward"
        out[f"gather_{key}_ms_per_step"] = round(ev[0].elapsed_time(ev[1]) / 50, 4)
        out[f"windows_{key}"] = n_win
        # ---- the forward step straight from the sequence buffer
        clf.predict_windows(seq, start, length, reverse=rev); torch.cuda.synchronize()
        t0 = time.perf_counter()
        p = clf.predict_windows(seq, start, length, reverse=rev); torch.cuda.synchronize()
        out[f"forward_windows_{key}_windows_per_s"] = round(n_win / (time.perf_counter() - t0))
        if rev:
            rows = clf.gather_windows(seq, start, length, reverse=True)
            assert torch.equal(p, clf.predict_ascii(rows)), "gnm_forward_windows_rc differs from gnm_forward_ascii"
            del rows
    out["gather_reverse_over_forward"] = round(out["gather_reverse_ms_per_step"] / out["gather_forward_ms_per_step"], 3)
    clf.check_status()
    clf.close()
    del seq, offs, stage
    torch.cuda.empty_cache()

    # ---- the module on the contigs as a FASTA file, without and with --both-strands, alternated
    tmp = Path(tempfile.mkdtemp(prefix="strands_"))
    try:
        fa = tmp / "contigs.fna"
        with open(fa, "wb") as fh:
            for i in range(a.contigs):
                s = seq_h[offs_h[i]:offs_h[i + 1]].tobytes()
                fh.write(b">c%d\n" % i + b"\n".join(s[j:j + 80] for j in range(0, len(s), 80)) + b"\n")
        threads = min(32, len(os.sched_getaffinity(0)))
        times = {False: [], True: []}
        for r in range(a.rounds + 1):                                     # round 0 warms up (CUDA context, weights, page cache)
            for both in (False, True):
                d = tmp / f"out_{int(both)}"
                shutil.rmtree(d, ignore_errors=True)
                t0 = time.perf_counter()
                nn_classification.main(fa, d, False, 128, True, threads, False, False, both_strands=both)
                if r:
                    times[both].append(time.perf_counter() - t0)
        out["module_forward_s"] = [round(t, 3) for t in times[False]]
        out["module_both_strands_s"] = [round(t, 3) for t in times[True]]
        out["module_both_over_forward"] = round(float(np.median(times[True]) / np.median(times[False])), 3)
        out["module_threads"] = threads
        # ---- host export of each list on the reader threads (what feeds the GPU)
        pf = sequence.ParsedFasta(fa, threads=threads)
        for rev in (False, True):
            wl = pf.windows(6000, reverse=rev)
            buf = np.empty((min(wl.n_windows, 16384), 6000), np.uint8)
            t0 = time.perf_counter()
            for s in range(0, wl.n_windows, buf.shape[0]):
                wl.export_windows(s, min(buf.shape[0], wl.n_windows - s), buf)
            out[f"export_{'reverse' if rev else 'forward'}_windows_per_s"] = round(wl.n_windows / (time.perf_counter() - t0))
            wl.close()
        pf.close()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        nn_classification.release_classifiers()
    print(json.dumps(out))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
