"""
Throughput of the contig -> window path on one H100 (a study, not part of bench.py).

A seeded contig set shaped like BASELINE config 5 (lengths log-uniform on [1 kb, 500 kb]; runs of N and n, lower-case
stretches and stripped ends mixed in) is timed through

  plan     gnm_contig_windows on device-resident sequences (strip, candidate windows, N rule, CSR)   ms, ms per Gbp
  gather   gnm_gather_windows of one max_batch step                                                  ms per step
  contigs  Classifier.classify_contigs on device-resident sequences: plan + gnm_forward_windows + segment mean   windows/s
  ascii    gnm_forward_ascii on the same windows, gathered beforehand                                windows/s
  host     FASTA text in host memory -> gnm_fasta_parse -> gnm_fasta_export -> gnm_classify_host -> segment mean   windows/s

and the per-window probabilities of the first three paths are checked to be bitwise equal.

    python tools/contig_throughput.py [--contigs 10000] [--seed 0] [--reps 3] [--max-batch 1024] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def make_contigs(n: int, seed: int):
    """uint8 [total] + int64 offsets [n + 1]"""
    rng = np.random.default_rng(seed)
    lens = np.exp(rng.uniform(np.log(1000), np.log(500_000), n)).astype(np.int64)
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    seq = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, int(offs[-1]), dtype=np.uint8)]
    for c in range(n):
        a, L = int(offs[c]), int(lens[c])
        for _ in range(int(rng.integers(0, 3))):                     # N runs (some long enough to drop a window)
            s = a + int(rng.integers(0, L)); seq[s:min(a + L, s + int(rng.integers(10, 8000)))] = ord("N")
        if rng.random() < 0.3:                                        # a lower-case stretch
            s = a + int(rng.integers(0, L)); e = min(a + L, s + int(rng.integers(100, 20000)))
            seq[s:e] |= 32
        if rng.random() < 0.2:                                        # n/N at the ends
            k = min(L, int(rng.integers(1, 200))); seq[a:a + k] = ord("n"); seq[a + L - k:a + L] = ord("N")
    return seq, offs


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--contigs", type=int, default=10000)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-batch", type=int, default=1024)
    ap.add_argument("--out", type=str, default="")
    a = ap.parse_args()

    import torch
    from genomad_b200 import engine
    if not torch.cuda.is_available():
        raise SystemExit("needs an H100")
    seq_h, offs_h = make_contigs(a.contigs, a.seed)
    gbp = seq_h.size / 1e9
    clf = engine.Classifier(None, device=0, max_batch=a.max_batch)
    lib = clf.lib
    seq = torch.from_numpy(seq_h).cuda()
    offs = torch.from_numpy(offs_h).cuda()

    def timed(fn):
        """median wall time (s) of fn() followed by a device synchronise, after one warm-up call"""
        fn(); torch.cuda.synchronize()
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); ts.append(time.perf_counter() - t0)
        return float(np.median(ts))

    # plan
    plan = {}
    t_plan = timed(lambda: plan.update(r=clf.contig_windows(seq, offs)))
    start, length, woff = plan["r"]
    n_win = start.numel()

    # gather of one step
    stage = torch.empty((a.max_batch, engine.WINDOW), dtype=torch.uint8, device="cuda")
    m = min(a.max_batch, n_win)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    clf.lib.gnm_gather_windows(clf._h, seq.data_ptr(), start.data_ptr(), length.data_ptr(), m, stage.data_ptr(), clf._stream())
    steps = 20
    ev[0].record()
    for i in range(steps):
        k = (i * m) % max(1, n_win - m + 1)
        engine._check(lib, lib.gnm_gather_windows(clf._h, seq.data_ptr(), start[k:].data_ptr(), length[k:].data_ptr(), m,
                                                  stage.data_ptr(), clf._stream()))
    ev[1].record(); torch.cuda.synchronize()
    t_gather = ev[0].elapsed_time(ev[1]) / steps

    # classify_contigs (device-resident sequences) and forward_ascii on the same windows, pre-gathered
    res = {}
    t_contigs = timed(lambda: res.update(c=clf.classify_contigs((seq, offs), return_window_probs=True)))
    ascii_w = clf.gather_windows(seq, start, length)
    t_ascii = timed(lambda: res.update(a=clf.predict_ascii(ascii_w)))
    assert torch.equal(res["c"][2], res["a"]), "classify_contigs and forward_ascii differ"
    del ascii_w

    # host path: FASTA text in memory -> parse -> export -> classify_host -> segment mean
    text = b"".join(b">c%d\n%s\n" % (i, seq_h[offs_h[i]:offs_h[i + 1]].tobytes()) for i in range(a.contigs))
    threads = min(32, len(os.sched_getaffinity(0)))
    win_pinned = torch.empty((n_win + 1, engine.WINDOW), dtype=torch.uint8).pin_memory()
    probs_pinned = torch.empty((n_win + 1, 3), dtype=torch.float32).pin_memory()
    host = {}

    def host_path():
        f = C.c_void_p()
        buf = C.cast(C.c_char_p(text), C.c_void_p)
        if lib.gnm_fasta_parse(buf, len(text), 0, threads, C.byref(f)):
            raise RuntimeError(lib.gnm_fasta_last_error().decode())
        nw, nc = C.c_int64(), C.c_int64()
        lib.gnm_fasta_info(f, None, None, C.byref(nc), C.byref(nw), None)
        o = np.zeros(nc.value + 1, np.int32)
        rc = lib.gnm_fasta_export(f, win_pinned.data_ptr(), o.ctypes.data, None, threads)
        lib.gnm_fasta_free(f)
        assert rc == 0 and nw.value == n_win
        clf.classify_host_into(win_pinned.data_ptr(), nw.value, probs_pinned.data_ptr())
        host["p"] = probs_pinned[:nw.value]
        host["m"] = clf.segment_mean(probs_pinned[:nw.value].cuda(), torch.from_numpy(o).cuda())
    t_host = timed(host_path)
    assert torch.equal(host["p"].cuda(), res["a"]), "host path and forward_ascii differ"
    kept = (woff[1:] - woff[:-1]) > 0
    assert torch.equal(host["m"], res["c"][0][kept]), "per-contig means differ"
    clf.check_status()

    out = {
        "card": card(), "contigs": a.contigs, "seed": a.seed, "gbp": round(gbp, 4), "windows": n_win, "max_batch": a.max_batch,
        "plan_ms": round(t_plan * 1e3, 3), "plan_ms_per_gbp": round(t_plan * 1e3 / gbp, 3),
        "gather_ms_per_step": round(t_gather, 4), "gather_windows_per_step": m,
        "classify_contigs_windows_per_s": round(n_win / t_contigs), "forward_ascii_windows_per_s": round(n_win / t_ascii),
        "contigs_over_ascii": round(t_ascii / t_contigs, 4),
        "host_fasta_path_windows_per_s": round(n_win / t_host), "host_threads": threads,
    }
    print(json.dumps(out))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(out, indent=1) + "\n")
    clf.close()


if __name__ == "__main__":
    main()
