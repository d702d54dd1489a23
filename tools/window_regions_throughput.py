"""
Time of the window-region decode on one H100 (a study, not part of bench.py), next to the time to classify the same windows,
with the card's name and power limit read in the same run.

  set      the seeded 10,000-contig set of tools/contig_throughput.py, windowed at stride 1000 and 100 by gnm_contig_windows_stride
           (~0.77 M and ~7.6 M windows), with seeded synthetic scores at C = 3 and C = 32 (the decode's cost does not depend on
           their values); kernel = one gnm_window_regions call over all windows (CUDA events), call = engine.window_regions
           (its device checks, whole-sequence calls within 1 GiB of workspace and the compaction; host clock after a
           synchronise)
  long     one 10 Mbp random sequence at stride 100 (~100 k windows in one warp: the serial worst case)
  module   window-regions (window_regions.main) on the stride-1000 windows file of the set, wall time
  classify Classifier.window_scores on the same contigs: measured at stride 1000 and for the 10 Mbp sequence; the stride-100
           figure is the stride-1000 rate (windows/s) applied to the stride-100 window count, as the per-window cost of the
           classifier does not depend on the stride

    python tools/window_regions_throughput.py [--reps 3] [--out DIR]   -> DIR/window_regions_h100.json (default: profiles/)
"""
from __future__ import annotations

import argparse
import json
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

L_MEAN = 30000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--contigs", type=int, default=10000)
    ap.add_argument("--out", type=Path, default=Path(__file__).resolve().parents[1] / "profiles")
    a = ap.parse_args()

    import torch
    from contig_throughput import card, make_contigs
    from genomad_b200 import engine, nn_classification as nnc, window_regions as WR
    if not torch.cuda.is_available():
        raise SystemExit("needs an H100")
    info = card()
    clf = engine.Classifier(None, device=0, max_batch=1024)
    lib = clf.lib
    seq_h, offs_h = make_contigs(a.contigs, 0)
    seq, offs = torch.from_numpy(seq_h).cuda(), torch.from_numpy(offs_h).cuda()

    def wall(fn, reps=a.reps):
        fn(); torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); ts.append(time.perf_counter() - t0)
        return float(np.median(ts))

    def kernel_ms(ws, stride, C):
        W = ws.probs.shape[0]
        need = int(lib.gnm_window_regions_workspace_bytes(W, C))
        work = torch.empty(need, dtype=torch.uint8, device="cuda")
        outs = [torch.empty((W, C), dtype=torch.float32, device="cuda"), torch.empty(W, dtype=torch.int32, device="cuda"),
                torch.empty(W, dtype=torch.uint8, device="cuda"), torch.empty(W, dtype=torch.int64, device="cuda"),
                torch.empty(W, dtype=torch.int64, device="cuda"), torch.empty(W, dtype=torch.int32, device="cuda"),
                torch.empty(W, dtype=torch.float32, device="cuda"), torch.empty((W, C), dtype=torch.float32, device="cuda")]
        stream = torch.cuda.current_stream().cuda_stream

        def run():
            engine._check(lib, lib.gnm_window_regions(ws.probs.data_ptr(), W, C, ws.offsets.data_ptr(), ws.offsets.numel() - 1,
                                                      ws.start.data_ptr(), ws.length.data_ptr(), stride, L_MEAN,
                                                      *[o.data_ptr() for o in outs], work.data_ptr(), need, stream))
        run()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ts = []
        for _ in range(a.reps):
            ev[0].record(); run(); ev[1].record(); torch.cuda.synchronize(); ts.append(ev[0].elapsed_time(ev[1]))
        del work, outs
        return float(np.median(ts))

    def profile(seq_t, offs_t, stride, C, seed):
        start, length, woff = clf.contig_windows(seq_t, offs_t, stride=stride)
        n = woff.numel() - 1
        contig = torch.repeat_interleave(torch.arange(n, dtype=torch.int32, device="cuda"), (woff[1:] - woff[:-1]).long())
        rel = start - offs_t[:-1].index_select(0, contig.long())
        g = torch.Generator(device="cuda").manual_seed(seed)
        p = torch.rand((start.numel(), C), generator=g, device="cuda") ** 4
        return engine.WindowScores(p / p.sum(1, keepdim=True), contig, rel, length, woff)

    rows = []
    for stride in (1000, 100):
        for C in (3, 32):
            ws = profile(seq, offs, stride, C, stride + C)
            W = ws.probs.shape[0]
            r = {"case": f"set s={stride} C={C}", "windows": W, "sequences": a.contigs,
                 "max_windows_per_sequence": int((ws.offsets[1:] - ws.offsets[:-1]).max()),
                 "kernel_ms": kernel_ms(ws, stride, C), "call_ms": 1e3 * wall(lambda: engine.window_regions(ws, stride, L_MEAN))}
            rows.append(r)
            print(json.dumps(r), flush=True)
            del ws
            torch.cuda.empty_cache()

    # classification of the same windows at stride 1000, measured once (about 10 s)
    t_cls = wall(lambda: clf.window_scores((seq, offs), 1000), reps=1)
    rate = rows[0]["windows"] / t_cls
    for r in rows:
        stride = int(r["case"].split("s=")[1].split()[0])
        r["classify_ms"] = 1e3 * (t_cls if stride == 1000 else r["windows"] / rate)
        r["classify_measured"] = stride == 1000
        r["call_share_of_classify"] = r["call_ms"] / r["classify_ms"]

    # one 10 Mbp sequence at stride 100
    rng = np.random.default_rng(1)
    long_h = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 10_000_000, dtype=np.uint8)].copy()
    lseq = torch.from_numpy(long_h).cuda()
    loff = torch.tensor([0, long_h.size], dtype=torch.int64, device="cuda")
    t_lcls = wall(lambda: clf.window_scores((lseq, loff), 100), reps=1)
    for C in (3, 32):
        ws = profile(lseq, loff, 100, C, 7 + C)
        r = {"case": f"10 Mbp s=100 C={C}", "windows": ws.probs.shape[0], "sequences": 1,
             "max_windows_per_sequence": ws.probs.shape[0], "kernel_ms": kernel_ms(ws, 100, C),
             "call_ms": 1e3 * wall(lambda: engine.window_regions(ws, 100, L_MEAN)), "classify_ms": 1e3 * t_lcls,
             "classify_measured": True}
        r["call_share_of_classify"] = r["call_ms"] / r["classify_ms"]
        r["kernel_us_per_window"] = r["kernel_ms"] * 1e3 / r["windows"]
        rows.append(r)
        print(json.dumps(r), flush=True)

    # the module on the stride-1000 windows file of the set (real classifier scores)
    ws = clf.window_scores((seq, offs), 1000)
    with tempfile.TemporaryDirectory() as d:
        d = Path(d)
        names = np.array([f"c{i}" for i in range(a.contigs)])
        npz = d / "set_nn_classification_windows.npz"
        nnc._write_window_scores(npz, d / "set_nn_classification_windows.tsv", "contig_names", names,
                                 ws.offsets.cpu().numpy(), ws.start.cpu().numpy(), ws.length.cpu().numpy(),
                                 ws.probs.cpu().numpy(), 1000, 8)
        t_mod = wall(lambda: WR.main(npz, d / "out", L_MEAN, verbose=False), reps=a.reps)
        n_regions = len(np.load(d / "out" / "set_nn_classification_regions.npz")["region_start"])
    rows.append({"case": "module s=1000 C=3", "windows": int(ws.probs.shape[0]), "sequences": a.contigs, "regions": n_regions,
                 "wall_ms": 1e3 * t_mod, "classify_ms": 1e3 * t_cls, "classify_measured": True,
                 "wall_share_of_classify": t_mod / t_cls})
    print(json.dumps(rows[-1]), flush=True)
    a.out.mkdir(parents=True, exist_ok=True)
    (a.out / "window_regions_h100.json").write_text(json.dumps({"card": info, "mean_region_length": L_MEAN, "rows": rows},
                                                               indent=1))
    clf.close()


if __name__ == "__main__":
    main()
