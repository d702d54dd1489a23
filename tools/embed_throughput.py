"""
What writing the encoder embeddings costs on one H100 (a study, not part of bench.py).  Three A/B comparisons, each run
alternately (A B A B A B) after a warm-up, plus the per-contig reduction alone:

  device   Classifier.predict_ascii vs embed_ascii, device-resident windows, max_batch 1024     ms per 1024 windows;
           also the summed kernel times of one call of each (torch.profiler), which the power-capped clock disturbs less
  host     gnm_classify_host vs gnm_embed_host + segment_sum_rows, pinned host windows           windows/s
  module   nn_classification.main without / with write_embeddings on the seeded contig set of
           tools/contig_throughput.py written as FASTA (10,000 contigs, 0.80 Gbp)                 s
  segsum   gnm_segment_sum_rows over all windows of that set, per-contig segments               ms, GB/s

and the probabilities of the A and B sides are checked to be bitwise equal.

    python tools/embed_throughput.py [--contigs 10000] [--seed 0] [--reps 5] [--device-windows 16384] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))


def alternate(fa, fb, reps):
    """median seconds of fa() and fb(), run A B A B ... after one warm-up each; fn() must synchronise before it returns"""
    fa(); fb()
    ta, tb = [], []
    for _ in range(reps):
        t0 = time.perf_counter(); fa(); ta.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); fb(); tb.append(time.perf_counter() - t0)
    return float(np.median(ta)), float(np.median(tb))


def kernel_ms(fn):
    """{kernel: ms} summed over one call of fn (torch.profiler, CUDA activity only)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    tot = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            name = e.name.split("(")[0].split("<")[0].replace("void ", "").replace("gnm::", "")
            tot[name] = tot.get(name, 0.0) + e.device_time / 1e3
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--contigs", type=int, default=10000)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--device-windows", type=int, default=16384)
    ap.add_argument("--host-windows", type=int, default=32768)
    ap.add_argument("--out", type=str, default="")
    a = ap.parse_args()

    import torch
    from contig_throughput import card, make_contigs
    from genomad_b200 import engine, nn_classification, synth
    if not torch.cuda.is_available():
        raise SystemExit("needs an H100")
    info = card()                                                     # name, power limit and max SM clock in one query
    clf = engine.Classifier(None, device=0, max_batch=1024)
    sync = torch.cuda.synchronize
    res = {}

    # ---- device-resident, batch 1024
    win = synth.windows_numpy(synth.subsample_indices(a.device_windows, 1_000_000, seed=a.seed), seed=a.seed)
    d_win = torch.from_numpy(win).cuda()

    def dev_a():
        res["pa"] = clf.predict_ascii(d_win); sync()

    def dev_b():
        res["pb"], res["eb"] = clf.embed_ascii(d_win); sync()
    t_pa, t_pb = alternate(dev_a, dev_b, a.reps)
    assert torch.equal(res["pa"], res["pb"]), "embed_ascii changed the probabilities"
    del res["eb"]
    kern = {k: kernel_ms(f) for k, f in (("predict", dev_a), ("embed", dev_b))}

    # ---- host path
    n_h = a.host_windows
    h_win = torch.empty((n_h, engine.WINDOW), dtype=torch.uint8).pin_memory()
    h_win.numpy()[:] = np.resize(win, (n_h, engine.WINDOW))
    pa = torch.empty((n_h, 3), dtype=torch.float32).pin_memory()
    pb = torch.empty_like(pa).pin_memory()
    d_emb = torch.empty((n_h, 512), dtype=torch.float32, device="cuda")
    h_off = torch.arange(0, n_h + 1, 8, dtype=torch.int32, device="cuda")      # 8-window "contigs"

    def host_a():
        clf.classify_host_into(h_win.data_ptr(), n_h, pa.data_ptr())

    def host_b():
        clf.embed_host_into(h_win.data_ptr(), n_h, pb.data_ptr(), d_emb.data_ptr())
        clf.segment_sum_rows(d_emb, h_off); sync()
    t_ha, t_hb = alternate(host_a, host_b, a.reps)
    assert torch.equal(pa, pb), "gnm_embed_host changed the probabilities"
    del d_emb

    # ---- segment_sum_rows alone, over the contig set's windows
    seq_h, offs_h = make_contigs(a.contigs, a.seed)
    seq, offs = torch.from_numpy(seq_h).cuda(), torch.from_numpy(offs_h).cuda()
    start, length, woff = clf.contig_windows(seq, offs)
    n_w = start.numel()
    rows = torch.rand((n_w, 512), dtype=torch.float32, device="cuda")
    clf.segment_sum_rows(rows, woff); sync()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(10):
        clf.segment_sum_rows(rows, woff)
    ev[1].record(); sync()
    t_seg = ev[0].elapsed_time(ev[1]) / 10
    del rows, seq, offs, start, length

    # ---- module, with and without --write-embeddings
    threads = min(32, len(os.sched_getaffinity(0)))
    with tempfile.TemporaryDirectory() as tmp:
        fa = Path(tmp) / "set.fna"
        with open(fa, "wb") as fh:
            for i in range(a.contigs):
                fh.write(b">c%d\n%s\n" % (i, seq_h[offs_h[i]:offs_h[i + 1]].tobytes()))
        nn_classification._CLASSIFIERS[(0, clf.max_batch)] = clf           # the module reuses this classifier

        def mod(flag):
            def run():
                nn_classification.main(fa, Path(tmp) / f"out{int(flag)}", False, 1024, True, threads, False, False,
                                       write_embeddings=flag)
            return run
        t_ma, t_mb = alternate(mod(False), mod(True), a.reps)
        p0 = np.load(Path(tmp) / "out0" / "set_nn_classification" / "set_nn_classification.npz")["predictions"]
        p1 = np.load(Path(tmp) / "out1" / "set_nn_classification" / "set_nn_classification.npz")["predictions"]
        assert np.array_equal(p0, p1), "the module's predictions changed with --write-embeddings"
        nn_classification._CLASSIFIERS.clear()
    clf.check_status()

    out = {
        "card": info, "max_batch": 1024, "reps": a.reps,
        "device_windows": a.device_windows,
        "predict_ascii_ms_per_1024": round(t_pa * 1e3 * 1024 / a.device_windows, 3),
        "embed_ascii_ms_per_1024": round(t_pb * 1e3 * 1024 / a.device_windows, 3),
        "device_embed_over_predict": round(t_pb / t_pa, 4),
        "kernel_ms_per_1024": {k: round(sum(v.values()) * 1024 / a.device_windows, 3) for k, v in kern.items()},
        "dense_epilogue_ms_per_1024": {k: round(v.get("splitk_reduce_epi_kernel", 0.0) * 1024 / a.device_windows, 4)
                                       for k, v in kern.items()},
        "host_windows": n_h,
        "classify_host_windows_per_s": round(n_h / t_ha), "embed_host_segsum_windows_per_s": round(n_h / t_hb),
        "host_embed_over_classify": round(t_hb / t_ha, 4),
        "contigs": a.contigs, "gbp": round(seq_h.size / 1e9, 4), "windows": n_w,
        "module_s": round(t_ma, 3), "module_write_embeddings_s": round(t_mb, 3), "module_ratio": round(t_mb / t_ma, 4),
        "segment_sum_rows_ms": round(t_seg, 3), "segment_sum_rows_gb_per_s": round(n_w * 2048 / t_seg / 1e6, 1),
    }
    print(json.dumps(out))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(out, indent=1) + "\n")
    clf.close()


if __name__ == "__main__":
    main()
