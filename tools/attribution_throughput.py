"""
What attributions cost on one H100 (a study, not part of bench.py), in one run:

  rate     Classifier.attribute_ascii vs predict_ascii on the same device-resident windows, at attribution chunks of
           ATTR_MAX_BATCH (256) and 1024 (handle max_batch 1024), run alternately after a warm-up          windows/s
  kernels  summed kernel times of one call of each (torch.profiler, CUDA activity only): the backward stages next to the
           forward convs of the same session                                                               ms per call
  stages   the stage timer of one more attribution call: conv2 / conv3 of its forward steps next to conv3's and conv2's
           backward passes, each on its own                                                                ms per call

The probabilities of attribute_ascii are checked to be bitwise predict_ascii's.

    python tools/attribution_throughput.py [--windows 4096] [--seed 0] [--reps 3] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import sys
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
    """{kernel (with template arguments): ms} summed over one call of fn"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    tot = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            name = e.name.split("(")[0].replace("void ", "").replace("gnm::", "")
            tot[name] = tot.get(name, 0.0) + e.device_time / 1e3
    return dict(sorted(tot.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=4096)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", type=str, default="")
    a = ap.parse_args()

    import torch
    from contig_throughput import card
    from genomad_b200 import engine, synth
    if not torch.cuda.is_available():
        raise SystemExit("needs an H100")
    info = card()
    win = synth.windows_numpy(synth.subsample_indices(a.windows, 1_000_000, seed=a.seed), seed=a.seed)
    d_win = torch.from_numpy(win).cuda()
    sync = torch.cuda.synchronize
    res = {"card": info, "windows": a.windows, "bytes_per_window": int(engine.load_library().gnm_attr_bytes_per_window())}
    for amb in (engine.ATTR_MAX_BATCH, 1024):
        clf = engine.Classifier(None, device=0, max_batch=1024)
        clf._attr_ctx(amb)
        out = {}

        def fwd():
            out["p"] = clf.predict_ascii(d_win); sync()

        def att():
            out["pa"], out["x"] = clf.attribute_ascii(d_win, "virus"); sync()

        tf, ta = alternate(fwd, att, a.reps)
        clf.check_status()
        assert torch.equal(out["p"], out["pa"]), "attribute_ascii probabilities differ from predict_ascii"
        kf, ka = kernel_ms(fwd), kernel_ms(att)
        # per stage of the same attribution call (stage timer events): each conv backward pass next to the forward convs
        clf.set_option("profile_stages", 1)
        att()
        stages = {}
        for name, ms in clf.stage_times():
            stages[name] = stages.get(name, 0.0) + ms
        clf.set_option("profile_stages", 0)
        res[f"attr_max_batch_{amb}"] = {
            "predict_windows_per_s": a.windows / tf, "attribute_windows_per_s": a.windows / ta, "time_ratio": ta / tf,
            "kernels_ms_predict": kf, "kernels_ms_attribute": ka,
            "kernel_total_ms_predict": sum(kf.values()), "kernel_total_ms_attribute": sum(ka.values()),
            "stages_ms_attribute": stages,
        }
        print("    stages: " + ", ".join(f"{k} {stages.get(k, 0.0):.2f} ms" for k in
                                       ("conv2", "conv3", "attr_conv3_bwd", "attr_conv2_bwd", "attr_route1", "attr_route0",
                                        "attr_igloo1", "attr_igloo0", "attr_layer1_attr")))
        print(f"attr chunk {amb}: predict {a.windows / tf:,.0f} windows/s, attribute {a.windows / ta:,.0f} windows/s "
              f"({ta / tf:.2f}x); kernel sums {sum(kf.values()):.1f} / {sum(ka.values()):.1f} ms", flush=True)
        for k, v in list(ka.items())[:14]:
            print(f"    {v:8.2f} ms  {k}")
        clf.close()
        del clf
        torch.cuda.empty_cache()
    print(json.dumps(res["card"]))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
