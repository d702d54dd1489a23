#!/usr/bin/env python
"""
Same-box A/B of library options: per-stage CUDA-event times and whole-step time at batch 1024 (device-resident windows).

    python tools/ab_stages.py fuse_gather=1 fuse_gather=0 [--batch 1024] [--steps 30] [--check]

Every positional argument is one configuration: comma-separated option=value pairs applied with gnm_set_option.
--check compares the probabilities of every configuration with the first one (max |dp|).
"""
import argparse
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from genomad_b200 import engine, synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("configs", nargs="*", default=["fuse_gather=1", "fuse_gather=0"])
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--steps-per-call", type=int, default=1, help="internal steps per API call (> 1 exercises the tail overlap)")
    ap.add_argument("--wvg-cycles", action="store_true", help="print the fused IGLOO kernel's per-CTA cycle breakdown (conv_experiment bit 512)")
    ap.add_argument("--wvg-exp", type=int, nargs="*", default=[0], help="timing-experiment bits to add to the cycle-counter runs (32 = no gather, 256 = gather reads only)")
    ap.add_argument("--wvg-fit", action="store_true", help="fit wv_split's unit cost model (wv_cost_base, wv_cost_group) to the per-CTA cycle counters")
    args = ap.parse_args()
    B = args.batch
    clf = engine.Classifier(None, device=0, max_batch=B)
    pool = [synth.windows_torch(1000 * i, B, 1, "cuda") for i in range(3)]
    out = torch.empty((B, 3), dtype=torch.float32, device="cuda")
    spc = max(1, args.steps_per_call)
    big = torch.cat([pool[i % 3] for i in range(spc)]) if spc > 1 else None
    big_out = torch.empty((spc * B, 3), dtype=torch.float32, device="cuda") if spc > 1 else None
    base = None
    for rep in range(2):                                       # two rounds: the second is at the settled clock
        for cfg in args.configs:
            for k in ("conv_experiment",):                       # options not named in a configuration are back at their defaults
                clf.set_option(k, 0)
            clf.set_option("fuse_gather", 1)
            clf.set_option("conv_cluster", 1)
            clf.set_option("tail_overlap", 1)
            for kv in cfg.split(","):
                k, v = kv.split("=")
                clf.set_option(k, int(v))
            for i in range(3):
                clf.predict_ascii(pool[i % 3], out)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            if spc > 1:
                for i in range(max(1, args.steps // spc)):
                    clf.predict_ascii(big, big_out)
                n_steps = max(1, args.steps // spc) * spc
            else:
                for i in range(args.steps):
                    clf.predict_ascii(pool[i % 3], out)
                n_steps = args.steps
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / n_steps
            clf.set_option("profile_stages", 1)
            for i in range(6):
                clf.predict_ascii(pool[i % 3], out)
            torch.cuda.synchronize()
            acc = {}
            for name, t in clf.stage_times():
                acc.setdefault(name, []).append(t)
            clf.set_option("profile_stages", 0)
            clf.check_status()
            line = "  ".join(f"{k}={sum(v) / len(v):.3f}" for k, v in acc.items())
            print(f"[round {rep}] {cfg}: {ms:.3f} ms/step = {B / ms * 1e3:,.0f} windows/s | {line}", flush=True)
            if args.check and rep == 0:
                pr = clf.predict_ascii(pool[0]).clone()
                if base is None:
                    base = pr
                else:
                    print(f"    max |dp| vs first configuration: {(pr - base).abs().max().item():.2e}", flush=True)
    if args.wvg_cycles:
        clf.set_option("fuse_gather", 1)
        for bits in args.wvg_exp:
            wvg_cycles(clf, pool, bits)
    if args.wvg_fit:
        clf.set_option("fuse_gather", 1)
        wvg_fit(clf, pool)


def wvg_cycles(clf, pool, bits=0):
    # counter layout: include/gnm.h, "conv_dbg"
    names = ["gather warp total", "gather warp wait a_full", "gather warp gather (reads + mma + release)", "MMA warpgroup MMA phase",
             "MMA warpgroup wait a_full", "units", "MMA warpgroup epilogue", "producer wait a_empty"]
    clf.set_option("conv_experiment", 512 | bits)
    clf.predict_ascii(pool[0]); torch.cuda.synchronize()
    d = clf.debug_fetch("conv_dbg", 1).cpu().view(torch.int64).numpy().astype(float)
    clf.set_option("conv_experiment", 0)
    units = max(d[:, 5].mean(), 1)
    print(f"wv_gather_kernel (IGLOO#1) cycle breakdown, experiment bits {bits}, mean over CTAs (first gather warp, first MMA warpgroup, producer):")
    for i, nm in enumerate(names):
        print(f"   {nm:42s} {d[:, i].mean():12.0f}   per unit {d[:, i].mean() / units:9.0f}   (min {d[:, i].min():.0f}, max {d[:, i].max():.0f})")


def wvg_fit(clf, pool, reps=8):
    """Least-squares fit of a CTA's cycles to wv_split's cost model, cycles = a * units + b * (sum over its units of the groups of
    the band's busiest gather warp), over the CTAs of one IGLOO#1 launch; wv_cost_group = b / a with wv_cost_base = 1.  A CTA's
    units are a contiguous band-major range, so the counters' unit counts give every CTA's range."""
    import numpy as np
    sys.path.insert(0, str(ROOT / "tests"))
    from test_host_cpu import _pack_patches
    from oracle import igloo_model as M
    w = M.load_npz_weights(ROOT / "genomad_b200" / "data" / "nn_classifier.npz")
    o = _pack_patches(w["ig1_random_patches"].reshape(2100, 4), w["ig1_w_mult"].reshape(2100, 4, 128), w["ig1_w_summer"].reshape(512))
    per_warp = (np.diff(o["band_first"]) + 6) // 7                     # groups of the busiest of the 7 gather warps, per band
    clf.set_option("conv_experiment", 512)
    d = 0
    for i in range(reps):                                             # back-to-back launches, counters averaged
        clf.predict_ascii(pool[i % len(pool)]); torch.cuda.synchronize()
        d = d + clf.debug_fetch("conv_dbg", 1).cpu().view(torch.int64).numpy().astype(float) / reps
    clf.set_option("conv_experiment", 0)
    n_units = pool[0].shape[0] // 8 * len(per_warp)
    units = np.rint(d[:, 5]).astype(np.int64)
    d = d[units > 0]
    start = np.concatenate([[0], np.cumsum(units)])[:-1][units > 0]
    units = units[units > 0]
    assert start[-1] + units[-1] == n_units, "the counters do not cover every unit"
    groups = n_units // len(per_warp)
    gsum = np.array([per_warp[np.arange(s, s + u) // groups].sum() for s, u in zip(start, units)], float)
    x = np.stack([units, gsum], 1).astype(float)
    (a, b), *_ = np.linalg.lstsq(x, d[:, 0], rcond=None)
    resid = d[:, 0] - x @ np.array([a, b])
    print(f"wv_split cost fit over {len(units)} CTAs: cycles = {a:.0f} x units + {b:.0f} x busiest-warp groups "
          f"(rms residual {np.sqrt(np.mean(resid ** 2)):.0f} of a mean {d[:, 0].mean():.0f}); "
          f"wv_cost_group / wv_cost_base = {b / a:.3f}")


if __name__ == "__main__":
    main()
