#!/usr/bin/env python
"""Timing experiments on the conv kernel (results are intentionally wrong for experiment != 0)."""
import sys
from pathlib import Path
import torch
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from genomad_b200 import engine
sys.path.insert(0, str(Path(__file__).resolve().parent))
from gpu_diag import make_windows

n = 1024
clf = engine.Classifier(None, device=0, max_batch=n)
a = torch.from_numpy(make_windows(n)).cuda()
out = torch.empty((n, 3), dtype=torch.float32, device="cuda")
for exp in [int(x) for x in (sys.argv[1:] or ["0", "2"])]:
    # experiment 8: A "lo" operand replaced by the "hi" plane (normal fp16 numbers instead of subnormals)
    clf.set_option("conv_experiment", exp)
    for _ in range(2):
        clf.predict_ascii(a, out)
    clf.set_option("profile_stages", 1)
    for _ in range(5):
        clf.predict_ascii(a, out)
    torch.cuda.synchronize()
    acc = {}
    for name, ms in clf.stage_times():
        acc.setdefault(name, []).append(ms)
    clf.set_option("profile_stages", 0)
    print(f"experiment={exp}: " + "  ".join(f"{k}={sum(v)/len(v):.3f}" for k, v in acc.items()), flush=True)

# per-CTA cycle breakdown of the two consumer warpgroups (experiment bit 4 = conv3, bit 8 = conv2), layout in include/gnm.h;
# once as built and once with bit 2 (no epilogue global stores), which gives the epilogue's floor without its stores
names = ["wg1_total", "wg1_mma_phase", "wg1_wait_a_full", "wg1_wait_w_full", "units", "wg2_mma_phase", "wg1_epilogue",
         "wg2_epilogue"]
for extra, what in ((0, "with stores"), (2, "bit 2: no global stores")):
    for bit, label in ((8, "conv2"), (4, "conv3")):
        clf.set_option("conv_experiment", bit | extra)
        clf.predict_ascii(a, out); torch.cuda.synchronize()
        d = clf.debug_fetch("conv_dbg", 1).cpu().view(torch.int64).numpy().astype(float)
        print(f"conv_t cycle breakdown, {label}, {what} (mean over CTAs):")
        for i, nm in enumerate(names):
            print(f"   {nm:22s} {d[:, i].mean():12.0f}  (per unit {d[:, i].mean() / max(d[:, 4].mean(), 1):9.0f})")
clf.set_option("conv_experiment", 0)
