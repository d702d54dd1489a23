"""
CPU check of what ptxas made of the novelty-attribution kernels (no GPU).  The build log (genomad_b200/build.log,
`-Xptxas -v`) must show no stack and no spills, and a register count within the cap.  The two DMMA kernels (128 threads) hold
a warp's 32 x 32 block of fp64 accumulators (64 registers) plus a k16 step's fragments, capped at 168 like nv_score_kernel,
whose mainloop nv_residual_kernel shares: 3 CTAs of 128 threads still fit an SM's register file.  nv_residual_kernel sits at
exactly 168 (its store epilogue keeps the target's row pointers live next to the accumulators; nv_score_kernel uses 155), so a
toolchain change may trip this cap: above it, occupancy drops to 2 CTAs, which the score kernel's shared memory already
imposes on it, so the cap is kept as the point where that should be looked at, not raised.  The gather and the per-window
backward stage are plain loops, capped at 64.
"""
import re

import pytest

from genomad_b200 import build as B

KERNELS = {   # mangled name: register cap
    "_ZN3gnm18nv_residual_kernelEPKfiPKdS3_S3_PKiPd": 168,
    "_ZN3gnm14nv_grad_kernelEPKdiS1_Pf": 168,
    "_ZN3gnm14nv_pick_kernelEPKfiiiPKiiPf": 64,
    "_ZN3gnm28attr_novelty_backward_kernelEPKfS1_S1_S1_Pf": 64,
}


@pytest.fixture(scope="module")
def log() -> str:
    B.build()
    path = B.PKG / "build.log"
    assert path.exists(), "the library build writes build.log next to libgnm.so"
    return path.read_text()


@pytest.mark.parametrize("mangled", sorted(KERNELS))
def test_novelty_attr_registers(log, mangled):
    m = re.search(r"Function properties for " + re.escape(mangled) + r"\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\n.*?Used (\d+) registers", log)
    assert m, f"no ptxas resource report for {mangled} in build.log"
    stack, stores, loads, regs = map(int, m.groups())
    assert stack == 0 and stores == 0 and loads == 0, f"{mangled}: stack {stack} B, spills {stores} / {loads} B"
    assert regs <= KERNELS[mangled], f"{mangled} uses {regs} registers, more than {KERNELS[mangled]}"
