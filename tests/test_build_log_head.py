"""
CPU check of what ptxas made of the classifier-head kernels (csrc/head.cuh): no stack, no spills, and register counts within
the caps that keep their planned occupancy (build.log, `-Xptxas -v`).
"""
import re

import pytest

from genomad_b200 import build as B

KERNELS = {   # kernel name (as in the mangled symbol): register cap
    "head_split_tf32_kernel": 32, "head_softmax_kernel": 80, "head_segment_reduce_kernelILb0": 40,
    "head_segment_reduce_kernelILb1": 40, "head_gather_kernel": 32, "head_bn_forward_kernel": 64,
    "head_softmax_xent_kernel": 40, "head_loss_db2_kernel": 40, "head_transpose_w2_kernel": 32,
    "head_bn_backward_kernel": 64, "head_adam_kernel": 32,
}


@pytest.fixture(scope="module")
def log() -> str:
    B.build()
    return (B.PKG / "build.log").read_text()


@pytest.mark.parametrize("name", sorted(KERNELS))
def test_head_kernel_registers(log, name):
    m = re.search(r"Function properties for _ZN3gnm\d+" + re.escape(name) + r"\S*\n.*?(\d+) bytes stack frame, (\d+) bytes spill "
                  r"stores, (\d+) bytes spill loads\n.*?Used (\d+) registers", log)
    assert m, f"no ptxas resource report for {name} in build.log"
    stack, stores, loads, regs = map(int, m.groups())
    assert stack == 0 and stores == 0 and loads == 0, f"{name}: stack {stack} B, spills {stores} / {loads} B"
    assert regs <= KERNELS[name], f"{name} uses {regs} registers, more than {KERNELS[name]}"
