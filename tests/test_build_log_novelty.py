"""
CPU check of what ptxas made of the head-novelty kernels (no GPU).  The build log (genomad_b200/build.log, `-Xptxas -v`) must
show no stack and no spills, and a register count within the cap.  The two DMMA kernels (128 threads) hold a warp's 32 x 32
block of fp64 accumulators (64 registers) plus the A and B fragments of a k16 step: at 168 registers, 3 CTAs of 128 threads
still fit an SM's register file (65,536 / 384 = 170), and the score kernel's 87 KB of shared memory allows only 2 per SM anyway,
so registers never bound their occupancy.  The other kernels are plain fp64 loops, capped at 64.
"""
import re

import pytest

from genomad_b200 import build as B

KERNELS = {   # mangled name: register cap
    "_ZN3gnm15nv_score_kernelEPKfiPKdS3_S3_iPf": 168,
    "_ZN3gnm17nv_scatter_kernelEPKflPKlPKiliPKdPdPNS_8NvStatusE": 168,
    "_ZN3gnm20nv_class_sums_kernelEPKflPKlPKiliPdPxPNS_8NvStatusE": 64,
    "_ZN3gnm15nv_means_kernelEPKdPKxiilPdS4_PxPNS_8NvStatusE": 64,
    "_ZN3gnm24nv_scatter_reduce_kernelEPKdilPd": 64,
    "_ZN3gnm16nv_factor_kernelEPKdPdPNS_8NvStatusE": 64,
    "_ZN3gnm17nv_inverse_kernelEPKdPdPKNS_8NvStatusE": 64,
    "_ZN3gnm22nv_whiten_means_kernelEPKdS1_S1_PdPKNS_8NvStatusE": 64,
}


@pytest.fixture(scope="module")
def log() -> str:
    B.build()
    path = B.PKG / "build.log"
    assert path.exists(), "the library build writes build.log next to libgnm.so"
    return path.read_text()


@pytest.mark.parametrize("mangled", sorted(KERNELS))
def test_novelty_registers(log, mangled):
    m = re.search(r"Function properties for " + re.escape(mangled) + r"\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\n.*?Used (\d+) registers", log)
    assert m, f"no ptxas resource report for {mangled} in build.log"
    stack, stores, loads, regs = map(int, m.groups())
    assert stack == 0 and stores == 0 and loads == 0, f"{mangled}: stack {stack} B, spills {stores} / {loads} B"
    assert regs <= KERNELS[mangled], f"{mangled} uses {regs} registers, more than {KERNELS[mangled]}"
