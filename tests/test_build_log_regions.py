"""
CPU check of what ptxas made of the window-region decode kernel (no GPU).  The build log (genomad_b200/build.log, `-Xptxas -v`)
must show no stack and no spills, and a register count within the cap: at 128 registers, the 3 CTAs of 128 threads that the
kernel's 68 KB of shared memory per CTA lets an SM hold still fit its register file.
"""
import re

import pytest

from genomad_b200 import build as B

KERNELS = {   # mangled name: register cap
    "_ZN3gnm16wr_decode_kernelENS_8WrParamsE": 128,
}


@pytest.fixture(scope="module")
def log() -> str:
    B.build()
    path = B.PKG / "build.log"
    assert path.exists(), "the library build writes build.log next to libgnm.so"
    return path.read_text()


@pytest.mark.parametrize("mangled", sorted(KERNELS))
def test_regions_registers(log, mangled):
    m = re.search(r"Function properties for " + re.escape(mangled) + r"\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\n.*?Used (\d+) registers", log)
    assert m, f"no ptxas resource report for {mangled} in build.log"
    stack, stores, loads, regs = map(int, m.groups())
    assert stack == 0 and stores == 0 and loads == 0, f"{mangled}: stack {stack} B, spills {stores} / {loads} B"
    assert regs <= KERNELS[mangled], f"{mangled} uses {regs} registers, more than {KERNELS[mangled]}"
