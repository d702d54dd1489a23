"""
CPU check of what ptxas made of the fused IGLOO kernel (no GPU).  The build log (genomad_b200/build.log, `-Xptxas -v`) must show
for wv_gather_kernel that the wgmma are not serialized (ptxas C7520), no spills, and a register count that fits its 512 threads
in one CTA per SM: the MMA warps hold 96 accumulator registers, so a spill or a lower cap would land in the MMA loop.
"""
import re

import pytest

from genomad_b200 import build as B

WV_GATHER = "_ZN3gnm16wv_gather_kernelE14CUtensorMap_stS0_NS_14WvGatherParamsE"


@pytest.fixture(scope="module")
def log() -> str:
    B.build()
    path = B.PKG / "build.log"
    assert path.exists(), "the library build writes build.log next to libgnm.so"
    return path.read_text()


def test_wv_gather_wgmma_not_serialized(log):
    serialized = [ln for ln in log.splitlines() if "C7520" in ln and WV_GATHER in ln]
    assert not serialized, serialized[0]


def test_wv_gather_registers(log):
    m = re.search(r"Function properties for " + re.escape(WV_GATHER) + r"\n.*?(\d+) bytes spill stores, (\d+) bytes spill loads"
                  r"\n.*?Used (\d+) registers", log)
    assert m, "no ptxas resource report for wv_gather_kernel in build.log"
    stores, loads, regs = map(int, m.groups())
    assert stores == 0 and loads == 0, f"wv_gather_kernel spills ({stores} B stored, {loads} B loaded)"
    assert regs <= 128, f"wv_gather_kernel uses {regs} registers; 512 threads per SM allow 128"
