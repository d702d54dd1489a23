"""
CPU check of what ptxas made of the kernels of clustering through the index (no GPU): the build log (genomad_b200/build.log,
`-Xptxas -v`) must show no stack and no spills, and register counts within the caps (ivf_grow_search_kernel runs
ivf_search_kernel's 384-thread CTA, one per SM, so at most 168 registers; the others run 256-thread CTAs).  The grow search
kernel's wgmma must not be serialized (ptxas C7514 / C7520 name the kernel when they are).
"""
import re

import pytest

from genomad_b200 import build as B

KERNELS = {   # mangled name: register cap
    "_ZN3gnm15ivf_ends_kernelEPKxiPx": 32,
    "_ZN3gnm21ivf_grow_lists_kernelEPKjiPKxiPiPxS5_": 32,
    "_ZN3gnm22ivf_grow_search_kernelE14CUtensorMap_stS0_S0_S0_NS_15IvfSearchParamsE": 168,
    "_ZN3gnm21ivf_grow_merge_kernelEPKfPKiS3_S3_iS3_PKxiS3_S5_iiS5_PfPx": 64,
    "_ZN3gnm22cl_probe_filter_kernelEPjiiPKiiS2_": 32,
}


@pytest.fixture(scope="module")
def log() -> str:
    B.build()
    path = B.PKG / "build.log"
    assert path.exists(), "the library build writes build.log next to libgnm.so"
    return path.read_text()


@pytest.mark.parametrize("mangled", sorted(KERNELS))
def test_registers(log, mangled):
    m = re.search(r"Function properties for " + re.escape(mangled) + r"\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\n.*?Used (\d+) registers", log)
    assert m, f"no ptxas resource report for {mangled} in build.log"
    stack, stores, loads, regs = map(int, m.groups())
    assert stack == 0 and stores == 0 and loads == 0, f"{mangled}: stack {stack} B, spills {stores} / {loads} B"
    assert regs <= KERNELS[mangled], f"{mangled} uses {regs} registers, more than {KERNELS[mangled]}"


def test_grow_search_wgmma_not_serialized(log):
    mangled = "_ZN3gnm22ivf_grow_search_kernelE14CUtensorMap_stS0_S0_S0_NS_15IvfSearchParamsE"
    serialized = [ln for ln in log.splitlines() if ("C7520" in ln or "C7514" in ln) and mangled in ln]
    assert not serialized, serialized[0]
