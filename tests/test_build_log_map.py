"""
CPU check of what ptxas made of the embedding-map kernels (no GPU): the build log (genomad_b200/build.log, `-Xptxas -v`) must
show no stack and no spills, and register counts within the caps (the warp-per-row kernels run 256-thread CTAs, the one-CTA
kernels 1024 threads, which allows at most 64 registers).
"""
import re

import pytest

from genomad_b200 import build as B

KERNELS = {   # mangled name: register cap
    "_ZN3gnm14mp_mean_kernelEPKfiiPd": 64,
    "_ZN3gnm15mp_sigma_kernelEPKfiiPKdPdS4_S4_": 64,
    "_ZN3gnm15mp_union_kernelEPKxPKdiiPd": 64,
    "_ZN3gnm19mp_normalize_kernelEPKfiPf": 80,
    "_ZN3gnm14mp_iota_kernelEiPxPi": 32,
    "_ZN3gnm13mp_eig_kernelEPKdPd": 64,
    "_ZN3gnm17mp_project_kernelEPKfiPKdS3_Pd": 64,
    "_ZN3gnm16mp_extent_kernelEPKdPKfxPd": 64,
    "_ZN3gnm15mp_noise_kernelEPKdiS1_jPf": 64,
    "_ZN3gnm17mp_rescale_kernelEPfiPKd": 64,
    "_ZN3gnm15mp_epoch_kernelEPKxPKiPKdiijfPK6float2PS6_": 64,
}


@pytest.fixture(scope="module")
def log() -> str:
    B.build()
    path = B.PKG / "build.log"
    assert path.exists(), "the library build writes build.log next to libgnm.so"
    return path.read_text()


@pytest.mark.parametrize("mangled", sorted(KERNELS))
def test_map_registers(log, mangled):
    m = re.search(r"Function properties for " + re.escape(mangled) + r"\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\n.*?Used (\d+) registers", log)
    assert m, f"no ptxas resource report for {mangled} in build.log"
    stack, stores, loads, regs = map(int, m.groups())
    assert stack == 0 and stores == 0 and loads == 0, f"{mangled}: stack {stack} B, spills {stores} / {loads} B"
    assert regs <= KERNELS[mangled], f"{mangled} uses {regs} registers, more than {KERNELS[mangled]}"
