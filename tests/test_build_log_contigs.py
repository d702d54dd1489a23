"""
CPU check of what ptxas made of the contig -> window kernels (csrc/contigs.cuh, no GPU): every one is in the sm_90a build log
(genomad_b200/build.log, `-Xptxas -v`) with no stack frame and no spills.
"""
import re

import pytest

from genomad_b200 import build as B

KERNELS = {"contig_plan_kernel<count>": "_ZN3gnm18contig_plan_kernelILb0EEEvPKhPKliPiPlS5_",
           "contig_plan_kernel<write>": "_ZN3gnm18contig_plan_kernelILb1EEEvPKhPKliPiPlS5_",
           "contig_scan_kernel": "_ZN3gnm18contig_scan_kernelEPii",
           "gather_windows_kernel": "_ZN3gnm21gather_windows_kernelEPKhPKlPKiPh"}


@pytest.fixture(scope="module")
def log() -> str:
    B.build()
    return (B.PKG / "build.log").read_text()


@pytest.mark.parametrize("kernel", sorted(KERNELS))
def test_contig_kernels_do_not_spill(log, kernel):
    assert f"Compiling entry function '{KERNELS[kernel]}' for 'sm_90a'" in log
    m = re.search(r"Function properties for " + re.escape(KERNELS[kernel]) +
                  r"\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert m, f"no ptxas resource report for {kernel} in build.log"
    assert tuple(map(int, m.groups())) == (0, 0, 0), f"{kernel}: stack frame / spills {m.groups()}"
