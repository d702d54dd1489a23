"""
CPU check of the head-attribution build (no GPU): libgnm.so exports the four gnm_attribute_head_* calls of include/gnm.h, and
ptxas made the two kernels they share with the shipped attributions, which now take C classes (the head gradient and log p),
without stack or spills (build.log, `-Xptxas -v`).
"""
import re
import shutil
import subprocess

import pytest

from genomad_b200 import build as B

EXPORTS = ["gnm_attribute_head_ascii", "gnm_attribute_head_windows", "gnm_attribute_head_ig_ascii",
           "gnm_attribute_head_ig_windows"]
KERNELS = {   # mangled name: register cap
    "_ZN3gnm25attr_head_backward_kernelEPKfS1_S1_S1_S1_S1_S1_S1_iPf": 64,
    "_ZN3gnm14ig_logp_kernelEPKfiiiPf": 64,
}


@pytest.fixture(scope="module")
def log() -> str:
    B.build()
    return (B.PKG / "build.log").read_text()


@pytest.mark.parametrize("name", EXPORTS)
def test_head_attribution_calls_are_exported(name):
    B.build()
    nm = shutil.which("nm") or "/usr/bin/nm"
    syms = subprocess.run([nm, "-D", "--defined-only", str(B.LIB)], capture_output=True, text=True, check=True).stdout
    assert re.search(r"\bT " + re.escape(name) + r"$", syms, re.M), f"{name} is not exported by libgnm.so"
    header = (B.PKG.parent / "include" / "gnm.h").read_text()
    assert re.search(r"\bint " + re.escape(name) + r"\(", header), f"{name} is not declared in include/gnm.h"


@pytest.mark.parametrize("mangled", sorted(KERNELS))
def test_class_count_kernels_do_not_spill(log, mangled):
    m = re.search(r"Function properties for " + re.escape(mangled) + r"\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\n.*?Used (\d+) registers", log)
    assert m, f"no ptxas resource report for {mangled} in build.log"
    stack, stores, loads, regs = map(int, m.groups())
    assert stack == 0 and stores == 0 and loads == 0, f"{mangled}: stack {stack} B, spills {stores} / {loads} B"
    assert regs <= KERNELS[mangled], f"{mangled} uses {regs} registers, more than {KERNELS[mangled]}"
