"""
CPU check of what ptxas made of the embedding-neighbour kernels (no GPU).  The build log (genomad_b200/build.log, `-Xptxas -v`)
must show no stack and no spills, register counts within the planned caps (the search kernel: 384 threads, one CTA per SM for
its ~225 KB of shared memory), no serialized wgmma (C7514 / C7517 / C7520) in the search kernel, and HGMMA in its SASS.
"""
import re
import shutil
import subprocess

import pytest

from genomad_b200 import build as B

SEARCH = "_ZN3gnm16nb_search_kernelE14CUtensorMap_stS0_S0_S0_NS_14NbSearchParamsE"
KERNELS = {   # mangled name: register cap
    SEARCH: 168,
    "_ZN3gnm14nb_prep_kernelEPKfiPfS2_": 64,
    "_ZN3gnm18nb_finalize_kernelEPKfPKiiiixPfPx": 64,
    "_ZN3gnm15nb_merge_kernelEPfPxPKfPKxii": 64,
}


@pytest.fixture(scope="module")
def log() -> str:
    B.build()
    path = B.PKG / "build.log"
    assert path.exists(), "the library build writes build.log next to libgnm.so"
    return path.read_text()


@pytest.mark.parametrize("mangled", sorted(KERNELS))
def test_neighbours_registers(log, mangled):
    m = re.search(r"Function properties for " + re.escape(mangled) + r"\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\n.*?Used (\d+) registers", log)
    assert m, f"no ptxas resource report for {mangled} in build.log"
    stack, stores, loads, regs = map(int, m.groups())
    assert stack == 0 and stores == 0 and loads == 0, f"{mangled}: stack {stack} B, spills {stores} / {loads} B"
    assert regs <= KERNELS[mangled], f"{mangled} uses {regs} registers, more than {KERNELS[mangled]}"


def test_search_wgmma_not_serialized(log):
    bad = [ln for ln in log.splitlines() if ("C7520" in ln or "C7514" in ln or "C7517" in ln) and SEARCH in ln]
    assert not bad, bad[0]


def test_search_contains_wgmma():
    B.build()
    cob = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([cob, "-sass", "-fun", SEARCH, str(B.LIB)], capture_output=True, text=True).stdout
    assert "HGMMA" in sass, f"{SEARCH}: no wgmma (HGMMA) in its SASS"
