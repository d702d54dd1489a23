"""
CPU check of what ptxas made of the embedding-cluster kernels (no GPU).  The build log (genomad_b200/build.log, `-Xptxas -v`)
must show no stack and no spills and register counts within the caps (the mask kernel: 384 threads, one CTA per SM, like the
search kernel whose mainloop it shares), no serialized wgmma (C7514 / C7517 / C7520) in the mask kernel, and HGMMA in its SASS.
"""
import re
import shutil
import subprocess

import pytest

from genomad_b200 import build as B

MASK = "_ZN3gnm14nb_mask_kernelE14CUtensorMap_stS0_S0_S0_NS_12NbMaskParamsE"
KERNELS = {   # mangled name: register cap
    MASK: 168,
    "_ZN3gnm17cl_resolve_kernelEPKjiiPKhPiS4_": 128,
}


@pytest.fixture(scope="module")
def log() -> str:
    B.build()
    path = B.PKG / "build.log"
    assert path.exists(), "the library build writes build.log next to libgnm.so"
    return path.read_text()


@pytest.mark.parametrize("mangled", sorted(KERNELS))
def test_clusters_registers(log, mangled):
    m = re.search(r"Function properties for " + re.escape(mangled) + r"\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\n.*?Used (\d+) registers", log)
    assert m, f"no ptxas resource report for {mangled} in build.log"
    stack, stores, loads, regs = map(int, m.groups())
    assert stack == 0 and stores == 0 and loads == 0, f"{mangled}: stack {stack} B, spills {stores} / {loads} B"
    assert regs <= KERNELS[mangled], f"{mangled} uses {regs} registers, more than {KERNELS[mangled]}"


def test_mask_wgmma_not_serialized(log):
    bad = [ln for ln in log.splitlines() if ("C7520" in ln or "C7514" in ln or "C7517" in ln) and MASK in ln]
    assert not bad, bad[0]


def test_mask_contains_wgmma():
    B.build()
    cob = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([cob, "-sass", str(B.LIB)], capture_output=True, text=True).stdout
    body = sass.split("Function : " + MASK, 1)
    assert len(body) == 2, f"{MASK} not in the SASS of {B.LIB}"
    assert "HGMMA" in body[1].split("Function : ", 1)[0], f"{MASK}: no wgmma (HGMMA) in its SASS"
