"""
CPU check of what ptxas made of the attribution kernels (no GPU).  The build log (genomad_b200/build.log, `-Xptxas -v`) must show
that the two tensor-core instantiations of the conv body used by the attribution pass (the routing w_v pass and the conv backward
pass) contain wgmma that is not serialized (ptxas C7514 / C7520), that no attribution kernel spills, and register counts that
keep their planned occupancy.
"""
import re
import shutil
import subprocess

import pytest

from genomad_b200 import build as B

ROUTE = "_ZN3gnm18conv_t_attr_kernelILi2EEEv14CUtensorMap_stS1_NS_12ConvTcParamsENS_11ConvAttrExtE"
BWD = "_ZN3gnm18conv_t_attr_kernelILi3EEEv14CUtensorMap_stS1_NS_12ConvTcParamsENS_11ConvAttrExtE"
KERNELS = {   # mangled name: register cap
    ROUTE: 168, BWD: 168,                                                          # 384 threads, one CTA per SM
    "_ZN3gnm25attr_head_backward_kernelEPKfS1_S1_S1_S1_S1_S1_S1_iPf": 64,
    "_ZN3gnm22attr_igloo_prep_kernelEPKfS1_S1_PfS2_": 64,
    "_ZN3gnm26attr_igloo_backward_kernelILb0EEEvNS_14IglooBwdParamsE": 64,
    "_ZN3gnm26attr_igloo_backward_kernelILb1EEEvNS_14IglooBwdParamsE": 64,
    "_ZN3gnm16attr_pack_kernelEPKfS1_PfPh": 64,
    "_ZN3gnm20attr_pack_gz2_kernelEPKfS1_PfPhPNS_12DeviceStatusE": 64,
    "_ZN3gnm19reverse_rows_kernelEPfi": 64,
    "_ZN3gnm18layer1_attr_kernelEPKhPKfS3_S3_Pf": 64,
}


@pytest.fixture(scope="module")
def log() -> str:
    B.build()
    path = B.PKG / "build.log"
    assert path.exists(), "the library build writes build.log next to libgnm.so"
    return path.read_text()


@pytest.mark.parametrize("mangled", sorted(KERNELS))
def test_attr_registers(log, mangled):
    m = re.search(r"Function properties for " + re.escape(mangled) + r"\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\n.*?Used (\d+) registers", log)
    assert m, f"no ptxas resource report for {mangled} in build.log"
    stack, stores, loads, regs = map(int, m.groups())
    assert stack == 0 and stores == 0 and loads == 0, f"{mangled}: stack {stack} B, spills {stores} / {loads} B"
    assert regs <= KERNELS[mangled], f"{mangled} uses {regs} registers, more than {KERNELS[mangled]}"


@pytest.mark.parametrize("mangled", [ROUTE, BWD])
def test_attr_tensor_core_passes_not_serialized(log, mangled):
    bad = [ln for ln in log.splitlines() if ("C7520" in ln or "C7514" in ln or "C7517" in ln) and mangled in ln]
    assert not bad, bad[0]


@pytest.mark.parametrize("mangled", [ROUTE, BWD])
def test_attr_tensor_core_passes_contain_wgmma(mangled):
    B.build()
    cob = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([cob, "-sass", "-fun", mangled, str(B.LIB)], capture_output=True, text=True).stdout
    assert "HGMMA" in sass or "QGMMA" in sass, f"{mangled}: no wgmma (HGMMA / QGMMA) in its SASS"
