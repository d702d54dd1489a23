"""
CPU check of what ptxas made of the conv kernel (no GPU).  The build log (genomad_b200/build.log, `-Xptxas -v`) must show, for
both instantiations of conv_t_kernel, that the wgmma are not serialized (ptxas C7520: a wgmma reached on a path the compiler
cannot prove warp-uniform makes it drain every wgmma before the next one issues), no spills, and a register count that fits
384 threads in one CTA per SM.
"""
import re

import pytest

from genomad_b200 import build as B

CONV_T = {"conv_t_kernel<false>": "_ZN3gnm13conv_t_kernelILb0EEEv14CUtensorMap_stS1_NS_12ConvTcParamsE",
          "conv_t_kernel<true>": "_ZN3gnm13conv_t_kernelILb1EEEv14CUtensorMap_stS1_NS_12ConvTcParamsE"}


@pytest.fixture(scope="module")
def log() -> str:
    B.build()
    path = B.PKG / "build.log"
    assert path.exists(), "the library build writes build.log next to libgnm.so"
    return path.read_text()


@pytest.mark.parametrize("kernel", sorted(CONV_T))
def test_conv_t_wgmma_not_serialized(log, kernel):
    mangled = CONV_T[kernel]
    serialized = [ln for ln in log.splitlines() if "C7520" in ln and mangled in ln]
    assert not serialized, f"{kernel}: {serialized[0]}"


@pytest.mark.parametrize("kernel", sorted(CONV_T))
def test_conv_t_registers(log, kernel):
    m = re.search(r"Function properties for " + re.escape(CONV_T[kernel]) + r"\n.*?(\d+) bytes spill stores, (\d+) bytes spill loads"
                  r"\n.*?Used (\d+) registers", log)
    assert m, f"no ptxas resource report for {kernel} in build.log"
    stores, loads, regs = map(int, m.groups())
    assert stores == 0 and loads == 0, f"{kernel} spills ({stores} B stored, {loads} B loaded)"
    assert regs <= 168, f"{kernel} uses {regs} registers; 384 threads per SM allow 168"


# Layer 1 from caller tokens checks each half's three tokens before it takes a triple-table row; that check must not cost the
# kernels their occupancy: embed_conv1_kernel runs 8 CTAs of 256 threads per SM (32 registers), layer1_wv_kernel 1024 threads.
LAYER1 = {"embed_conv1_kernel<false>": ("_ZN3gnm18embed_conv1_kernelILb0EEEvPKhPKtPKfS6_S6_PhiPNS_12DeviceStatusE", 32),
          "embed_conv1_kernel<true>": ("_ZN3gnm18embed_conv1_kernelILb1EEEvPKhPKtPKfS6_S6_PhiPNS_12DeviceStatusE", 32),
          "layer1_wv_kernel<false>": ("_ZN3gnm16layer1_wv_kernelILb0EEEv14CUtensorMap_stNS_11FusedParamsE", 64),
          "layer1_wv_kernel<true>": ("_ZN3gnm16layer1_wv_kernelILb1EEEv14CUtensorMap_stNS_11FusedParamsE", 64)}


@pytest.mark.parametrize("kernel", sorted(LAYER1))
def test_layer1_registers(log, kernel):
    mangled, cap = LAYER1[kernel]
    m = re.search(r"Function properties for " + re.escape(mangled) + r"\n.*?(\d+) bytes spill stores, (\d+) bytes spill loads"
                  r"\n.*?Used (\d+) registers", log)
    assert m, f"no ptxas resource report for {kernel} in build.log"
    stores, loads, regs = map(int, m.groups())
    assert stores == 0 and loads == 0, f"{kernel} spills ({stores} B stored, {loads} B loaded)"
    assert regs <= cap, f"{kernel} uses {regs} registers, more than {cap}"
