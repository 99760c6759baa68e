"""CPU: what the compiler made of the bf16 and fp8 GEMM kernels (sm_90a SASS of the built library; no GPU needed)."""

import re
import shutil
import subprocess

import pytest


@pytest.fixture(scope="module")
def lib_path():
    from dolomite_engine_b200 import _lib, build

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    build.build()
    return _lib.LIB_PATH


def test_wide_tile_instructions(lib_path):
    """the 128 x 256 tile issues wgmma m64n256k16 and moves registers from the producer to the consumers (setmaxnreg)"""
    sass = subprocess.run(["cuobjdump", "-sass", lib_path], capture_output=True, text=True).stdout
    assert "HGMMA.64x256x16.F32.BF16" in sass
    assert "HGMMA.64x128x16.F32.BF16" in sass
    assert "USETMAXREG" in sass


def test_gemm_kernels_do_not_spill(lib_path):
    """every gemm_bf16_kernel instantiation (four operand layouts x two tile widths) keeps its accumulators in registers:
    no stack frame, no local memory"""
    res = subprocess.run(["cuobjdump", "-res-usage", lib_path], capture_output=True, text=True).stdout
    found = re.findall(r"Function (\S*gemm_bf16_kernel\S*):\s*\n\s*(REG:.*)", res)
    assert len(found) == 8, [f[0] for f in found]
    for name, usage in found:
        stack = int(re.search(r"STACK:(\d+)", usage).group(1))
        local = int(re.search(r"LOCAL:(\d+)", usage).group(1))
        assert stack == 0 and local == 0, (name, usage)


def test_fp8_gemm_kernels_do_not_spill(lib_path):
    """every gemm_fp8_kernel instantiation (four format pairs x split accumulation on / off) keeps its accumulators (and
    the split accumulator's second register set) in registers: no stack frame, no local memory"""
    res = subprocess.run(["cuobjdump", "-res-usage", lib_path], capture_output=True, text=True).stdout
    found = re.findall(r"Function (\S*gemm_fp8_kernel\S*):\s*\n\s*(REG:.*)", res)
    assert len(found) == 8, [f[0] for f in found]
    for name, usage in found:
        stack = int(re.search(r"STACK:(\d+)", usage).group(1))
        local = int(re.search(r"LOCAL:(\d+)", usage).group(1))
        assert stack == 0 and local == 0, (name, usage)
