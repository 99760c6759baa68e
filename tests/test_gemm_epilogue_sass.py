"""CPU: the bf16 and fp8 GEMMs write their output tiles with TMA stores from shared memory, never with per-thread global stores
(sm_90a SASS of the built library; no GPU needed)."""

import re
import shutil
import subprocess

import pytest


@pytest.fixture(scope="module")
def gemm_sass():
    from dolomite_engine_b200 import _lib, build

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    build.build()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    funcs = {}
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split("\n", 1)[0].strip()
        if "gemm_bf16_kernel" in name or "gemm_fp8_kernel" in name:
            funcs[name] = body
    return funcs


def _opcodes(body):
    return re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9]*)", body)


def test_every_instantiation_stores_through_tma(gemm_sass):
    """four operand layouts x two tile widths: UTMASTG (and the split-K UTMAREDG), STSM for the bf16 slabs, no STG"""
    bf16 = {n: b for n, b in gemm_sass.items() if "gemm_bf16_kernel" in n}
    assert len(bf16) == 8, sorted(bf16)
    for name, body in bf16.items():
        ops = _opcodes(body)
        assert "UTMASTG" in ops and "UTMAREDG" in ops and "STSM" in ops, name
        assert "STG" not in ops and "RED" not in ops, name


def test_every_fp8_instantiation_stores_through_tma(gemm_sass):
    """four format pairs x split accumulation on / off: the m64n128k32 fp8 MMA of the instance's format pair, and the
    bf16 kernel's epilogue -- UTMASTG, STSM for the bf16 slabs, no STG"""
    fmt = {"0": "E4M3", "1": "E5M2"}
    fp8 = {n: b for n, b in gemm_sass.items() if "gemm_fp8_kernel" in n}
    assert len(fp8) == 8, sorted(fp8)
    for name, body in fp8.items():
        fa, fb = re.search(r"gemm_fp8_kernelILi(\d)ELi(\d)ELb[01]E", name).groups()
        assert f"QGMMA.64x128x32.F32.{fmt[fa]}.{fmt[fb]}" in body, name
        ops = _opcodes(body)
        assert "UTMASTG" in ops and "STSM" in ops, name
        assert "STG" not in ops and "RED" not in ops, name
