"""CPU: the bf16 GEMM writes its output tiles with TMA stores from shared memory, never with per-thread global stores
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
        if "gemm_bf16_kernel" in name:
            funcs[name] = body
    return funcs


def test_every_instantiation_stores_through_tma(gemm_sass):
    """four operand layouts x two tile widths: UTMASTG (and the split-K UTMAREDG), STSM for the bf16 slabs, no STG"""
    assert len(gemm_sass) == 8, sorted(gemm_sass)
    for name, body in gemm_sass.items():
        ops = re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9]*)", body)
        assert "UTMASTG" in ops and "UTMAREDG" in ops and "STSM" in ops, name
        assert "STG" not in ops and "RED" not in ops, name
