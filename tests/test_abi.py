"""CPU: the C-ABI library builds/loads and exports every symbol include/dolomite_b200.h declares (no compute calls)."""

import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "dolomite_b200.h")


def _declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dolomite_b200_\w+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib():
    from dolomite_engine_b200 import _lib, build

    build.build()
    return _lib.load()


def test_header_declares_symbols():
    syms = _declared_symbols()
    assert len(syms) >= 20
    assert "dolomite_b200_gemm_bf16" in syms and "dolomite_b200_attn_varlen_fwd" in syms


def test_library_exports_every_declared_symbol(lib):
    for s in _declared_symbols():
        assert hasattr(lib, s), f"{s} declared in the header but not exported"


def test_binding_table_matches_header(lib):
    from dolomite_engine_b200 import _lib

    assert sorted(_lib.SIGNATURES) == _declared_symbols()


def test_abi_version_and_error_string(lib):
    assert lib.dolomite_b200_abi_version() == 1
    lib.dolomite_b200_last_error.restype = ctypes.c_char_p
    assert isinstance(lib.dolomite_b200_last_error(), bytes)


def test_argument_validation_happens_before_any_launch(lib):
    """bad shapes are rejected on the host with a message (no GPU needed for this path)"""
    from dolomite_engine_b200 import _lib

    with pytest.raises(_lib.DolomiteB200Error, match="multiple of 8"):
        _lib.call("dolomite_b200_rmsnorm_fwd", None, None, None, None, 4, 30, 1e-5, None)
    with pytest.raises(_lib.DolomiteB200Error, match="unsupported head_dim"):
        _lib.call("dolomite_b200_attn_varlen_fwd", None, 1024, None, None, None, 1, 16, 16, 1, 1, 24, 1.0, None)


def test_sass_is_hopper_native():
    """the GEMM/attention kernels really are wgmma + TMA (HGMMA / UTMALDG in the sm_90a SASS), no mma.sync path"""
    import shutil
    import subprocess

    from dolomite_engine_b200 import _lib

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "HGMMA" in sass and "UTMALDG" in sass
    assert "HMMA." not in sass, "legacy mma.sync path found"


def test_data_feed_library_exports_every_symbol_of_its_header():
    """include/dolomite_data.h <-> lib/libdolomite_data.so (host C++, no CUDA)"""
    from dolomite_engine_b200 import build

    build.build()
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dolomite_data.h")).read(), flags=re.S)
    syms = sorted(set(re.findall(r"\b(dolomite_data_\w+)\s*\(", src)))
    assert len(syms) == 5
    lib = ctypes.CDLL(os.path.join(ROOT, "dolomite_engine_b200", "lib", "libdolomite_data.so"))
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in dolomite_data.h but not exported"
    lib.dolomite_data_num_samples.restype = ctypes.c_int64
    lib.dolomite_data_num_samples.argtypes = [ctypes.c_int64] * 3
    assert lib.dolomite_data_num_samples(8, 2, 100) == (2 * 100 - 1) // 8
