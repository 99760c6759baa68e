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


# demangled (cu++filt) kernel name -> its template arguments as integers: gemm_bf16_kernel<(bool)0, (bool)1, (int)128>
_INSTANCE = re.compile(r"(gemm_bf16_kernel|gemm_fp8_kernel)<\(\w+\)(\d+), \(\w+\)(\d+), \(\w+\)(\d+)>")


def _built_gemm_instances(lib_path) -> set:
    res = subprocess.run(["cuobjdump", "-res-usage", lib_path], capture_output=True, text=True, check=True).stdout
    mangled = "\n".join(re.findall(r"Function (\S*gemm_\w+_kernel\S*):", res))
    filt = shutil.which("cu++filt") or shutil.which("c++filt")
    if filt is None:
        pytest.skip("no demangler (cu++filt / c++filt)")
    names = subprocess.run([filt], input=mangled, capture_output=True, text=True, check=True).stdout
    return {f"{m[0]}<{m[1]}, {m[2]}, {m[3]}>" for m in _INSTANCE.findall(names)}


def test_every_built_gemm_instance_has_per_element_cases(lib_path):
    """4 layouts x 2 tile widths of the bf16 kernel and 4 format pairs x split / fast accumulation of the fp8 kernel; a
    new instance without a case of tests/gemm_instances.py, or a case whose instance is not built, fails here"""
    from gemm_instances import INSTANCES

    built = _built_gemm_instances(lib_path)
    assert len(built) == 16, sorted(built)
    assert built == set(INSTANCES), (sorted(built - set(INSTANCES)), sorted(set(INSTANCES) - built))


def test_gemm_cases_reach_their_instances_by_the_host_rule():
    """the host's dispatch, restated, sends every case to the instance it names, and every entry point reaches each
    instance it can run"""
    from gemm_instances import CASES, FP8_PAIRS, LAYOUTS, bf16_instance, fp8_instance, instance_of

    for name, c in CASES.items():
        assert instance_of(c) == c["instance"], name

    def reached(entry, **match):
        return {c["instance"] for c in CASES.values()
                if c["entry"] == entry and all(c.get(k) == v for k, v in match.items())}

    assert reached("gemm") == {bf16_instance(*l, tn) for l in LAYOUTS for tn in (128, 256)}
    splitk = reached("gemm_splitk")
    assert bf16_instance(True, True, 128) in splitk and len(splitk) >= 2
    assert all(c["tile_n"] == 256 for c in CASES.values() if c["entry"] in ("gemm_splitk", "grouped_m", "grouped_k"))
    assert reached("wgrad_multi") == {bf16_instance(True, True, tn) for tn in (128, 256)}
    for bias in (False, True):
        assert reached("grouped_m", bias=bias) == {bf16_instance(False, False, 128), bf16_instance(False, True, 128)}
        assert reached("grouped_m_gather", bias=bias) == {bf16_instance(False, False, 128)}
    for beta in (0.0, 1.0):
        assert reached("grouped_k", beta=beta) == {bf16_instance(True, True, 128)}
    assert reached("gemm_fp8") == {fp8_instance(fa, fb, s) for fa, fb in FP8_PAIRS for s in (False, True)}
    fp8_multi = reached("fp8_wgrad_multi")
    assert {fp8_instance(1, 0, False), fp8_instance(1, 0, True)} <= fp8_multi and len(fp8_multi) >= 3
    # the shapes the per-element cases promise: M, N and K tails, a long contraction with hints, more tiles than SMs
    dense = [c["shape"] for c in CASES.values() if c["entry"] == "gemm"]
    assert {m % 128 for m, _, _ in dense} >= {1, 63, 64, 65, 127}
    assert {1, 8, 136, 264} <= {n for _, n, _ in dense} and {8, 136} <= {n % 256 for _, n, _ in dense}
    assert {1, 8, 40} <= {k for _, _, k in dense} and {8, 56} <= {k % 64 for _, _, k in dense}
    assert any(k >= 4096 and (m + n) * k * 2 > (24 << 20) for m, n, k in dense)
    assert any(-(-m // 128) * -(-n // 256) >= 2 * 132 for m, n, _ in dense)
    fp8 = [c["shape"] for c in CASES.values() if c["entry"] == "gemm_fp8"]
    assert all(k % 16 == 0 and n % 16 == 0 for _, n, k in fp8) and {16, 144} <= {k for _, _, k in fp8}
