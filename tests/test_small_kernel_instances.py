"""CPU: the template instances of the norm and RoPE kernels in the built library are exactly the ones
test_gpu_small_kernels.py reaches (INSTANCES), and host-side argument checks of the small kernels (no GPU needed)."""

import re
import shutil
import subprocess

import pytest

from small_kernel_instances import INSTANCES, chosen_instance

# mangled template arguments: Li<n>E = int n, i = int32_t, l = int64_t
_FAMILIES = "rmsnorm_fwd_kernel|rmsnorm_fwd_warp_kernel|rmsnorm_bwd_kernel|layernorm_fwd_kernel|layernorm_bwd_kernel|rope_kernel"
_MANGLED = re.compile(rf"\d+({_FAMILIES})I([il]?)Li(\d+)EE")
_POS = {"i": "int32_t", "l": "int64_t"}


@pytest.fixture(scope="module")
def lib_path():
    from dolomite_engine_b200 import _lib, build

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    build.build()
    return _lib.LIB_PATH


def _built_instances(lib_path) -> set:
    res = subprocess.run(["cuobjdump", "-res-usage", lib_path], capture_output=True, text=True, check=True).stdout
    found = set()
    for name in re.findall(r"Function (\S+):", res):
        m = _MANGLED.search(name)
        if m:
            fam, pos, n = m.groups()
            found.add(f"{fam}<{_POS[pos]}, {n}>" if pos else f"{fam}<{n}>")
    return found


def test_every_built_instance_has_a_kernel_test(lib_path):
    """a new instance without an entry in INSTANCES (and so without a GPU test) fails here"""
    built = _built_instances(lib_path)
    assert len(built) == 24, sorted(built)
    assert built == set(INSTANCES), (sorted(built - set(INSTANCES)), sorted(set(INSTANCES) - built))


@pytest.mark.parametrize("name", sorted(INSTANCES))
def test_instance_shape_reaches_its_instance(name):
    """the host's choice rule (restated in small_kernel_instances.py) sends INSTANCES[name] to `name`"""
    assert chosen_instance(name) == name


def test_embedding_bwd_rejects_a_misaligned_gradient_buffer():
    """dwte is written through float4: a pointer that is not 16-byte aligned is refused on the host, before any launch"""
    from dolomite_engine_b200 import _lib, build

    build.build()
    with pytest.raises(_lib.DolomiteB200Error, match="16-byte aligned"):
        _lib.call("dolomite_b200_embedding_bwd", None, 256, 4, 4, 64, 16, 1.0, None)
    with pytest.raises(_lib.DolomiteB200Error, match="16-byte aligned"):
        _lib.call("dolomite_b200_embedding_bwd", None, 8, 256, 4, 64, 16, 1.0, None)
    # aligned pointers and no tokens: accepted, nothing launched
    _lib.call("dolomite_b200_embedding_bwd", None, 256, 512, 0, 64, 16, 1.0, None)
