"""CPU: the KV-cache attention kernel (csrc/attention_cache.cu) in the built library has exactly the instances
test_gpu_attention_cache.py reaches, none of them uses local memory, and the C entry points and kernels.attn_cache reject
bad arguments before any launch."""

import re
import shutil
import subprocess

import pytest
import torch

from attention_cache_instances import CASES, HEAD_CONFIGS, HEAD_DIMS, INSTANCES, NEWS, PASTS

# mangled template arguments: Li<n>E = int n, Lb<0|1>E = bool
_CACHE = re.compile(r"\d+(attn_cache_kernel)ILi(\d+)ELb([01])EE")


@pytest.fixture(scope="module")
def res_usage():
    from dolomite_engine_b200 import _lib, build

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    build.build()
    return subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout


def _instances(res: str) -> dict:
    found = {}
    for name, usage in re.findall(r"Function (\S+):\s*\n\s*(REG:[^\n]*)", res):
        m = _CACHE.search(name)
        if m:
            fam, hd, alibi = m.groups()
            found[f"{fam}<{hd}, {alibi}>"] = usage
    return found


def test_every_cache_instance_has_a_per_element_case(res_usage):
    """9 head dims x {plain, ALiBi}"""
    built = _instances(res_usage)
    assert len(built) == 18, sorted(built)
    assert set(built) == set(INSTANCES), (sorted(set(built) - set(INSTANCES)), sorted(set(INSTANCES) - set(built)))


def test_no_cache_instance_uses_local_memory(res_usage):
    for inst, usage in _instances(res_usage).items():
        assert re.search(r"\bLOCAL:0\b", usage) and re.search(r"\bSTACK:0\b", usage), (inst, usage)


def test_case_grid_covers_what_the_per_element_tests_promise():
    assert {(c["hd"], c["alibi"]) for c in CASES.values()} == {(hd, a) for hd in HEAD_DIMS for a in (False, True)}
    assert {(c["ng"], c["g"]) for c in CASES.values()} == set(HEAD_CONFIGS)
    assert {c["scale"] for c in CASES.values()} == {"rsqrt", "mup"}
    assert {c["dist"] for c in CASES.values()} == {"normal", "peaked", "flat"}
    for c in CASES.values():
        assert c["past"] == list(PASTS) and set(c["n"]) == set(NEWS)


# ------------------------------------------------------------------------------------------------
# argument checks of the C entry points (null pointers never reach a kernel) and of the wrapper
# ------------------------------------------------------------------------------------------------
def _call(name, **kw):
    from dolomite_engine_b200 import _lib

    a = dict(qkv=None, row_stride=4096, cu_new=None, past=None, k=None, v=None, out=None, batch=2, max_new=4, max_end=8,
             L_max=16, ng=1, g=2, hd=64, scale=1.0)
    slopes = kw.pop("slopes", 16)  # a non-null pointer value, never dereferenced before the checks
    a.update(kw)
    args = list(a.values()) + ([slopes] if name.endswith("alibi") else [])
    _lib.call(name, *args, None)


@pytest.mark.parametrize("name", ["dolomite_b200_attn_cache", "dolomite_b200_attn_cache_alibi"])
@pytest.mark.parametrize("hd", [8, 48, 112, 144, 224, 288])
def test_c_entry_points_reject_head_dims_without_kernels(name, hd):
    from dolomite_engine_b200 import _lib

    with pytest.raises(_lib.DolomiteB200Error, match="unsupported head_dim .*160,192,256"):
        _call(name, hd=hd)


@pytest.mark.parametrize("name", ["dolomite_b200_attn_cache", "dolomite_b200_attn_cache_alibi"])
@pytest.mark.parametrize("bad", [dict(qkv=8), dict(k=24), dict(v=40), dict(out=4), dict(row_stride=4100)])
def test_c_entry_points_reject_misaligned_operands(name, bad):
    from dolomite_engine_b200 import _lib

    with pytest.raises(_lib.DolomiteB200Error, match="attn_cache: alignment"):
        _call(name, **bad)


@pytest.mark.parametrize("name", ["dolomite_b200_attn_cache", "dolomite_b200_attn_cache_alibi"])
def test_c_entry_points_reject_past_plus_n_beyond_the_cache(name):
    from dolomite_engine_b200 import _lib

    with pytest.raises(_lib.DolomiteB200Error, match="exceeds the cache length 16"):
        _call(name, max_end=17)
    with pytest.raises(_lib.DolomiteB200Error, match="bad sizes"):
        _call(name, max_new=-1)


def test_alibi_entry_point_rejects_null_slopes():
    from dolomite_engine_b200 import _lib

    with pytest.raises(_lib.DolomiteB200Error, match="alibi_slopes is null"):
        _call("dolomite_b200_attn_cache_alibi", slopes=None)


NG, G, HD, B, L = 2, 3, 64, 3, 32
NH, W = NG * G, NG * (G + 2) * HD


def _args(**kw):
    a = dict(qkv=torch.zeros(5, W, dtype=torch.bfloat16), cu_new=torch.tensor([0, 2, 2, 5], dtype=torch.int32),
             past=torch.zeros(B, dtype=torch.int32), k=torch.zeros(B, L, NG * HD, dtype=torch.bfloat16),
             v=torch.zeros(B, L, NG * HD, dtype=torch.bfloat16), out=None, max_new=3, max_end=8)
    a.update(kw)
    return a


def _wrap(a):
    from dolomite_engine_b200 import kernels

    return kernels.attn_cache(a["qkv"], a["cu_new"], a["past"], a["k"], a["v"], NG, G, HD, 0.125, max_new=a["max_new"],
                              max_end=a["max_end"], out=a["out"])


@pytest.mark.parametrize("bad,match", [
    (dict(qkv=torch.zeros(W, 5, dtype=torch.bfloat16).t()), "^qkv must"),
    (dict(out=torch.zeros(5, NH * HD + 8, dtype=torch.bfloat16)[:, :NH * HD]), "^out must"),
    (dict(out=torch.zeros(4, NH * HD, dtype=torch.bfloat16)), "^out must"),
    (dict(k=torch.zeros(B, L, NG * HD + 8, dtype=torch.bfloat16)[:, :, :NG * HD]), "^k_cache / v_cache must"),
    (dict(v=torch.zeros(B, L + 1, NG * HD, dtype=torch.bfloat16)), "^k_cache / v_cache must"),
    (dict(k=torch.zeros(B, L, HD, dtype=torch.bfloat16)), "^k_cache / v_cache must"),
    (dict(cu_new=torch.zeros(B, dtype=torch.int32)), "^cu_new / past must"),
    (dict(past=torch.zeros(B + 1, dtype=torch.int32)), "^cu_new / past must"),
])
def test_wrapper_rejects_layouts_the_kernel_does_not_address(bad, match):
    with pytest.raises(ValueError, match=match):
        _wrap(_args(**bad))


def test_wrapper_with_good_layouts_reaches_the_device_check():
    from dolomite_engine_b200 import _lib

    with pytest.raises(_lib.DolomiteB200Error, match="CUDA tensor"):
        _wrap(_args(qkv=torch.zeros(5, W + 8, dtype=torch.bfloat16)[:, :W]))


def test_wrapper_rejects_past_plus_n_beyond_the_cache():
    with pytest.raises(ValueError, match="past \\+ n \\(up to 33\\) exceeds the cache length 32"):
        _wrap(_args(max_end=33))
    # bounds read from the tensors: sequence 2 has 3 new tokens after 30 cached ones
    with pytest.raises(ValueError, match="past \\+ n \\(up to 33\\) exceeds the cache length 32"):
        _wrap(_args(past=torch.tensor([0, 0, 30], dtype=torch.int32), max_new=None, max_end=None))
