"""CPU: the template instances of the attention kernels in the built library are exactly the ones
test_gpu_attention_elementwise.py reaches (attention_instances.INSTANCES), and the host-side layout checks of the attention
wrappers (no GPU needed: they run before any launch)."""

import re
import shutil
import subprocess

import pytest
import torch

from attention_instances import DECODE_CASES, FWD_BWD_CASES, INSTANCES

# mangled template arguments: Li<n>E = int n, Lb<0|1>E = bool
_TEMPLATED = re.compile(r"\d+(attn_fwd_kernel|attn_bwd_kernel|attn_dq_kernel|attn_decode_kernel)ILi(\d+)ELb([01])EE")
_PLAIN = re.compile(r"\d+(attn_delta_kernel)E")


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
        m = _TEMPLATED.search(name)
        if m:
            fam, hd, alibi = m.groups()
            found.add(f"{fam}<{hd}, {alibi}>")
        elif _PLAIN.search(name):
            found.add(_PLAIN.search(name).group(1))
    return found


def test_every_built_attention_instance_has_a_per_element_case(lib_path):
    """4 families x 6 head dims x {plain, ALiBi} + the Delta kernel; a new instance without a case fails here"""
    built = _built_instances(lib_path)
    assert len(built) == 49, sorted(built)
    assert built == set(INSTANCES), (sorted(built - set(INSTANCES)), sorted(set(INSTANCES) - built))


def test_case_grid_covers_what_the_per_element_tests_promise():
    ragged = [c for c in FWD_BWD_CASES.values() if c["dist"] != "late"]
    # every head_dim x {plain, ALiBi} x {dropout 0, dropout > 0}
    assert {(c["hd"], c["alibi"], c["dropout"] > 0) for c in ragged} == {
        (hd, a, d) for hd in (16, 32, 64, 80, 96, 128) for a in (False, True) for d in (False, True)}
    assert len(ragged) == 24
    # MHA, GQA with g = 2..5, MQA; 16 heads with ALiBi; both scales; every input distribution
    gs = {c["g"] for c in ragged if c["ng"] > 1}
    assert {1, 2, 3, 4, 5} <= gs and any(c["ng"] == 1 and c["g"] > 1 for c in ragged)
    assert any(c["alibi"] and c["ng"] * c["g"] == 16 for c in ragged)
    assert any(bin(c["ng"] * c["g"]).count("1") > 1 for c in ragged)  # head counts that are not powers of two
    assert {c["scale"] for c in ragged} == {"rsqrt", "mup"} and {c["dist"] for c in ragged} == {"normal", "peaked", "flat"}
    for c in ragged:
        assert c["lens"][0] == 0 and c["lens"][-1] == 0 and sorted(x for x in c["lens"] if x) == [
            1, 63, 64, 65, 127, 128, 129, 255, 257, 601]
    longs = [c for c in FWD_BWD_CASES.values() if c["dist"] == "late"]
    assert {(c["hd"], c["alibi"]) for c in longs} == {(hd, a) for hd in (64, 80, 128) for a in (False, True)}
    assert all(max(c["lens"]) >= 2100 for c in longs)
    assert {(c["hd"], c["alibi"]) for c in DECODE_CASES.values()} == {
        (hd, a) for hd in (16, 32, 64, 80, 96, 128) for a in (False, True)}
    for c in DECODE_CASES.values():
        assert {1, 127, 128, 129, 255, 256, 257} <= set(c["lens"]) and max(c["lens"]) % 128 != 0


# ------------------------------------------------------------------------------------------------
# wrapper layout checks (CPU tensors: the checks run before the device check and any launch)
# ------------------------------------------------------------------------------------------------
NG, G, HD, T = 2, 2, 16, 5
NH, W = NG * G, NG * (G + 2) * HD


def K():
    from dolomite_engine_b200 import kernels

    return kernels


def _bwd_args(**over):
    a = dict(dout=torch.zeros(T, NH * HD, dtype=torch.bfloat16), qkv=torch.zeros(T, W, dtype=torch.bfloat16),
             out=torch.zeros(T, NH * HD, dtype=torch.bfloat16), lse=torch.zeros(NH, T), dqkv=None)
    a.update(over)
    return a


def _bwd(a):
    return K().attn_varlen_bwd(a["dout"], a["qkv"], a["out"], a["lse"], torch.zeros(2, dtype=torch.int32), T, NG, G, HD,
                               0.25, dqkv=a["dqkv"])


def test_backward_allocates_dqkv_with_the_row_stride_of_qkv():
    """the kernels write dqkv with qkv's row stride: a row-strided qkv view gets a dqkv of the same strides (empty_like
    would give a contiguous, shorter buffer that the kernel writes past)"""
    big = torch.zeros(T, 24, dtype=torch.bfloat16)
    qkv = big[:, :16]
    assert torch.empty_like(qkv).stride() == (16, 1)
    d = K()._attn_dqkv(qkv)
    assert d.shape == qkv.shape and d.stride() == (24, 1)
    assert K()._attn_dqkv(big).stride() == (24, 1)
    given = torch.zeros(T, 24, dtype=torch.bfloat16)[:, :16]
    assert K()._attn_dqkv(qkv, given) is given
    with pytest.raises(ValueError, match="dqkv must have qkv's shape"):
        K()._attn_dqkv(qkv, torch.zeros(T, 16, dtype=torch.bfloat16))


@pytest.mark.parametrize("bad", ["dout_strided", "out_strided", "out_shape", "lse_dtype", "lse_shape", "lse_strided",
                                 "qkv_columns", "dqkv_stride"])
def test_backward_rejects_layouts_the_kernels_do_not_address(bad):
    wide = torch.zeros(T, NH * HD + 8, dtype=torch.bfloat16)
    over = {
        "dout_strided": dict(dout=wide[:, :NH * HD]),
        "out_strided": dict(out=wide[:, :NH * HD]),
        "out_shape": dict(out=torch.zeros(T, NH * HD - 8, dtype=torch.bfloat16)),
        "lse_dtype": dict(lse=torch.zeros(NH, T, dtype=torch.float64)),
        "lse_shape": dict(lse=torch.zeros(T, NH)),
        "lse_strided": dict(lse=torch.zeros(T, NH).t()),
        "qkv_columns": dict(qkv=torch.zeros(W, T, dtype=torch.bfloat16).t()),
        "dqkv_stride": dict(dqkv=torch.zeros(T, W + 8, dtype=torch.bfloat16)[:, :W]),
    }[bad]
    name = bad.split("_")[0]
    with pytest.raises(ValueError, match=f"^{name} must"):
        _bwd(_bwd_args(**over))


def test_backward_with_good_layouts_reaches_the_device_check():
    """the layout checks pass a row-strided qkv with a matching dqkv; what stops the CPU tensors is the device check"""
    from dolomite_engine_b200 import _lib

    qkv = torch.zeros(T, W + 8, dtype=torch.bfloat16)[:, :W]
    with pytest.raises(_lib.DolomiteB200Error, match="CUDA tensor"):
        _bwd(_bwd_args(qkv=qkv, dqkv=torch.zeros(T, W + 8, dtype=torch.bfloat16)[:, :W]))


@pytest.mark.parametrize("bad", ["out_strided", "out_shape", "qkv_columns"])
def test_forward_rejects_layouts_the_kernels_do_not_address(bad):
    qkv = torch.zeros(T, W, dtype=torch.bfloat16)
    out = None
    if bad == "out_strided":
        out = torch.zeros(T, NH * HD + 8, dtype=torch.bfloat16)[:, :NH * HD]
    elif bad == "out_shape":
        out = torch.zeros(T + 1, NH * HD, dtype=torch.bfloat16)
    else:
        qkv = torch.zeros(W, T, dtype=torch.bfloat16).t()
    with pytest.raises(ValueError, match=f"^{bad.split('_')[0]} must"):
        K().attn_varlen_fwd(qkv, torch.zeros(2, dtype=torch.int32), T, NG, G, HD, 0.25, out=out)
