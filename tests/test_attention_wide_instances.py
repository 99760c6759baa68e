"""CPU: the wide-head attention kernels (head_dim 160, 192, 256) in the built library are exactly the instances
test_gpu_attention_wide.py reaches, none of them uses local memory, check_supported accepts exactly the new head dims, and
the wrappers' layout checks run for a wide head_dim before any launch."""

import re
import shutil
import subprocess

import pytest
import torch

from attention_wide_instances import DECODE_CASES, FWD_BWD_CASES, HEAD_DIMS, INSTANCES

# mangled template arguments: Li<n>E = int n, Lb<0|1>E = bool
_WIDE = re.compile(r"\d+(attn_wide_fwd_kernel|attn_wide_bwd_kernel|attn_wide_dq_kernel|attn_wide_decode_kernel)ILi(\d+)ELb([01])EE")


@pytest.fixture(scope="module")
def res_usage():
    from dolomite_engine_b200 import _lib, build

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    build.build()
    return subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout


def _wide_instances(res: str) -> dict:
    """instance -> its resource line"""
    found = {}
    for name, usage in re.findall(r"Function (\S+):\s*\n\s*(REG:[^\n]*)", res):
        m = _WIDE.search(name)
        if m:
            fam, hd, alibi = m.groups()
            found[f"{fam}<{hd}, {alibi}>"] = usage
    return found


def test_every_wide_instance_has_a_per_element_case(res_usage):
    """4 families x 3 head dims x {plain, ALiBi}"""
    built = _wide_instances(res_usage)
    assert len(built) == 24, sorted(built)
    assert set(built) == set(INSTANCES), (sorted(set(built) - set(INSTANCES)), sorted(set(INSTANCES) - set(built)))


def test_no_wide_instance_uses_local_memory(res_usage):
    for inst, usage in _wide_instances(res_usage).items():
        assert re.search(r"\bLOCAL:0\b", usage) and re.search(r"\bSTACK:0\b", usage), (inst, usage)


def test_case_grid_covers_what_the_per_element_tests_promise():
    ragged = [c for c in FWD_BWD_CASES.values() if c["dist"] != "late"]
    assert {(c["hd"], c["alibi"], c["dropout"] > 0) for c in ragged} == {
        (hd, a, d) for hd in HEAD_DIMS for a in (False, True) for d in (False, True)}
    gs = {c["g"] for c in ragged if c["ng"] > 1}
    assert {1, 2, 3, 4, 5} <= gs
    assert any(c["ng"] == 1 and c["g"] == 16 for c in ragged)  # MQA with 16 heads
    assert {c["scale"] for c in ragged} == {"rsqrt", "mup"}
    for c in ragged:
        assert c["lens"][0] == 0 and c["lens"][-1] == 0 and 0 in c["lens"][1:-1]
        assert sorted(x for x in c["lens"] if x) == [1, 63, 64, 65, 127, 128, 129, 255, 257, 601]
    longs = [c for c in FWD_BWD_CASES.values() if c["dist"] == "late"]
    assert sorted(c["hd"] for c in longs) == list(HEAD_DIMS) and all(2150 in c["lens"] for c in longs)
    assert {(c["hd"], c["alibi"]) for c in DECODE_CASES.values()} == {(hd, a) for hd in HEAD_DIMS for a in (False, True)}
    for c in DECODE_CASES.values():
        assert c["lens"] == [1, 127, 128, 129, 255, 256, 257, 700]


# ------------------------------------------------------------------------------------------------
# check_supported
# ------------------------------------------------------------------------------------------------
def _cfg(hd: int, n_head: int = 2):
    from dolomite_engine_b200.hf_models.config import GPTDolomiteConfig

    return GPTDolomiteConfig(n_embd=hd * n_head, n_head=n_head, attention_head_type="mqa", num_key_value_heads=1,
                             position_embedding_type="rope", activation_function="swiglu", normalization_function="rmsnorm",
                             resid_pdrop=0, embd_pdrop=0, attn_pdrop=0, vocab_size=512, n_layer=1)


@pytest.mark.parametrize("hd", [16, 32, 64, 80, 96, 128, 160, 192, 256])
def test_check_supported_accepts_every_kernel_head_dim(hd):
    from dolomite_engine_b200.engine import check_supported

    check_supported(_cfg(hd))


@pytest.mark.parametrize("hd", [8, 24, 48, 112, 144, 176, 208, 224, 240, 288, 320, 512])
def test_check_supported_rejects_head_dims_without_kernels(hd):
    from dolomite_engine_b200.engine import check_supported

    with pytest.raises(NotImplementedError, match=f"head_dim={hd}: supported head dims are 16, 32, 64, 80, 96, 128, 160, 192, 256"):
        check_supported(_cfg(hd))


def test_the_c_entry_points_reject_head_dims_without_kernels():
    """the head_dim switch of each entry point runs before any launch (null pointers never reach a kernel)"""
    from dolomite_engine_b200 import _lib

    for hd in (144, 224, 288):
        with pytest.raises(_lib.DolomiteB200Error, match="unsupported head_dim .*160,192,256"):
            _lib.call("dolomite_b200_attn_varlen_fwd", None, 4096, None, None, None, 1, 16, 16, 1, 1, hd, 1.0, None)
        with pytest.raises(_lib.DolomiteB200Error, match="unsupported head_dim .*160,192,256"):
            _lib.call("dolomite_b200_attn_varlen_bwd", None, None, 4096, None, None, None, None, 1, 16, 16, 1, 1, hd, 1.0,
                      None, None)
        with pytest.raises(_lib.DolomiteB200Error, match="unsupported head_dim .*160,192,256"):
            _lib.call("dolomite_b200_attn_decode", None, 4096, None, None, None, None, 1, 16, 1, 1, hd, 1.0, None)


# ------------------------------------------------------------------------------------------------
# wrapper layout checks at a wide head_dim (CPU tensors: the checks run before the device check and any launch)
# ------------------------------------------------------------------------------------------------
NG, G, T = 1, 2, 5
HD = 256
NH, W = NG * G, NG * (G + 2) * HD


def K():
    from dolomite_engine_b200 import kernels

    return kernels


@pytest.mark.parametrize("bad", ["dout_strided", "out_shape", "lse_shape", "qkv_columns", "dqkv_stride"])
def test_wide_backward_rejects_layouts_the_kernels_do_not_address(bad):
    wide = torch.zeros(T, NH * HD + 8, dtype=torch.bfloat16)
    a = dict(dout=torch.zeros(T, NH * HD, dtype=torch.bfloat16), qkv=torch.zeros(T, W, dtype=torch.bfloat16),
             out=torch.zeros(T, NH * HD, dtype=torch.bfloat16), lse=torch.zeros(NH, T), dqkv=None)
    a.update({
        "dout_strided": dict(dout=wide[:, :NH * HD]),
        "out_shape": dict(out=torch.zeros(T, NH * HD - 8, dtype=torch.bfloat16)),
        "lse_shape": dict(lse=torch.zeros(T, NH)),
        "qkv_columns": dict(qkv=torch.zeros(W, T, dtype=torch.bfloat16).t()),
        "dqkv_stride": dict(dqkv=torch.zeros(T, W + 8, dtype=torch.bfloat16)[:, :W]),
    }[bad])
    with pytest.raises(ValueError, match=f"^{bad.split('_')[0]} must"):
        K().attn_varlen_bwd(a["dout"], a["qkv"], a["out"], a["lse"], torch.zeros(2, dtype=torch.int32), T, NG, G, HD, 0.25,
                            dqkv=a["dqkv"])


@pytest.mark.parametrize("bad", ["out_strided", "out_shape", "qkv_columns"])
def test_wide_forward_rejects_layouts_the_kernels_do_not_address(bad):
    qkv, out = torch.zeros(T, W, dtype=torch.bfloat16), None
    if bad == "out_strided":
        out = torch.zeros(T, NH * HD + 8, dtype=torch.bfloat16)[:, :NH * HD]
    elif bad == "out_shape":
        out = torch.zeros(T + 1, NH * HD, dtype=torch.bfloat16)
    else:
        qkv = torch.zeros(W, T, dtype=torch.bfloat16).t()
    with pytest.raises(ValueError, match=f"^{bad.split('_')[0]} must"):
        K().attn_varlen_fwd(qkv, torch.zeros(2, dtype=torch.int32), T, NG, G, HD, 0.25, out=out)


def test_wide_forward_with_good_layouts_reaches_the_device_check():
    from dolomite_engine_b200 import _lib

    with pytest.raises(_lib.DolomiteB200Error, match="CUDA tensor"):
        K().attn_varlen_fwd(torch.zeros(T, W + 8, dtype=torch.bfloat16)[:, :W], torch.zeros(2, dtype=torch.int32), T, NG,
                            G, HD, 0.25)
