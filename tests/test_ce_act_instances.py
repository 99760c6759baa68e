"""CPU: the template instances of the cross-entropy and MLP activation kernels in the built library are exactly the ones
test_gpu_cross_entropy_elementwise.py and test_gpu_activations_elementwise.py reach (ce_act_instances), and the
host-side layout checks of their wrappers (no GPU needed: they run before the device check and any launch)."""

import re
import shutil
import subprocess

import pytest
import torch

from ce_act_instances import (ACT_CASES, ACT_IDS, CE_CASES, CE_OTHER, GLU, PLAIN, SIGMOID_GLU, act_instance, act_instances,
                              ce_instance)

_CE = re.compile(r"ce_rows_kernel<(\d+), (\d+), (true|false)>")
_ACT = re.compile(r"(act_fwd_kernel|act_bwd_kernel|act_bwd_bias_kernel)<\(anonymous namespace\)::act::(\w+(?:<\d>)?), "
                  r"(\w+)>")
_OTHER = re.compile(r"\b(ce_count_kernel|ce_mean_kernel)\(")


@pytest.fixture(scope="module")
def built():
    from dolomite_engine_b200 import _lib, build

    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("cuobjdump / c++filt not available")
    build.build()
    res = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    names = re.findall(r"Function (\S+):", res)
    demangled = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout
    ce, act, other = set(), set(), set()
    for line in demangled.splitlines():
        if m := _CE.search(line):
            ce.add(m.group(0))
        elif m := _ACT.search(line):
            act.add(f"{m.group(1)}<{m.group(2)}, {m.group(3)}>")
        elif m := _OTHER.search(line):
            other.add(m.group(1))
    return ce, act, other


def test_every_built_cross_entropy_instance_has_a_case(built):
    """13 ce_rows_kernel instances plus the count and mean kernels; a new instance without a case fails here"""
    ce, _, other = built
    assert len(ce) == 13, sorted(ce)
    assert ce == set(CE_CASES), (sorted(ce - set(CE_CASES)), sorted(set(CE_CASES) - ce))
    assert other == CE_OTHER


def test_every_built_activation_instance_has_a_case(built):
    """45 forward (22 functors x {plain, GLU} + sigmoid-GLU), 44 backward and 44 bias-gradient backward instances"""
    _, act, _ = built
    fam = lambda f: {n for n in act if n.startswith(f + "<")}  # noqa: E731
    assert (len(fam("act_fwd_kernel")), len(fam("act_bwd_kernel")), len(fam("act_bwd_bias_kernel"))) == (45, 44, 44)
    assert act == act_instances(), (sorted(act - act_instances()), sorted(act_instances() - act))


@pytest.mark.parametrize("name", sorted(CE_CASES))
def test_cross_entropy_case_reaches_its_instance(name):
    for V in CE_CASES[name]:
        assert ce_instance(V) == name, V
    assert ce_instance(131073) is None  # wider than one 4-CTA cluster: refused


def test_activation_cases_reach_every_instance_through_every_entry_point():
    assert len({(i, f) for i, f, _ in ACT_CASES.values()}) == 23 * 2 + 1
    # CELU and ELU share one functor; each has its own case
    assert act_instance(ACT_IDS["celu"], PLAIN, "act_fwd") == act_instance(ACT_IDS["elu"], PLAIN, "act_fwd")
    assert act_instance(ACT_IDS["sigmoid"], SIGMOID_GLU, "act_bwd") == act_instance(ACT_IDS["sigmoid"], GLU, "act_bwd")
    assert act_instance(ACT_IDS["sigmoid"], SIGMOID_GLU, "act_fwd") == "act_fwd_kernel<Sigmoid, 2>"


# ------------------------------------------------------------------------------------------------
# wrapper layout checks (CPU tensors: the checks run before the device check and any launch)
# ------------------------------------------------------------------------------------------------
def K():
    from dolomite_engine_b200 import kernels

    return kernels


def _bf(*shape):
    return torch.zeros(*shape, dtype=torch.bfloat16)


T, V = 5, 2051
_LD = 2056  # rows_empty's row stride for V = 2051


def _strided_logits():
    return _bf(T, _LD)[:, :V]


def test_cross_entropy_rejects_a_contiguous_dlogits_for_row_strided_logits():
    """the kernel writes dlogits with the logits' row stride: a contiguous [T, V] buffer is T * (ld - V) elements short"""
    with pytest.raises(ValueError, match="^dlogits must have logits' shape"):
        K().cross_entropy_fwd_bwd(_strided_logits(), torch.zeros(T, dtype=torch.int64), dlogits=_bf(T, V))


def test_cross_entropy_rejects_a_dlogits_of_another_shape():
    with pytest.raises(ValueError, match="^dlogits must have logits' shape"):
        K().cross_entropy_fwd_bwd(_bf(T, 64), torch.zeros(T, dtype=torch.int64), dlogits=_bf(T + 1, 64))


def test_cross_entropy_rejects_logits_without_unit_column_stride():
    with pytest.raises(ValueError, match="^logits must be a 2-D tensor with unit column stride"):
        K().cross_entropy_fwd_bwd(_bf(64, T).t(), torch.zeros(T, dtype=torch.int64))


def test_cross_entropy_rejects_logits_that_are_not_2d():
    with pytest.raises(ValueError, match="^logits must be a 2-D tensor"):
        K().cross_entropy_fwd_bwd(_bf(2, T, 64), torch.zeros(2 * T, dtype=torch.int64))


@pytest.mark.parametrize("bad", ["count", "strided", "dtype"])
def test_cross_entropy_rejects_labels_that_are_not_t_contiguous_int64(bad):
    labels = {"count": torch.zeros(T + 1, dtype=torch.int64), "strided": torch.zeros(2 * T, dtype=torch.int64)[::2],
              "dtype": torch.zeros(T, dtype=torch.int32)}[bad]
    with pytest.raises(ValueError, match="^labels must be a contiguous int64 tensor of 5 elements"):
        K().cross_entropy_fwd_bwd(_bf(T, 64), labels)
    with pytest.raises(ValueError, match="^labels must be a contiguous int64 tensor of 5 elements"):
        K().cross_entropy_rows(_bf(T, 64), labels, torch.zeros(T), torch.zeros(2))


@pytest.mark.parametrize("bad", ["count", "strided"])
def test_cross_entropy_rows_rejects_a_loss_tok_that_is_not_t_contiguous(bad):
    loss_tok = {"count": torch.zeros(T - 1), "strided": torch.zeros(2 * T)[::2]}[bad]
    with pytest.raises(ValueError, match="^loss_tok must be a contiguous tensor of 5 elements"):
        K().cross_entropy_rows(_bf(T, 64), torch.zeros(T, dtype=torch.int64), loss_tok, torch.zeros(2))


def test_cross_entropy_count_rejects_strided_labels():
    with pytest.raises(ValueError, match="^labels must be a contiguous"):
        K().cross_entropy_count(torch.zeros(2 * T, dtype=torch.int64)[::2])


def test_cross_entropy_with_good_layouts_reaches_the_device_check():
    """a row-strided logits with a dlogits of the same strides passes the layout checks; the CPU tensors stop at the
    device check"""
    from dolomite_engine_b200 import _lib

    with pytest.raises(_lib.DolomiteB200Error, match="CUDA tensor"):
        K().cross_entropy_fwd_bwd(_strided_logits(), torch.zeros(T, dtype=torch.int64), dlogits=_strided_logits())
    with pytest.raises(_lib.DolomiteB200Error, match="CUDA tensor"):
        K().cross_entropy_rows(_strided_logits(), torch.zeros(T, dtype=torch.int64), torch.zeros(T), torch.zeros(2))


F = 16


def _wide(cols):
    return _bf(T, cols + 8)[:, :cols]


def _act_calls():
    """(name, call(x, dy, out, bias)) of every activation wrapper: a plain and a GLU form of each entry point"""
    k = K()
    seg = torch.tensor([0, 2, T], dtype=torch.int32)
    return {
        "act_fwd": lambda x, dy, out, b: k.act_fwd(x, ACT_IDS["relu"], PLAIN, out=out),
        "act_fwd_glu": lambda x, dy, out, b: k.act_fwd(x, ACT_IDS["relu"], GLU, out=out),
        "act_bwd": lambda x, dy, out, b: k.act_bwd(dy, x, ACT_IDS["relu"], PLAIN, out=out, bias_grad_accum=b),
        "act_bwd_glu": lambda x, dy, out, b: k.act_bwd(dy, x, ACT_IDS["relu"], GLU, out=out, bias_grad_accum=b),
        "act_bwd_segmented": lambda x, dy, out, b: k.act_bwd_segmented(dy, x, ACT_IDS["relu"], PLAIN, seg,
                                                                         torch.zeros(2, x.shape[1]), out=out),
        "gelu_fwd": lambda x, dy, out, b: k.gelu_fwd(x, out=out),
        "gelu_bwd": lambda x, dy, out, b: k.gelu_bwd(dy, x, out=out, bias_grad_accum=b),
        "swiglu_fwd": lambda x, dy, out, b: k.swiglu_fwd(x, out=out),
        "swiglu_bwd": lambda x, dy, out, b: k.swiglu_bwd(dy, x, out=out, bias_grad_accum=b),
    }


def _glu(name):
    return "glu" in name


def _good(name):
    W = 2 * F if _glu(name) else F
    fwd = "fwd" in name
    return dict(x=_bf(T, W), dy=_bf(T, F), out=_bf(T, F if fwd else W), b=None)


BWD = ["act_bwd", "act_bwd_glu", "act_bwd_segmented", "gelu_bwd", "swiglu_bwd"]
ALL = ["act_fwd", "act_fwd_glu", "gelu_fwd", "swiglu_fwd"] + BWD


@pytest.mark.parametrize("name", ALL)
def test_activation_rejects_a_row_strided_x(name):
    a = _good(name)
    a["x"] = _wide(a["x"].shape[1])
    with pytest.raises(ValueError, match="^x must be a contiguous"):
        _act_calls()[name](**a)


@pytest.mark.parametrize("name", ALL)
def test_activation_rejects_an_out_of_another_layout(name):
    a = _good(name)
    for out in (_wide(a["out"].shape[1]), _bf(T + 1, a["out"].shape[1])):
        with pytest.raises(ValueError, match="^out must be a contiguous"):
            _act_calls()[name](**dict(a, out=out))


@pytest.mark.parametrize("name", BWD)
def test_activation_backward_rejects_a_dy_of_another_layout(name):
    a = _good(name)
    for dy in (_wide(F), _bf(T, F + 8), _bf(F, T).t()):
        with pytest.raises(ValueError, match="^dy must be a contiguous"):
            _act_calls()[name](**dict(a, dy=dy))


@pytest.mark.parametrize("name", ["act_bwd", "act_bwd_glu", "gelu_bwd", "swiglu_bwd"])
def test_activation_backward_rejects_a_bias_gradient_of_another_layout(name):
    a = _good(name)
    W = a["x"].shape[1]
    for b in (torch.zeros(2 * W)[::2], torch.zeros(W + 1)):
        with pytest.raises(ValueError, match="^bias_grad_accum must be a contiguous"):
            _act_calls()[name](**dict(a, b=b))


def test_activation_segmented_rejects_a_bias_gradient_of_another_layout():
    seg = torch.tensor([0, 2, T], dtype=torch.int32)
    for b in (torch.zeros(2, F + 8), torch.zeros(F, 2).t(), torch.zeros(3, F)):
        with pytest.raises(ValueError, match="^bias_grad_accum must be a"):
            K().act_bwd_segmented(_bf(T, F), _bf(T, F), ACT_IDS["relu"], PLAIN, seg, b)


@pytest.mark.parametrize("name", ["act_fwd_glu", "act_bwd_glu", "swiglu_fwd", "swiglu_bwd"])
def test_activation_glu_rejects_an_odd_width(name):
    a = _good(name)
    a["x"] = _bf(T, 2 * F + 1)
    with pytest.raises(ValueError, match="^x must have an even width"):
        _act_calls()[name](**a)


@pytest.mark.parametrize("name", ALL)
def test_activation_with_good_layouts_reaches_the_device_check(name):
    from dolomite_engine_b200 import _lib

    with pytest.raises(_lib.DolomiteB200Error, match="CUDA tensor"):
        _act_calls()[name](**_good(name))
