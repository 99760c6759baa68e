"""CPU: MLP activation names resolve as the reference resolves them, the activation oracle reproduces the reference's
modules (tests/golden/activations.npz, model_act_*.npz from tools/pin_activations.py), and the activation kernels compile
for sm_90a without local memory."""

import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import act_oracle
import oracle.dolomite_oracle as O
from dolomite_engine_b200 import activations as A
from dolomite_engine_b200.engine import check_supported
from dolomite_engine_b200.hf_models import GPTDolomiteConfig, MoEDolomiteConfig
from tools.pin_activations import GRAD_STRIDE, MODEL_CONFIGS

# torch / transformers class the reference builds for each function id
CLASS = {
    A.CELU: "CELU", A.ELU: "ELU", A.GELU: "GELU", A.GELU_TANH: "GELU", A.SELU: "SELU", A.HARDSHRINK: "Hardshrink",
    A.HARDSIGMOID: "Hardsigmoid", A.HARDSWISH: "Hardswish", A.HARDTANH: "Hardtanh", A.LAPLACE: "LaplaceActivation",
    A.LEAKY_RELU: "LeakyReLU", A.LOG_SIGMOID: "LogSigmoid", A.MISH: "Mish", A.RELU: "ReLU",
    A.RELU2: "ReLUSquaredActivation", A.RELU6: "ReLU6", A.SIGMOID: "Sigmoid", A.SILU: "SiLU", A.SOFTPLUS: "Softplus",
    A.SOFTSHRINK: "Softshrink", A.SOFTSIGN: "Softsign", A.TANH: "Tanh", A.TANHSHRINK: "Tanhshrink",
}


@pytest.fixture(scope="module")
def fx(golden_dir):
    return np.load(os.path.join(golden_dir, "activations.npz"))


def _names(fx):
    return [k[len("status_"):] for k in fx.files if k.startswith("status_")]


def _computed(fx):
    return [n for n in _names(fx) if f"fwd32_{n}" in fx.files]


def test_name_resolution_matches_reference(fx):
    names = _names(fx)
    assert len(names) >= 70 and {"relu_glu", "tanh_glu", "gelu_pytorch_tanh_glu", "leaky_reLU"} <= set(names)
    for name in names:
        status = str(fx[f"status_{name}"])
        if status != "accepted":
            assert status == "ValueError", name
            with pytest.raises(ValueError):
                A.resolve(name)
            continue
        module = str(fx[f"module_{name}"])
        if "PReLU" in module or "RReLU" in module or name == "geglu":
            with pytest.raises(NotImplementedError):
                A.resolve(name)
            continue
        act_id, form = A.resolve(name)
        expect = {A.PLAIN: CLASS[act_id], A.GLU: f"GLUActivation({CLASS[act_id]})", A.SIGMOID_GLU: "GLU"}[form]
        assert module == expect, (name, module, act_id, form)
        assert A.is_glu(name) == (form != A.PLAIN)
    # the character-stripping quirk of name.rstrip("_glu"), kept as the reference has it
    for name in ("relu_glu", "gelu_glu", "silu_glu", "elu_glu", "celu_glu", "selu_glu"):
        assert str(fx[f"status_{name}"]) == "ValueError"
    assert A.resolve("tanh_glu") == (A.TANH, A.GLU) and A.resolve("relu6_glu") == (A.RELU6, A.GLU)
    assert A.resolve("gelu_pytorch_tanh_glu") == (A.GELU_TANH, A.GLU) and A.resolve("gelu") == (A.GELU, A.PLAIN)
    assert A.resolve("glu") == A.resolve("sigmoid_glu") == (A.SIGMOID, A.SIGMOID_GLU)
    # the reference builds GLUActivation(GELU) for geglu; the engine keeps rejecting it
    assert str(fx["module_geglu"]) == "GLUActivation(GELU)" and A.reference_rule("geglu") == (A.GELU, A.GLU)


def _dense(**kw):
    d = dict(n_embd=256, n_head=4, attention_head_type="mha", position_embedding_type="rope", activation_function="swiglu",
             normalization_function="rmsnorm", resid_pdrop=0, embd_pdrop=0, attn_pdrop=0, vocab_size=2048)
    d.update(kw)
    return GPTDolomiteConfig(**d)


def test_check_supported_follows_the_name_rule():
    for name in ("gelu", "gelu_pytorch_tanh_glu", "reglu", "relu2", "glu", "sigmoid_glu", "tanh_glu", "laplace", "soft_sign", "mish"):
        check_supported(_dense(activation_function=name))
    for name in ("relu_glu", "silu_glu", "gelu_new", "leaky_relu", "foo"):
        with pytest.raises(ValueError):
            check_supported(_dense(activation_function=name))
    for name, why in (("prelu", "learnable"), ("preglu", "learnable"), ("rrelu", "random"), ("rreglu", "random"),
                      ("geglu", "GeGLU")):
        with pytest.raises(NotImplementedError, match=why):
            check_supported(_dense(activation_function=name))
    moe = dict(n_embd=256, n_head=4, attention_head_type="mha", position_embedding_type="rope",
               normalization_function="rmsnorm", num_experts=16, num_experts_per_tok=2, n_inner=512, add_bias=False,
               resid_pdrop=0, embd_pdrop=0, attn_pdrop=0, vocab_size=2048)
    for name in ("reglu", "softplus", "swiglu"):
        check_supported(MoEDolomiteConfig(activation_function=name, **moe))
    with pytest.raises(NotImplementedError, match="rmsnorm"):
        check_supported(MoEDolomiteConfig(activation_function="reglu", **{**moe, "normalization_function": "layernorm"}))


def _input(fx, name):
    return torch.from_numpy(fx["xg"] if name.endswith("glu") else fx["x"])


def test_oracle_forward_fp32(fx):
    for name in _computed(fx):
        y = act_oracle.activation(_input(fx, name), name)
        np.testing.assert_allclose(y.numpy(), fx[f"fwd32_{name}"], rtol=1e-6, atol=1e-6, err_msg=name)


def test_oracle_forward_bf16_rounding_points_bit_exact(fx):
    for name in _computed(fx):
        y = act_oracle.activation(_input(fx, name), name, bf16=True)
        assert np.array_equal(y.numpy(), fx[f"fwd16_{name}"]), name


def test_oracle_gradient_fp32_including_kinks(fx):
    dy = torch.from_numpy(fx["dy"])
    kinks = fx["kinks"].size
    for name in _computed(fx):
        x = _input(fx, name).clone().requires_grad_(True)
        (act_oracle.activation(x, name) * dy).sum().backward()
        ref = fx[f"grad32_{name}"]
        np.testing.assert_allclose(x.grad.numpy(), ref, rtol=1e-6, atol=1e-6, err_msg=name)
        g = x.grad[0, -64:][:kinks].numpy()  # the kink points (the gate half for GLU forms)
        assert np.array_equal(g, ref[0, -64:][:kinks]), name


@pytest.mark.parametrize("name", list(MODEL_CONFIGS))
@pytest.mark.parametrize("mode", ["uniform", "ragged"])
def test_oracle_model_against_golden(golden_dir, name, mode):
    """the bars of test_oracle_golden.test_model_against_golden, on every parameter's gradient"""
    act_oracle.install()
    cfg = O.OracleConfig(**MODEL_CONFIGS[name])
    fx = np.load(os.path.join(golden_dir, f"model_act_{name}.npz"))
    p = O.init_params(cfg, seed=42)
    if cfg.add_bias:
        g = torch.Generator().manual_seed(7)
        for k in p:
            if k.endswith(".bias"):
                p[k] = torch.randn(p[k].shape, generator=g) * 0.02
    p = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    ram = rpi = mode == "ragged"
    loss, logits = O.pretraining_loss(p, cfg, fx["tokens"], int(fx["eos"]), ram, rpi)
    loss.backward()
    np.testing.assert_allclose(loss.item(), fx[f"{mode}_loss"], rtol=1e-6)
    np.testing.assert_allclose(logits.detach()[::8].numpy(), fx[f"{mode}_logits_rows"], atol=3e-5)
    keys = [k for k in fx.files if k.startswith(f"{mode}_grad:")]
    assert len(keys) >= 8
    for k in keys:
        pname = k.split(":", 1)[1]
        np.testing.assert_allclose(p[pname].grad.flatten()[::GRAD_STRIDE].numpy(), fx[k], atol=1e-6, rtol=1e-4,
                                   err_msg=pname)


def test_activation_kernels_have_no_local_memory():
    """every act_fwd / act_bwd / act_bwd_bias instantiation (22 functors; celu is elu) keeps its values in registers"""
    from dolomite_engine_b200 import _lib, build

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    build.build()
    res = subprocess.run(["cuobjdump", "-res-usage", _lib.LIB_PATH], capture_output=True, text=True).stdout
    found = re.findall(r"Function (\S*act_(?:fwd|bwd|bwd_bias)_kernel\S*):\s*\n\s*(REG:.*)", res)
    assert len(found) == 45 + 44 + 44, len(found)
    for name, usage in found:
        assert int(re.search(r"STACK:(\d+)", usage).group(1)) == 0, (name, usage)
        assert int(re.search(r"LOCAL:(\d+)", usage).group(1)) == 0, (name, usage)
