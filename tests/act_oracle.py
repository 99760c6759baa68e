"""Oracle of every MLP activation name the reference accepts, in fp32 and with bf16 rounding emulated at the points the
reference's eager modules round (activations/{base,glu}.py; transformers' LaplaceActivation / ReLUSquaredActivation;
torch's composite softsign and tanhshrink).  Names resolve through dolomite_engine_b200.activations.reference_rule,
the rule tests/test_activations.py pins against the reference.

`install()` points oracle.dolomite_oracle's MLP and MoE expert code at this function.  For swiglu and gelu_pytorch_tanh it
performs the same torch ops as dolomite_oracle.activation, so nothing an existing test computes changes.
"""

from __future__ import annotations

import math

import torch
import torch.nn.functional as F

import oracle.dolomite_oracle as O
from dolomite_engine_b200 import activations as A

LAPLACE_MU, LAPLACE_SIGMA = 0.707107, 0.282095


def _r(x, bf16: bool):
    return x.bfloat16().float() if bf16 else x


def base(x: torch.Tensor, act_id: int, bf16: bool = False) -> torch.Tensor:
    """one plain function on fp32 `x` (bf16-representable values when bf16)"""
    r = lambda t: _r(t, bf16)  # noqa: E731
    if act_id in (A.CELU, A.ELU):  # CELU(alpha=1) is torch.elu(x, 1, 1, 1)
        return r(F.elu(x))
    if act_id == A.LAPLACE:
        # a bf16 `x - mu` rounds the scalar mu to bf16 first
        mu = torch.tensor(LAPLACE_MU).bfloat16().float().item() if bf16 else LAPLACE_MU
        z = r(r(x - mu).div(LAPLACE_SIGMA * math.sqrt(2.0)))
        return r(0.5 * r(1.0 + r(torch.erf(z))))
    if act_id == A.RELU2:
        return r(torch.square(F.relu(x)))
    if act_id == A.SOFTSIGN:
        return r(x / r(x.abs() + 1))
    if act_id == A.TANHSHRINK:
        return r(x - r(x.tanh()))
    fn = {
        A.GELU: F.gelu, A.GELU_TANH: lambda t: F.gelu(t, approximate="tanh"), A.SELU: F.selu,
        A.HARDSHRINK: F.hardshrink, A.HARDSIGMOID: F.hardsigmoid, A.HARDSWISH: F.hardswish, A.HARDTANH: F.hardtanh,
        A.LEAKY_RELU: F.leaky_relu, A.LOG_SIGMOID: F.logsigmoid, A.MISH: F.mish, A.RELU: F.relu, A.RELU6: F.relu6,
        A.SIGMOID: torch.sigmoid, A.SILU: F.silu, A.SOFTPLUS: F.softplus, A.SOFTSHRINK: F.softshrink, A.TANH: torch.tanh,
    }[act_id]
    return r(fn(x))


def apply(x: torch.Tensor, act_id: int, form: int, bf16: bool = False) -> torch.Tensor:
    if form == A.PLAIN:
        return base(x, act_id, bf16)
    u, g = x.chunk(2, dim=-1)
    if form == A.SIGMOID_GLU:  # nn.GLU: one rounding of u * sigmoid(g)
        return _r(F.glu(x, dim=-1), bf16)
    return _r(u * base(g, act_id, bf16), bf16)


def activation(x: torch.Tensor, name: str, bf16: bool = False) -> torch.Tensor:
    """activations/__init__.py get_activation_function(name)(x)"""
    return apply(x, *A.reference_rule(name), bf16=bf16)


def install() -> None:
    O.activation = activation
