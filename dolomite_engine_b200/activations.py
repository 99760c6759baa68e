"""activation_function names -> (CUDA function id, form), by the reference's own rule
(hf_models/modeling_utils/activations/{__init__,base,glu}.py: get_activation_function).

    is_glu(name) = name.endswith("glu")
    GLU:  "glu" / "sigmoid_glu" -> nn.GLU;  else _GLU_BASE_MAPPING[name], else name.rstrip("_glu") for a name ending in
          "_glu" (rstrip strips the CHARACTERS _ g l u, so "relu_glu" -> "re" is rejected while "tanh_glu" -> "tanh" is
          accepted), then the base table
    else: the base table

The rule is copied as it is, so that a reference config either runs here or fails the same way.  Names the reference
rejects raise ValueError.  PReLU / RReLU (and their GLU forms) raise NotImplementedError, and so does "geglu", which
check_supported has rejected with NotImplementedError since the first release; the exact-erf GELU runs as the plain
"gelu", and "gelu_pytorch_tanh_glu" is the GELU-gated MLP.
"""

from __future__ import annotations

# ids of include/dolomite_b200.h (enum DOLO_ACT_*)
CELU, ELU, GELU, GELU_TANH, SELU, HARDSHRINK, HARDSIGMOID, HARDSWISH, HARDTANH, LAPLACE, LEAKY_RELU, LOG_SIGMOID, MISH, \
    RELU, RELU2, RELU6, SIGMOID, SILU, SOFTPLUS, SOFTSHRINK, SOFTSIGN, TANH, TANHSHRINK = range(23)
# forms (DOLO_ACT_PLAIN / _GLU / _SIGMOID_GLU)
PLAIN, GLU, SIGMOID_GLU = 0, 1, 2

# activations/base.py _BASE_ACTIVATIONS (keys exactly as the reference spells them)
_BASE = {
    "celu": CELU, "elu": ELU, "gelu": GELU, "gelu_pytorch_tanh": GELU_TANH, "selu": SELU, "hard_shrink": HARDSHRINK,
    "hard_sigmoid": HARDSIGMOID, "hard_swish": HARDSWISH, "hard_tanh": HARDTANH, "laplace": LAPLACE,
    "leaky_reLU": LEAKY_RELU, "log_sigmoid": LOG_SIGMOID, "mish": MISH, "prelu": None, "relu": RELU, "relu2": RELU2,
    "relu_squared": RELU2, "relu6": RELU6, "rrelu": None, "sigmoid": SIGMOID, "silu": SILU, "swish": SILU,
    "softplus": SOFTPLUS, "soft_plus": SOFTPLUS, "soft_shrink": SOFTSHRINK, "soft_sign": SOFTSIGN, "tanh": TANH,
    "tanh_shrink": TANHSHRINK,
}
# activations/glu.py _GLU_BASE_MAPPING
_GLU_BASE_MAPPING = {
    "ceglu": "celu", "eglu": "elu", "geglu": "gelu", "miglu": "mish", "mishglu": "mish", "preglu": "prelu",
    "reglu": "relu", "rreglu": "rrelu", "seglu": "selu", "swiglu": "swish",
}
_NOT_IMPLEMENTED_NAMES = {
    "geglu": "GeGLU stays unsupported, as check_supported has always reported it (gelu_pytorch_tanh_glu is the GELU-gated "
             "MLP, with the tanh approximation)",
}
_NOT_IMPLEMENTED = {
    "prelu": "PReLU has a learnable weight, which would add a parameter to the MLP block layout and the state dict",
    "rrelu": "RReLU draws random slopes from torch's RNG in training mode",
}


def is_glu(name: str) -> bool:
    """activations/glu.py is_glu: the c_fc output is [u | g], twice the MLP width"""
    return name.endswith("glu")


def resolve(name: str) -> tuple[int, int]:
    """(function id, form) of an activation_function name the engine trains; ValueError where the reference raises it"""
    if name in _NOT_IMPLEMENTED_NAMES:
        raise NotImplementedError(f"activation_function={name!r}: {_NOT_IMPLEMENTED_NAMES[name]}")
    return reference_rule(name)


def reference_rule(name: str) -> tuple[int, int]:
    """(function id, form) the reference's rule gives, without the engine's refusal of geglu (the oracle computes it)"""
    if is_glu(name):
        if name in ("glu", "sigmoid_glu"):
            return SIGMOID, SIGMOID_GLU
        if name in _GLU_BASE_MAPPING:
            base = _GLU_BASE_MAPPING[name]
        elif name.endswith("_glu"):
            base = name.rstrip("_glu")
        else:
            raise ValueError(f"invalid activation function {name!r}")
        form = GLU
    else:
        base, form = name, PLAIN
    if base not in _BASE:
        raise ValueError(f"invalid activation function {name!r}")
    if base in _NOT_IMPLEMENTED:
        raise NotImplementedError(f"activation_function={name!r}: {_NOT_IMPLEMENTED[base]}")
    return _BASE[base], form
