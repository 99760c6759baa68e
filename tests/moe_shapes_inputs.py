"""Inputs of the MoE layer fixtures of tools/pin_moe_shapes.py (tests/golden/moe_shapes_layer.npz), drawn from a seed
so that the fixture stores only results: bf16-exact parameters under the reference's SparseMoE names and the layer input.
Also the gradient sampling of every moe_shapes fixture (`subsample`)."""

from __future__ import annotations

import numpy as np
import torch

GATE_STD = 0.2  # router logits of std ~2 at unit inputs: top-k gaps that bf16 resolves
WEIGHT_STD = 0.05
BIAS_STD = 0.25  # a zero bias would hide a missing one
FULL_GRAD = 4096  # gradients up to this size are kept whole
GRAD_STRIDE = 61  # larger ones keep every 61st element: a prime, so the samples of a [E, rows, cols] tensor cycle through
# every column and every expert (a stride that divides the row length would only ever see a few columns)


def subsample(g: torch.Tensor) -> torch.Tensor:
    """the flattened gradient as the moe_shapes fixtures store it"""
    g = g.flatten()
    return g if g.numel() <= FULL_GRAD else g[::GRAD_STRIDE]


def _bf16(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(a.astype(np.float32)).bfloat16().float()


def layer_inputs(T: int, H: int, F: int, E: int, act: str, add_bias: bool, seed: int):
    """-> (x [T, H], {name: parameter}) with names gate.weight, c_fc.weight, c_fc.bias, c_proj.weight, c_proj.bias"""
    g = np.random.default_rng(seed)
    fc_out = 2 * F if act.endswith("glu") else F
    p = {"gate.weight": _bf16(g.standard_normal((E, H)) * GATE_STD),
         "c_fc.weight": _bf16(g.standard_normal((E, fc_out, H)) * WEIGHT_STD)}
    if add_bias:
        p["c_fc.bias"] = _bf16(g.standard_normal((E, fc_out)) * BIAS_STD)
    p["c_proj.weight"] = _bf16(g.standard_normal((E, H, F)) * WEIGHT_STD)
    if add_bias:
        p["c_proj.bias"] = _bf16(g.standard_normal((E, H)) * BIAS_STD)
    x = _bf16(g.standard_normal((T, H)))
    return x, p
