"""ALiBi slopes (modeling_utils/position_embedding/alibi.py:32-44).

The attention kernels take the slopes as an fp32 [n_heads] device buffer and add bf16(slope * kpos) to the logit of every
key (see include/dolomite_b200.h, dolomite_b200_attn_varlen_fwd_alibi), so the slopes are computed here, on the host, with
the reference's torch arithmetic: an fp32 base raised to int32 powers by torch.pow.  Power-of-two head counts take
base = 2^(-8 / n) and powers 1..n; other counts take the slopes of the largest power of two m < n_heads, then the
odd powers 1, 3, 5, ... of 2^(-8 / 2m) for the remaining heads.
"""

from __future__ import annotations

import math

import torch


def _powers(m: int, start: int, count: int, step: int) -> torch.Tensor:
    # 2 ** (-(2 ** -(log2(m) - 3))) of the reference is exactly 2 ** (-8 / m) in double precision for a power of two m
    base = torch.tensor(2.0 ** (-8.0 / m), dtype=torch.float32)
    return torch.pow(base, torch.arange(start, start + step * count, step, dtype=torch.int32))


def alibi_slopes(n_heads: int) -> torch.Tensor:
    """fp32 [n_heads] CPU tensor, bit-identical to the reference's `Alibi(n_heads).slopes`"""
    if n_heads < 1:
        raise ValueError(f"alibi needs at least one head, got {n_heads}")
    m = 2 ** math.floor(math.log2(n_heads))
    slopes = _powers(m, 1, m, 1)
    if m != n_heads:
        slopes = torch.cat([slopes, _powers(2 * m, 1, min(m, n_heads - m), 2)], dim=0)
    return slopes
