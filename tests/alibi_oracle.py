"""CPU oracle of ALiBi (modeling_utils/position_embedding/alibi.py, gpt_dolomite/base.py:261-287): the per-(head, key)
bias and causal packed attention with that bias.  The slopes are dolomite_engine_b200.alibi.alibi_slopes, which
tests/test_alibi.py pins bit for bit against the reference's.  `install(slopes, bf16)` makes oracle.dolomite_oracle's model
forward (block -> packed_causal_attention) add the bias, as act_oracle.install does for the activations.

TEST INFRASTRUCTURE ONLY, like oracle/dolomite_oracle.py.
"""

from __future__ import annotations

import contextlib

import numpy as np
import torch

import oracle.dolomite_oracle as O


def key_positions(attention_mask: np.ndarray | None, batch: int, length: int) -> torch.Tensor:
    """alibi.py:22-27: arange(L) without a mask, (cumsum(mask) - 1) with masked keys at 0 with one -> int64 [B, L]"""
    if attention_mask is None:
        return torch.arange(length).unsqueeze(0).expand(batch, -1)
    m = torch.as_tensor(np.asarray(attention_mask)).long()
    return (m.cumsum(-1) - 1).masked_fill(m == 0, 0)


def alibi_bias(slopes: torch.Tensor, kpos: torch.Tensor, bf16: bool) -> torch.Tensor:
    """alibi.py:29-30: slope * kpos in fp32, cast to the hidden-state dtype -> fp32 [B, n_heads, L] (bf16 values if bf16)"""
    b = slopes.view(1, -1, 1) * kpos.unsqueeze(1)
    return b.to(torch.bfloat16).float() if bf16 else b


def packed_causal_attention(q, k, v, cu_seqlens, scale: float, slopes: torch.Tensor, bias_bf16: bool, bf16: bool = False,
                            dropout_site=None, dropout_p: float = 0.0) -> torch.Tensor:
    """O.packed_causal_attention with the fp32 logits scale * q.k + bias[h, key index inside the document].  Runs on the
    device of q / k / v (a CUDA device for documents whose [heads, L, L] scores do not fit the host comfortably)."""
    T, nh, hd = q.shape
    dev = q.device
    slopes = slopes.to(dev)
    g = nh // k.shape[1]
    k = k.repeat_interleave(g, dim=1) if g > 1 else k
    v = v.repeat_interleave(g, dim=1) if g > 1 else v
    out = torch.zeros(T, nh, hd, dtype=torch.float32, device=dev)
    for d in range(len(cu_seqlens) - 1):
        s, e = int(cu_seqlens[d]), int(cu_seqlens[d + 1])
        if e == s:
            continue
        qd, kd, vd = q[s:e].transpose(0, 1), k[s:e].transpose(0, 1), v[s:e].transpose(0, 1)
        bias = alibi_bias(slopes, torch.arange(e - s, device=dev).unsqueeze(0), bias_bf16)[0]  # [nh, L]
        sc = torch.matmul(qd, kd.transpose(1, 2)) * scale + bias.unsqueeze(1)
        mask = torch.ones(e - s, e - s, dtype=torch.bool, device=dev).tril()
        p = torch.softmax(sc.masked_fill(~mask, float("-inf")).float(), dim=-1)
        if O.DROPOUT is not None and dropout_p and dropout_site is not None:
            tok = np.arange(s, e)
            p = p * torch.stack([O.DROPOUT.attn_scale(dropout_site, h, tok, tok, dropout_p) for h in range(nh)]).to(dev)
        out[s:e] = torch.matmul(O._r(p, bf16), vd).transpose(0, 1)
    return O._r(out.reshape(T, nh * hd), bf16)


@contextlib.contextmanager
def install(slopes: torch.Tensor, bias_bf16: bool = True):
    """O.forward_logits / O.pretraining_loss add the ALiBi bias while the context is active"""
    saved = O.packed_causal_attention

    def attn(q, k, v, cu_seqlens, scale, bf16=False, dropout_site=None, dropout_p=0.0):
        return packed_causal_attention(q, k, v, cu_seqlens, scale, slopes, bias_bf16, bf16, dropout_site, dropout_p)

    O.packed_causal_attention = attn
    try:
        yield
    finally:
        O.packed_causal_attention = saved
