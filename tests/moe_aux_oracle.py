"""CPU oracle of the MoE load-balancing loss: transformers' Mixtral `load_balancing_loss_func` (called by the reference's
`get_moe_loss`, moe_dolomite/base.py:24-43) written out, and the MoEDolomite forward with each layer's router logits.

    p = softmax(logits) over all E experts, C_e = #(layer, token, slot) selecting e, P_e = sum_{layer, token} p_e,
    N = layers * real tokens,  aux = E * sum_e C_e P_e / N^2,  loss = CE + coef * aux

`attention_mask` drops padding tokens from every sum (the masked form of load_balancing_loss_func); `selected` gives the
experts of each layer's routing plan (top-k on the raw logits, moe/base.py:142-151) instead of a top-k of p.
"""

from __future__ import annotations

import torch

import oracle.dolomite_oracle as O


def load_balancing_loss(router_logits, num_experts: int, top_k: int, attention_mask=None, selected=None):
    """router_logits: per-layer [tokens, E] tensors (differentiable; computed in their own dtype after a float cast)"""
    logits = torch.cat([lg.float() if lg.dtype in (torch.bfloat16, torch.float16) else lg for lg in router_logits], 0)
    p = torch.softmax(logits, dim=-1)
    if selected is None:
        selected = torch.topk(p, top_k, dim=-1).indices
    else:
        selected = torch.cat(list(selected), 0)
    one_hot = torch.nn.functional.one_hot(selected, num_experts).to(p.dtype)  # [tokens, k, E]
    if attention_mask is not None:
        keep = attention_mask.reshape(-1).to(p.dtype).repeat(len(router_logits))
        p = p * keep[:, None]
        one_hot = one_hot * keep[:, None, None]
        n = keep.sum()
    else:
        n = torch.tensor(float(logits.shape[0]), dtype=p.dtype)
    counts = one_hot.sum((0, 1)).detach()  # C_e: no gradient
    return num_experts * (counts * p.sum(0)).sum() / (n * n)


def moe_loss(ce, aux, coef: float):
    """get_moe_loss (moe_dolomite/base.py:24-43): (CE + coef * aux, aux); CE None (no labels) -> (None, aux)"""
    return (None if ce is None else ce + coef * aux), aux


def forward_logits_with_router(p: dict, cfg: O.OracleConfig, input_ids, position_ids, cu_seqlens, bf16: bool = False):
    """O.forward_logits, also returning the router logits of every layer (what SparseMoE returns next to its output)"""
    router = []
    sparse_moe = O.sparse_moe

    def recording(x, p_, prefix, cfg_, bf16_=False):
        out, logits = sparse_moe(x, p_, prefix, cfg_, bf16_)
        router.append(logits)
        return out, logits

    O.sparse_moe = recording  # O.block looks the function up at call time
    try:
        logits = O.forward_logits(p, cfg, input_ids, position_ids, cu_seqlens, bf16)
    finally:
        O.sparse_moe = sparse_moe
    return logits, tuple(router)
