"""Attention backward (Delta, dK/dV and dQ kernels): long documents whose query / key-value ring wraps many times, query
tiles that end mid-document, and the full C2 size against an fp32 autograd reference, bit-identical from run to run."""

import math

import numpy as np
import pytest
import torch

import oracle.dolomite_oracle as O

pytestmark = pytest.mark.gpu


def K():
    from dolomite_engine_b200 import kernels

    return kernels


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


@pytest.mark.parametrize("lens,ng,g,hd", [([2100], 2, 4, 80), ([200, 330, 95], 2, 1, 64), ([700, 45], 1, 2, 128)])
def test_attention_bwd_long_and_mid_tile_documents_vs_oracle(lens, ng, g, hd):
    """2,100 tokens (GQA 4 q heads per kv group): each key tile walks up to 132 query steps, so the rings wrap many times
    and the two consumer warpgroups can drift apart; lengths 200 / 330 / 95 / 45 end a query tile mid-document in both
    the dK/dV and the dQ kernel"""
    gen = torch.Generator().manual_seed(5)
    T = sum(lens)
    qkv = torch.randn(T, ng * (g + 2) * hd, generator=gen).bfloat16()
    dout = torch.randn(T, ng * g * hd, generator=gen).bfloat16()
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    scale = 1.0 / math.sqrt(hd)
    cfg = O.OracleConfig(n_embd=ng * g * hd, n_head=ng * g, num_key_value_heads=ng,
                         attention_head_type="mha" if g == 1 else "gqa")
    x = qkv.float().requires_grad_(True)
    q, k, v = O.split_qkv_activations(x, cfg)
    O.packed_causal_attention(q, k, v, cu, scale).backward(dout.float())
    cu_d = torch.from_numpy(cu).cuda()
    out, lse = K().attn_varlen_fwd(qkv.cuda(), cu_d, max(lens), ng, g, hd, scale)
    dqkv = K().attn_varlen_bwd(dout.cuda(), qkv.cuda(), out, lse, cu_d, max(lens), ng, g, hd, scale)
    assert rel_l2(dqkv, x.grad) < 1.2e-2


def test_full_size_attention_backward_vs_fp32_autograd_and_run_to_run():
    """C2 attention size (S = 4096, hd 80), 4 heads: dQ, dK, dV against fp32 autograd on the GPU; two calls bit-identical"""
    S, nh, hd = 4096, 4, 80
    g = torch.Generator(device="cuda").manual_seed(21)
    qkv = torch.randn(S, nh * 3 * hd, device="cuda", generator=g).bfloat16()
    dout = torch.randn(S, nh * hd, device="cuda", generator=g).bfloat16()
    cu = torch.tensor([0, S], dtype=torch.int32, device="cuda")
    scale = hd**-0.5
    out, lse = K().attn_varlen_fwd(qkv, cu, S, nh, 1, hd, scale)
    d1 = K().attn_varlen_bwd(dout, qkv, out, lse, cu, S, nh, 1, hd, scale)
    d2 = K().attn_varlen_bwd(dout, qkv, out, lse, cu, S, nh, 1, hd, scale)
    torch.cuda.synchronize()
    assert torch.equal(d1.view(torch.int16), d2.view(torch.int16))

    x = qkv.float().view(S, nh, 3, hd).requires_grad_(True)
    q, k, v = (x[:, :, i].transpose(0, 1) for i in range(3))  # [nh, S, hd]
    s = (q @ k.transpose(1, 2)) * scale
    s = s.masked_fill(torch.triu(torch.ones(S, S, dtype=torch.bool, device="cuda"), 1), float("-inf"))
    o = torch.softmax(s, -1) @ v
    o.transpose(0, 1).reshape(S, nh * hd).backward(dout.float())
    ref = x.grad.view(S, nh * 3 * hd)
    got = d1.float().view(S, nh, 3, hd)
    for i, name in enumerate("qkv"):
        assert rel_l2(got[:, :, i], ref.view(S, nh, 3, hd)[:, :, i]) < 1.2e-2, name
