"""Wide attention heads on one GPU: forward and backward of the packed attention at equal model width, with head dim 128
against 160 / 192 / 256, decode, and a training step of the 3B research baseline's shape.

    python tools/bench_attention_wide.py

- attention: K.attn_varlen_fwd and K.attn_varlen_bwd (Delta, dK/dV, dQ), median of 50 launches after warm-up; width 3072
  as 24 x 128, 16 x 192 and 12 x 256 (MHA and MQA), width 2560 as 20 x 128 and 16 x 160 (MHA), each on T = 4096 as one
  document and as 4 documents of 1024.  TFLOP/s is algorithmic: 2 causal matmuls forward, 5 backward, of 2 * S^2/2 * hd
  flops per head and document.
- decode: K.attn_decode at cache length 4096, batch 8; GB/s counts the K and V cache bytes read.
- step: forward + backward of a 4-layer model of base.yml's shape (n_embd 3072, 12 heads, MQA, RoPE, RMSNorm, SwiGLU,
  biases, n_inner 8192, vocab 50304) on 2 x 2048 tokens, median of 10 steps; tokens/s.

Prints one JSON line per measurement, then the card's name, power limit and max SM clock from the same run.
"""

from __future__ import annotations

import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_attention import gpu_info, time_call  # noqa: E402

# name: (n_groups, q_per_group, head_dim)
ATTN = {
    "3072_mha_24x128": (24, 1, 128), "3072_mha_16x192": (16, 1, 192), "3072_mha_12x256": (12, 1, 256),
    "3072_mqa_24x128": (1, 24, 128), "3072_mqa_16x192": (1, 16, 192), "3072_mqa_12x256": (1, 12, 256),
    "2560_mha_20x128": (20, 1, 128), "2560_mha_16x160": (16, 1, 160),
}
DOCS = {"1x4096": [4096], "4x1024": [1024] * 4}


def attention(ng, g, hd, lens):
    import numpy as np
    import torch

    from dolomite_engine_b200 import kernels as K

    gen = torch.Generator(device="cuda").manual_seed(0)
    T = sum(lens)
    qkv = torch.randn(T, ng * (g + 2) * hd, device="cuda", generator=gen).bfloat16()
    dout = torch.randn(T, ng * g * hd, device="cuda", generator=gen).bfloat16()
    cu = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)).cuda()
    scale = 1.0 / math.sqrt(hd)
    out, lse = K.attn_varlen_fwd(qkv, cu, max(lens), ng, g, hd, scale)
    dqkv = torch.empty_like(qkv)
    fwd_ms = time_call(lambda: K.attn_varlen_fwd(qkv, cu, max(lens), ng, g, hd, scale, out=out))
    bwd_ms = time_call(lambda: K.attn_varlen_bwd(dout, qkv, out, lse, cu, max(lens), ng, g, hd, scale, dqkv=dqkv))
    per = 2 * sum(L * L / 2 for L in lens) * hd * ng * g
    return {"fwd_ms": round(fwd_ms, 4), "fwd_tflops": round(2 * per / fwd_ms / 1e9, 1), "bwd_ms": round(bwd_ms, 4),
            "bwd_tflops": round(5 * per / bwd_ms / 1e9, 1)}


def decode(ng, g, hd, L=4096, B=8):
    import torch

    from dolomite_engine_b200 import kernels as K

    gen = torch.Generator(device="cuda").manual_seed(0)
    kc = torch.randn(B, L, ng * hd, device="cuda", generator=gen).bfloat16()
    vc = torch.randn(B, L, ng * hd, device="cuda", generator=gen).bfloat16()
    qkv = torch.randn(B, ng * (g + 2) * hd, device="cuda", generator=gen).bfloat16()
    lens = torch.full((B,), L, dtype=torch.int32, device="cuda")
    ms = time_call(lambda: K.attn_decode(qkv, kc, vc, lens, ng, g, hd, hd**-0.5))
    return {"us": round(ms * 1e3, 2), "GB/s": round(2 * kc.numel() * 2 / ms / 1e6, 1)}


def step(n_layer=4, B=2, S=2048):
    import torch

    from dolomite_engine_b200.hf_models import GPTDolomiteConfig, GPTDolomiteForCausalLM

    cfg = GPTDolomiteConfig(vocab_size=50304, n_positions=S, n_embd=3072, n_layer=n_layer, n_head=12, n_inner=8192,
                            attention_head_type="mqa", num_key_value_heads=1, position_embedding_type="rope",
                            normalization_function="rmsnorm", activation_function="swiglu", add_bias=True,
                            resid_pdrop=0.0, embd_pdrop=0.0, attn_pdrop=0.0)
    model = GPTDolomiteForCausalLM(cfg, seed=42, use_padding_free_transformer=True)
    model.assume_unit_loss_grad = True
    T = B * S
    ids = torch.randint(0, cfg.vocab_size, (T,), device="cuda")
    pos = torch.arange(S, device="cuda").repeat(B)
    cu = torch.arange(0, T + 1, S, dtype=torch.int32, device="cuda")
    labels = torch.randint(0, cfg.vocab_size, (T,), device="cuda")

    def one():
        model.engine.zero_grad()
        model.forward_pretraining_loss(ids, pos, cu, S, labels).backward()

    ms = time_call(one, iters=10, warmup=3)
    return {"layers": n_layer, "tokens": T, "ms": round(ms, 2), "tokens_per_s": round(T / ms * 1e3, 1)}


def main():
    import torch

    assert torch.cuda.is_available(), "bench_attention_wide needs a GPU"
    for name, (ng, g, hd) in ATTN.items():
        for dname, lens in DOCS.items():
            print(json.dumps({"attention": name, "docs": dname, **attention(ng, g, hd, lens)}), flush=True)
    for name in ("3072_mha_24x128", "3072_mha_12x256", "3072_mqa_24x128", "3072_mqa_12x256", "2560_mha_16x160",
                 "3072_mha_16x192"):
        ng, g, hd = ATTN[name]
        print(json.dumps({"decode": name, "L": 4096, "batch": 8, **decode(ng, g, hd)}), flush=True)
    print(json.dumps({"step": "base.yml shape, 4 layers", **step()}), flush=True)
    print(json.dumps(gpu_info()))


if __name__ == "__main__":
    main()
