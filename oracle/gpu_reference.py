"""GPU baseline: the reference's own PyTorch / flash-attn training path, restated with library kernels only.

TEST / MEASUREMENT INFRASTRUCTURE ONLY (same rule as oracle/dolomite_oracle.py): nothing under dolomite_engine_b200/
imports this module; `bench.py --impl gpu_reference` (and the `gpu_reference` key of the normal bench line) times it next
to the H100 engine on the same GPU, tests use it as a bf16 cross-check.  It answers: what the
unmodified reference would run on the same GPU --

    nn.Linear                    -> F.linear on bf16 copies of fp32 parameters (cuBLAS; FSDP MixedPrecision(param_dtype=bf16),
                                    distributed/__init__.py:146-159)
    PaddingFreeAttention         -> flash_attn.flash_attn_varlen_func(causal=True)     (attention/padding_free.py:51-62)
    RMSNorm / RoPE / SwiGLU / CE -> the eager tensor expressions of normalization/rmsnorm/base.py:18-25,
                                    position_embedding/rope.py:104-114, activations/glu.py:26-28, model_wrapper/pretraining.py:107-127
    MoE                          -> the eager SparseMoE loop (moe_dolomite/moe/base.py:108-173); scattermoe is not installable here
    backward                     -> torch autograd;  optimizer -> torch.optim.AdamW (optimization/optimizer.py:55-84 `TorchAdamW`),
                                    torch.nn.utils.clip_grad_norm_ (train_utils.py:99-103)

The reference package itself does not import under torch 2.11 / transformers 5.5 (DESIGN.md section 2), so its leaf
arithmetic is restated here; none of this repository's kernels are on this path.
"""

from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def _std(cfg: dict) -> tuple[float, float]:
    std = cfg.get("initializer_range", 0.02)
    return std, std / math.sqrt(2 * cfg["n_layer"])


def init_params(cfg: dict, device, seed: int = 1) -> dict[str, torch.nn.Parameter]:
    """fp32 master parameters under the reference's state-dict names (same shapes as engine._block_specs / _root_specs)"""
    g = torch.Generator(device=device).manual_seed(seed)
    H, Fi, V, L = cfg["n_embd"], cfg["n_inner"], cfg["vocab_size"], cfg["n_layer"]
    hd = H // cfg["n_head"]
    nkv = cfg.get("num_key_value_heads") or cfg["n_head"]
    qkv = H + 2 * nkv * hd
    E = cfg.get("num_experts", 0) if cfg.get("model_type") == "moe_dolomite" else 0
    std, std_proj = _std(cfg)
    bias = bool(cfg.get("add_bias", True))

    def n(*shape, sd):
        return torch.nn.Parameter(torch.randn(*shape, generator=g, device=device) * sd)

    p = {"transformer.wte.weight": n(V, H, sd=cfg.get("initializer_range", 0.02))}
    for i in range(L):
        pre = f"transformer.h.{i}."
        p[pre + "ln_1.weight"] = torch.nn.Parameter(torch.ones(H, device=device))
        p[pre + "ln_2.weight"] = torch.nn.Parameter(torch.ones(H, device=device))
        p[pre + "attn.c_attn.weight"] = n(qkv, H, sd=std)
        p[pre + "attn.c_proj.weight"] = n(H, H, sd=std_proj)
        if E:
            p[pre + "mlp.gate.weight"] = n(E, H, sd=std)
            p[pre + "mlp.c_fc.weight"] = n(E, 2 * Fi, H, sd=std)
            p[pre + "mlp.c_proj.weight"] = n(E, H, Fi, sd=std_proj)
        else:
            p[pre + "mlp.c_fc.weight"] = n(2 * Fi, H, sd=std)
            p[pre + "mlp.c_proj.weight"] = n(H, Fi, sd=std_proj)
        if bias and not E:
            p[pre + "attn.c_attn.bias"] = torch.nn.Parameter(torch.zeros(qkv, device=device))
            p[pre + "attn.c_proj.bias"] = torch.nn.Parameter(torch.zeros(H, device=device))
            p[pre + "mlp.c_fc.bias"] = torch.nn.Parameter(torch.zeros(2 * Fi, device=device))
            p[pre + "mlp.c_proj.bias"] = torch.nn.Parameter(torch.zeros(H, device=device))
    p["transformer.ln_f.weight"] = torch.nn.Parameter(torch.ones(H, device=device))
    if not cfg.get("tie_word_embeddings", True):
        p["lm_head.weight"] = n(V, H, sd=cfg.get("initializer_range", 0.02))
    return p


def rmsnorm(x, w, eps):
    """normalization/rmsnorm/base.py:18-25: fp32 statistics, cast back, then the weight"""
    dt = x.dtype
    xf = x.to(torch.float32)
    var = xf.pow(2).mean(-1, keepdim=True)
    xf = xf * torch.rsqrt(var + eps)
    return w * xf.to(dt)


def rotate_half(x):
    x1, x2 = torch.chunk(x, 2, dim=-1)
    return torch.cat((-x2, x1), dim=-1)


def apply_rope(x, cos, sin):
    """position_embedding/rope.py:104-114"""
    return (x * cos) + (rotate_half(x) * sin)


def rope_tables(hd: int, n_positions: int, base: float, device):
    inv_freq = 1.0 / (base ** (torch.arange(0, hd, 2, dtype=torch.float32, device=device) / hd))
    t = torch.arange(n_positions, dtype=torch.float32, device=device)
    freqs = torch.outer(t, inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos().to(torch.bfloat16), emb.sin().to(torch.bfloat16)


def eager_sparse_moe(x, gate_w, wfc, wproj, top_k: int):
    """SparseMoE.forward (moe_dolomite/moe/base.py:108-173) with moe_implementation: eager"""
    T, H = x.shape
    logits = F.linear(x, gate_w)
    w, idx = logits.topk(top_k, dim=-1)
    w = torch.softmax(w.float(), dim=-1).to(x.dtype)
    out = torch.zeros(T, H, dtype=x.dtype, device=x.device)
    for e in range(wfc.shape[0]):
        tok, slot = torch.nonzero(idx == e, as_tuple=True)
        if tok.numel() == 0:
            continue
        h = F.linear(x[tok], wfc[e])
        u, g = h.chunk(2, dim=-1)
        h = F.linear(u * F.silu(g), wproj[e])
        out = out.index_add(0, tok, h * w[tok, slot].unsqueeze(-1))
    return out


def forward_loss(p: dict, cfg: dict, input_ids, position_ids, cu_seqlens, max_seqlen: int, labels, tables):
    """GPTDolomiteModel / MoEDolomiteModel forward with PaddingFreeAttention + mean CE on fp32-upcast logits"""
    from flash_attn import flash_attn_varlen_func

    bf = torch.bfloat16
    H, nh = cfg["n_embd"], cfg["n_head"]
    hd = H // nh
    nkv = cfg.get("num_key_value_heads") or nh
    g = nh // nkv
    eps = cfg.get("layer_norm_epsilon", 1e-5)
    E = cfg.get("num_experts", 0) if cfg.get("model_type") == "moe_dolomite" else 0
    cos_t, sin_t = tables
    cos, sin = cos_t[position_ids].unsqueeze(1), sin_t[position_ids].unsqueeze(1)
    W = lambda k: p[k].to(bf)  # noqa: E731  (FSDP param_dtype=bf16: compute sees bf16 copies of the fp32 parameters)
    Wb = lambda k: p[k].to(bf) if k in p else None  # noqa: E731
    T = input_ids.numel()
    h = F.embedding(input_ids, W("transformer.wte.weight"))
    for i in range(cfg["n_layer"]):
        pre = f"transformer.h.{i}."
        res = h
        x = rmsnorm(h, W(pre + "ln_1.weight"), eps)
        qkv = F.linear(x, W(pre + "attn.c_attn.weight"), Wb(pre + "attn.c_attn.bias"))
        qkv = qkv.view(T, nkv, (g + 2) * hd)  # attention/padding_free.py:79-116
        q, k, v = qkv.split((g * hd, hd, hd), dim=-1)
        q = apply_rope(q.reshape(T, nh, hd), cos, sin)
        k = apply_rope(k, cos, sin)
        a = flash_attn_varlen_func(q, k, v, cu_seqlens_q=cu_seqlens, cu_seqlens_k=cu_seqlens, max_seqlen_q=max_seqlen,
                                   max_seqlen_k=max_seqlen, dropout_p=0.0, softmax_scale=1.0 / math.sqrt(hd), causal=True)
        a = F.linear(a.reshape(T, H), W(pre + "attn.c_proj.weight"), Wb(pre + "attn.c_proj.bias"))
        h = a + res
        res = h
        x = rmsnorm(h, W(pre + "ln_2.weight"), eps)
        if E:
            m = eager_sparse_moe(x, W(pre + "mlp.gate.weight"), W(pre + "mlp.c_fc.weight"), W(pre + "mlp.c_proj.weight"),
                                 cfg["num_experts_per_tok"])
        else:
            f = F.linear(x, W(pre + "mlp.c_fc.weight"), Wb(pre + "mlp.c_fc.bias"))
            u, gt = f.chunk(2, dim=-1)
            m = F.linear(u * F.silu(gt), W(pre + "mlp.c_proj.weight"), Wb(pre + "mlp.c_proj.bias"))
        h = res + m
    h = rmsnorm(h, W("transformer.ln_f.weight"), eps)
    head = W("transformer.wte.weight") if cfg.get("tie_word_embeddings", True) else W("lm_head.weight")
    logits = F.linear(h, head)
    return F.cross_entropy(logits.float(), labels, ignore_index=-100)


def time_train_steps(cfg: dict, seq: int, mbs: int, steps: int, warmup: int, device, docs_per_row: int = 1) -> dict:
    """K full training steps (fwd + bwd + clip + AdamW) on synthetic packed tokens already resident in HBM; CUDA-event timed"""
    p = init_params(cfg, device)
    params = list(p.values())
    opt = torch.optim.AdamW(params, lr=1e-5, betas=(0.9, 0.95), eps=1e-10, weight_decay=0.1)
    hd = cfg["n_embd"] // cfg["n_head"]
    tables = rope_tables(hd, max(seq, cfg.get("n_positions", seq)), float(cfg.get("rope_theta", 10000)), device)
    T = mbs * seq
    gen = torch.Generator(device=device).manual_seed(0)
    doc = seq // docs_per_row
    cu = torch.arange(0, T + 1, doc, dtype=torch.int32, device=device)
    pos = torch.arange(T, device=device) % doc

    def step():
        ids = torch.randint(0, cfg["vocab_size"], (T,), generator=gen, device=device)
        labels = torch.randint(0, cfg["vocab_size"], (T,), generator=gen, device=device)
        opt.zero_grad(set_to_none=True)
        loss = forward_loss(p, cfg, ids, pos, cu, doc, labels, tables)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(params, 1.0)
        opt.step()
        return loss

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    return {"ms_per_step": ms, "tokens_per_s": T / (ms / 1e3), "micro_batch_size": mbs, "seq_len": seq, "loss": float(loss.item()),
            "peak_hbm_gb": torch.cuda.max_memory_allocated(device) / 1e9}
