"""Pin the oracle against the UNMODIFIED reference and (re)generate tests/golden/*.npz.

Runs only in the build container (needs /root/reference, read-only).  The reference package does not import as a
whole under torch 2.11 / transformers 5.5 (SURVEY.md section 8c), but its leaf modules do with two import shims and
a duck-typed config; those leaf modules are the ground truth here:

    GPTDolomiteBlock (eager Attention + MLP + RMSNorm), RoPE / apply_rotary_pos_emb, SparseMoE,
    ParameterizedEmbedding, interleave/split helpers, convert_padding_free_lists_to_tensors (logic), F.cross_entropy.

The padding-free (packed) semantics are obtained from the reference by running each document as its own batch row
through the eager attention with the reference's causal mask -- the equivalence the reference itself certifies in
tests/hf_models/single_gpu/hf_models/gpt_dolomite_test.py:90-137.

    python oracle/validate_against_reference.py            # validate + write fixtures
"""

from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = "/root/reference"
GOLDEN = os.path.join(ROOT, "tests", "golden")


def import_reference():
    if not os.path.isdir(REF):
        raise SystemExit("reference not present; this script only runs in the build container")
    sys.modules["fla"] = None  # is_fla_available() -> False (utils/packages.py:130-144)
    from torch.distributed.tensor import placement_types

    if not hasattr(placement_types, "_Partial"):
        placement_types._Partial = placement_types.Partial
    try:
        import torch.distributed._tensor.placement_types as pt2

        if not hasattr(pt2, "_Partial"):
            pt2._Partial = pt2.Partial
    except Exception:
        pass
    sys.path.insert(0, REF)
    import dolomite_engine.hf_models  # noqa: F401
    from dolomite_engine.hf_models.modeling_utils import RMSNorm, RoPE, apply_rotary_pos_emb  # noqa: F401
    from dolomite_engine.hf_models.modeling_utils import get_normalization_function
    from dolomite_engine.hf_models.modeling_utils.position_embedding.rope import YaRNScaledRoPE
    from dolomite_engine.hf_models.models.gpt_dolomite.layer import GPTDolomiteBlock
    from dolomite_engine.hf_models.models.moe_dolomite.moe.base import SparseMoE

    return types.SimpleNamespace(
        GPTDolomiteBlock=GPTDolomiteBlock, RMSNorm=RMSNorm, RoPE=RoPE, apply_rotary_pos_emb=apply_rotary_pos_emb,
        SparseMoE=SparseMoE, get_normalization_function=get_normalization_function, YaRNScaledRoPE=YaRNScaledRoPE,
    )


def ref_config(cfg):
    """duck-typed config carrying the attributes the leaf modules read"""
    return types.SimpleNamespace(
        n_embd=cfg.n_embd, hidden_size=cfg.n_embd, n_head=cfg.n_head, num_attention_heads=cfg.n_head,
        num_key_value_heads=cfg.num_key_value_heads, n_inner=cfg.n_inner, n_layer=cfg.n_layer,
        num_hidden_layers=cfg.n_layer, activation_function=cfg.activation_function,
        attention_head_type=cfg.attention_head_type, resid_pdrop=0.0, embd_pdrop=0.0, attn_pdrop=0.0,
        normalization_function=cfg.normalization_function, layer_norm_epsilon=cfg.layer_norm_epsilon,
        initializer_range=cfg.initializer_range, scale_attn_weights=cfg.scale_attn_weights,
        attention_multiplier=cfg.attention_multiplier, attention_softmax_in_fp32=True, add_bias=cfg.add_bias,
        position_embedding_type=cfg.position_embedding_type, rope_theta=cfg.rope_theta, m_emb=cfg.m_emb,
        m_width=cfg.m_width, m_residual=cfg.m_residual, init_method=cfg.init_method,
        num_experts=cfg.num_experts, num_experts_per_tok=cfg.num_experts_per_tok, vocab_size=cfg.vocab_size,
        n_positions=cfg.n_positions, max_position_embeddings=cfg.n_positions,
    )


def reference_forward(R, cfg, params, input_ids, position_ids, cu_seqlens):
    """reference leaf modules glued as gpt_dolomite/base.py:170-244 + main.py:143-177; one document per batch row"""
    rc = ref_config(cfg)
    blocks = []
    for i in range(cfg.n_layer):
        b = R.GPTDolomiteBlock(rc, "torch", "eager", False, i)
        sd = {k[len(f"transformer.h.{i}."):]: v for k, v in params.items() if k.startswith(f"transformer.h.{i}.")}
        b.load_state_dict(sd)
        blocks.append(b)
    ln_f = R.get_normalization_function(cfg.normalization_function, cfg.n_embd, eps=cfg.layer_norm_epsilon)  # base.py:57-61
    ln_f.load_state_dict({k[len("transformer.ln_f."):]: v for k, v in params.items() if k.startswith("transformer.ln_f.")})
    rope = R.RoPE(cfg.head_dim, max_position_embeddings=cfg.n_positions, base=cfg.rope_theta)
    wte = params["transformer.wte.weight"].clone().requires_grad_(True)
    learned = cfg.position_embedding_type == "learned_absolute"
    wpe = params["transformer.wpe.weight"].clone().requires_grad_(True) if learned else None
    ids = torch.as_tensor(input_ids, dtype=torch.long)
    pos = torch.as_tensor(position_ids, dtype=torch.long)
    outs = []
    for d in range(len(cu_seqlens) - 1):
        s, e = int(cu_seqlens[d]), int(cu_seqlens[d + 1])
        if e == s:
            continue
        h = torch.nn.functional.embedding(ids[s:e], wte).unsqueeze(0)
        if learned:  # base.py:351-372: inputs_embeds + wpe(position_ids)
            h = h + torch.nn.functional.embedding(pos[s:e], wpe).unsqueeze(0)
        if cfg.m_emb is not None:
            h = h * cfg.m_emb
        n = e - s
        cs = None
        if cfg.position_embedding_type == "rope":
            cos, sin = rope(cfg.n_positions, dtype=torch.float32, device=None)
            cs = (cos[pos[s:e]].unsqueeze(0).unsqueeze(1), sin[pos[s:e]].unsqueeze(0).unsqueeze(1))  # base.py:289-296
        causal = torch.ones(n, n, dtype=torch.bool).tril()[None, None]
        mask = torch.where(causal, torch.tensor(0.0), torch.tensor(torch.finfo(torch.float32).min))  # base.py:587-596
        for b in blocks:
            h = b(h, attention_mask=mask, rope_cos_sin=cs)
        outs.append(h[0])
    h = ln_f(torch.cat(outs, 0))
    head = wte if cfg.tie_word_embeddings else params["lm_head.weight"]
    logits = torch.nn.functional.linear(h, head)
    if cfg.m_width is not None:
        logits = logits / cfg.m_width
    ln_f_grads = lambda: {"transformer.ln_f." + k: v.grad for k, v in ln_f.named_parameters()}  # noqa: E731
    return logits, blocks, wte, wpe, ln_f_grads


def close(a, b, atol, what):
    err = (a - b).abs().max().item()
    ref = b.abs().max().item()
    status = "ok" if err <= atol else "MISMATCH"
    print(f"  {what:55s} max_abs_err={err:.3e} (ref absmax {ref:.3e}) [{status}]")
    if err > atol:
        raise SystemExit(f"oracle disagrees with the reference on {what}")


CONFIGS = {
    # C1 of SURVEY section 8d
    "c1": dict(vocab_size=2048, n_positions=1024, n_embd=256, n_layer=2, n_head=4, n_inner=1024,
               activation_function="swiglu", attention_head_type="mha", add_bias=False),
    # granite-style multipliers + bias + gqa, head_dim 16
    "gqa_bias_mup": dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_head=8, num_key_value_heads=2,
                         n_inner=256, attention_head_type="gqa", add_bias=True, m_emb=12.0, m_width=2.0,
                         m_residual=0.22, attention_multiplier=0.015625, tie_word_embeddings=False),
    "mqa_gelu": dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=1, n_head=4, n_inner=512,
                     attention_head_type="mqa", activation_function="gelu_pytorch_tanh", add_bias=True),
    # the StarCoder / bigcode shape of configs/pretraining-examples (dropout 0): LayerNorm + tanh-GELU + learned positions + MQA
    "bigcode": dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_head=8, n_inner=512,
                    attention_head_type="mqa", activation_function="gelu_pytorch_tanh", add_bias=True,
                    normalization_function="layernorm", position_embedding_type="learned_absolute"),
}


def main():
    import oracle.dolomite_oracle as O

    R = import_reference()
    os.makedirs(GOLDEN, exist_ok=True)
    torch.manual_seed(0)
    print("== leaf ops ==")
    x = torch.randn(37, 256)
    w = 1 + 0.1 * torch.randn(256)
    rn = R.RMSNorm(256, eps=1e-5)
    rn.load_state_dict({"weight": w})
    close(O.rmsnorm(x, w, 1e-5), rn(x), 1e-6, "RMSNorm fp32")
    close(O.rmsnorm(x.bfloat16().float(), w.bfloat16().float(), 1e-5, bf16=True),
          rn.to(torch.bfloat16)(x.bfloat16()).float(), 0.0, "RMSNorm bf16 rounding points")
    rope = R.RoPE(80, max_position_embeddings=128, base=10000)
    cos, sin = rope(128, dtype=torch.float32, device=None)
    oc, os_ = O.rope_tables(80, 128, 10000)
    close(oc, cos, 0.0, "RoPE cos table")
    close(os_, sin, 0.0, "RoPE sin table")
    q = torch.randn(128, 4, 80)
    close(O.apply_rope(q, oc.unsqueeze(1), os_.unsqueeze(1)), R.apply_rotary_pos_emb(q, (cos.unsqueeze(1), sin.unsqueeze(1))),
          1e-6, "apply_rotary_pos_emb fp32")
    cb, sb = rope(128, dtype=torch.bfloat16, device=None)
    ocb, osb = O.rope_tables(80, 128, 10000, bf16=True)
    close(O.apply_rope(q.bfloat16().float(), ocb.unsqueeze(1), osb.unsqueeze(1), bf16=True),
          R.apply_rotary_pos_emb(q.bfloat16(), (cb.unsqueeze(1), sb.unsqueeze(1))).float(), 0.0, "apply_rotary_pos_emb bf16")

    for hd_, npos, base, factor, orig in [(80, 512, 10000, 4.0, 128), (128, 1024, 500000, 8.0, 256), (64, 256, 10000, 1.0, 256)]:
        yr = R.YaRNScaledRoPE(hd_, max_position_embeddings=npos, base=base, scale=factor, original_max_position_embeddings=orig)
        yc, ys = yr(npos, dtype=torch.float32, device=None)
        oc2, os2 = O.rope_tables(hd_, npos, base, rope_scaling={"factor": factor, "original_max_position_embeddings": orig})
        close(oc2, yc, 0.0, f"YaRN cos table hd{hd_} x{factor}")
        close(os2, ys, 0.0, f"YaRN sin table hd{hd_} x{factor}")

    for name, kw in CONFIGS.items():
        print(f"== model {name} ==")
        cfg = O.OracleConfig(**kw)
        params = O.init_params(cfg, seed=42)
        if cfg.add_bias:  # non-zero biases so that the bias path is actually checked
            g = torch.Generator().manual_seed(7)
            for k in params:
                if k.endswith(".bias"):
                    params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        rng = np.random.default_rng(1234)
        seq, mbs = (128, 2) if name == "c1" else (64, 2)
        tokens = rng.integers(0, cfg.vocab_size, size=(mbs, seq + 1), dtype=np.int64)
        eos = 7
        tokens[0, 20] = eos
        tokens[1, 5] = eos
        tokens[1, 40] = eos
        fixtures = {"tokens": tokens, "eos": np.int64(eos)}
        for mode, (ram, rpi) in {"uniform": (False, False), "ragged": (True, True)}.items():
            inp, labels = O.split_tokens(tokens)
            b = O.prepare_model_inputs(inp.copy(), eos, ram, rpi)
            logits_ref, blocks, wte, wpe, ln_f_grads = reference_forward(R, cfg, params, b["input_ids"], b["position_ids"],
                                                                         b["cu_seqlens"])
            lab = torch.as_tensor(np.ascontiguousarray(labels).reshape(-1))
            loss_ref = torch.nn.functional.cross_entropy(logits_ref, lab)  # model_wrapper/pretraining.py:124-125
            loss_ref.backward()
            p_req = {k: v.clone().requires_grad_(True) for k, v in params.items()}
            loss_o, logits_o = O.pretraining_loss(p_req, cfg, tokens, eos, ram, rpi)
            loss_o.backward()
            close(logits_o.detach(), logits_ref.detach(), 2e-5, f"{mode}: logits")
            close(loss_o.detach(), loss_ref.detach(), 1e-6, f"{mode}: loss")
            g_ref = {f"transformer.h.{i}.{k}": v.grad for i, blk in enumerate(blocks) for k, v in blk.named_parameters()}
            g_ref["transformer.wte.weight"] = wte.grad
            g_ref.update(ln_f_grads())
            if wpe is not None:
                g_ref["transformer.wpe.weight"] = wpe.grad
            for k, gr in g_ref.items():
                if k == "transformer.wte.weight" and not cfg.tie_word_embeddings:
                    pass
                close(p_req[k].grad, gr, 5e-6 + 1e-4 * gr.abs().max().item(), f"{mode}: grad {k}")
            fixtures[f"{mode}_cu_seqlens"] = b["cu_seqlens"]
            fixtures[f"{mode}_position_ids"] = b["position_ids"]
            fixtures[f"{mode}_max_seqlen"] = np.int64(b["max_seqlen"])
            fixtures[f"{mode}_loss"] = loss_ref.detach().numpy()
            fixtures[f"{mode}_logits_rows"] = logits_ref.detach()[::8].numpy()
            fixtures[f"{mode}_grad_ln_f"] = p_req["transformer.ln_f.weight"].grad.numpy()
            fixtures[f"{mode}_grad_c_attn_0"] = g_ref["transformer.h.0.attn.c_attn.weight"][::4].numpy()
            fixtures[f"{mode}_grad_wte_rows"] = g_ref["transformer.wte.weight"][tokens[0, :16]].numpy()
        np.savez_compressed(os.path.join(GOLDEN, f"model_{name}.npz"), **fixtures)

    print("== MoE (eager SparseMoE, moe_dolomite/moe/base.py) ==")
    # own seed: the fixture must not depend on how many model configurations ran above (their module constructors draw
    # from the global generator).  NOTE: tests/golden/moe_layer.npz in git predates this line (it was produced after three
    # model configurations); regenerating gives a different, equally valid fixture.
    torch.manual_seed(4321)
    cfg = O.OracleConfig(vocab_size=256, n_embd=64, n_layer=1, n_head=4, n_inner=128, num_experts=8,
                         num_experts_per_tok=2, add_bias=False)
    rc = ref_config(cfg)
    moe = R.SparseMoE(rc, use_padding_free_transformer=True, layer_idx=0)
    sd = {k: v.detach().clone() for k, v in moe.state_dict().items()}
    x = torch.randn(96, 64)
    y_ref, logits_ref = moe(x)
    p = {"m.gate.weight": sd["gate.weight"], "m.c_fc.weight": sd["c_fc.weight"], "m.c_proj.weight": sd["c_proj.weight"]}
    y_o, logits_o = O.sparse_moe(x, p, "m.", cfg)
    close(y_o, y_ref.detach(), 1e-6, "SparseMoE output")
    close(logits_o, logits_ref.detach(), 1e-6, "SparseMoE router logits")
    w_o, idx_o, _ = O.moe_route(x, p["m.gate.weight"], 2)
    moe_path = os.path.join(GOLDEN, "moe_layer.npz")
    if os.path.exists(moe_path) and not os.environ.get("REGENERATE_MOE_FIXTURE"):
        moe_path = os.path.join("/tmp", "moe_layer_regenerated.npz")  # keep the committed fixture stable
    np.savez_compressed(
        moe_path, x=x.numpy(), gate=sd["gate.weight"].numpy(), c_fc=sd["c_fc.weight"].numpy(),
        c_proj=sd["c_proj.weight"].numpy(), y=y_ref.detach().numpy(), router_logits=logits_ref.detach().numpy(),
        counts=O.moe_expert_counts(idx_o, 8),
    )

    print("== bookkeeping (bit exact) ==")
    from dolomite_engine.hf_models.modeling_utils.attention.utils import (
        interleave_query_key_value_tensor_for_gqa, interleave_query_key_value_tensor_for_mha,
        split_query_key_value_tensor_for_gqa, split_query_key_value_tensor_for_mha,
    )

    cfg = O.OracleConfig(n_embd=64, n_head=8, num_key_value_heads=2, attention_head_type="gqa")
    qw, kw_, vw = torch.randn(64, 64), torch.randn(16, 64), torch.randn(16, 64)
    ref_i = interleave_query_key_value_tensor_for_gqa(qw, kw_, vw, 8, 2, 8)
    assert torch.equal(O.interleave_qkv(qw, kw_, vw, cfg), ref_i)
    for a, b_ in zip(O.split_qkv(ref_i, cfg), split_query_key_value_tensor_for_gqa(ref_i, 8, 2, 8)):
        assert torch.equal(a, b_)
    cfg = O.OracleConfig(n_embd=64, n_head=8, attention_head_type="mha")
    qw, kw_, vw = torch.randn(64, 64), torch.randn(64, 64), torch.randn(64, 64)
    ref_i = interleave_query_key_value_tensor_for_mha(qw, kw_, vw, 8, 8)
    assert torch.equal(O.interleave_qkv(qw, kw_, vw, cfg), ref_i)
    for a, b_ in zip(O.split_qkv(ref_i, cfg), split_query_key_value_tensor_for_mha(ref_i, 8)):
        assert torch.equal(a, b_)
    print("  interleave/split qkv (mha, gqa): exact")
    # hf_models/utils.py:20-57 needs a CUDA device in the reference; restate its three integer lines here
    ids = [[5, 6, 7, 8, 9, 1, 2, 3, 4, 5], [9, 8, 7, 6, 5]]
    seqlens = torch.tensor([0] + [len(x) for x in ids])
    ref_cu = seqlens.cumsum(dim=-1).to(torch.int32).numpy()
    o = O.convert_padding_free_lists_to_tensors(ids, labels=ids)
    assert np.array_equal(o["cu_seqlens"], ref_cu) and o["cu_seqlens"].dtype == np.int32
    assert o["max_seqlen"] == int(seqlens.max())
    assert np.array_equal(o["position_ids"], np.array(list(range(10)) + list(range(5))))
    np.savez_compressed(os.path.join(GOLDEN, "bookkeeping.npz"), cu_seqlens=ref_cu, max_seqlen=np.int64(10),
                        position_ids=o["position_ids"], input_ids=o["input_ids"],
                        shift_labels=O.finetune_shift_labels(o["labels"], o["cu_seqlens"]))
    print("  convert_padding_free_lists_to_tensors: exact")
    print("oracle pinned; fixtures written to", GOLDEN)


if __name__ == "__main__":
    main()
