"""Pin MoE experts with biases against the reference and write tests/golden/moe_bias_*.npz (CPU, fp32).

    python tools/pin_moe_bias.py

Imports the reference read-only (oracle/validate_against_reference.py) and writes:

  moe_bias_layer.npz   the reference's eager SparseMoE (moe/base.py) with add_bias=True, per case "<case>/..." for
                       E 8 / top-2 and E 16 / top-4: input x, parameters (gate, c_fc{,_bias}, c_proj{,_bias}), output y,
                       router logits, and the gradients of x and every parameter for the upstream gradient dy.  Inputs
                       and parameters are bf16 values (stored as their bf16 bit patterns, uint16), so a bf16
                       implementation reads exactly what the fp32 reference computed with; the expert weight gradients
                       keep every GRAD_STRIDE-th element (pin_vocab.subsample).
  moe_bias_model_<act>.npz
                       a two-layer MoEDolomite (rmsnorm, rope, add_bias=True: attention and expert biases) with swiglu and
                       with gelu_pytorch_tanh, run through the reference's SparseMoEBlock with eager experts as
                       tools/pin_vocab.py does, on a packed ragged batch and on a padded batch: loss, logits of every
                       8th real position and every parameter's gradient (see pin_vocab.subsample), plus the biases.

Biases are drawn with std 0.25 (a zero bias would hide a missing one).  Seeds are chosen so that no router logit row has
its k-th and (k+1)-th largest values within a minimum gap: a top-k flip from the last bits of a different summation order
would otherwise decide the result.  The layer's gate weights are scaled by GATE_SCALE (router logits of std ~2) and its
gap, LAYER_GAP, is wide enough for bf16 router logits, so a bf16 implementation routes every token as the reference does;
the model's gap, MODEL_GAP, covers fp32 only (bf16 comparisons pin the routing, oracle.FORCED_ROUTING).  The oracle
(oracle/dolomite_oracle.py) is checked against the reference before anything is written.
"""

from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

GOLDEN = os.path.join(ROOT, "tests", "golden")
BIAS_STD = 0.25
GATE_SCALE = 10.0
LAYER_GAP = 2e-2
MODEL_GAP = 1e-4
LAYER_CASES = {  # name -> (tokens, hidden, n_inner, experts, top-k, activation)
    "e8_k2": (96, 64, 64, 8, 2, "swiglu"),
    "e16_k4": (80, 64, 64, 16, 4, "gelu_pytorch_tanh"),
}
MODEL_KW = dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_head=8, n_inner=192, attention_head_type="mha",
                add_bias=True, num_experts=8, num_experts_per_tok=2, normalization_function="rmsnorm",
                position_embedding_type="rope")
MODEL_ACTS = ("swiglu", "gelu_pytorch_tanh")


def topk_gap(logits: torch.Tensor, k: int) -> float:
    """smallest distance between the k-th and (k+1)-th largest logit of a row"""
    v = logits.detach().float().topk(min(k + 1, logits.shape[1]), dim=-1).values
    return float((v[:, k - 1] - v[:, k]).min()) if logits.shape[1] > k else float("inf")


def biased(params: dict, seed: int) -> dict:
    g = torch.Generator().manual_seed(seed)
    return {k: (torch.randn(v.shape, generator=g) * BIAS_STD if k.endswith(".bias") else v) for k, v in params.items()}


def bf16_bits(t: torch.Tensor) -> np.ndarray:
    return t.detach().bfloat16().view(torch.int16).numpy().view(np.uint16)


def pin_layer(R, O) -> dict:
    import pin_vocab as PV
    from oracle.validate_against_reference import ref_config

    out = {}
    for ci, (name, (T, H, F, E, k, act)) in enumerate(LAYER_CASES.items()):
        cfg = O.OracleConfig(vocab_size=256, n_embd=H, n_layer=1, n_head=4, n_inner=F, num_experts=E, num_experts_per_tok=k,
                             add_bias=True, activation_function=act)
        for seed in range(1000 * (ci + 1), 1000 * (ci + 1) + 500):
            torch.manual_seed(seed)
            moe = R.SparseMoE(ref_config(cfg), use_padding_free_transformer=True, layer_idx=0)
            with torch.no_grad():
                moe.gate.weight.mul_(GATE_SCALE)
                for n, prm in moe.named_parameters():
                    if n.endswith(".bias"):
                        prm.normal_(0.0, BIAS_STD)
                for prm in moe.parameters():
                    prm.copy_(prm.bfloat16().float())
            x = torch.randn(T, H).bfloat16().float().requires_grad_(True)
            y, logits = moe(x)
            if topk_gap(logits, k) > LAYER_GAP:
                break
        else:
            raise SystemExit(f"{name}: no seed without near-tied router logits")
        dy = torch.randn(T, H, generator=torch.Generator().manual_seed(seed + 1))
        y.backward(dy)
        sd = {n: prm.detach().clone() for n, prm in moe.named_parameters()}
        p = {"m." + n: v for n, v in sd.items()}
        p_req = {n: v.clone().requires_grad_(True) for n, v in p.items()}
        x_o = x.detach().clone().requires_grad_(True)
        y_o, logits_o = O.sparse_moe(x_o, p_req, "m.", cfg)
        y_o.backward(dy)
        err = max(((y_o - y).abs().max() / y.abs().max()).item(), ((logits_o - logits).abs().max()).item(),
                  ((x_o.grad - x.grad).abs().max() / x.grad.abs().max()).item(),
                  *[((p_req["m." + n].grad - prm.grad).abs().max() / prm.grad.abs().max()).item()
                    for n, prm in moe.named_parameters()])
        print(f"layer {name}: seed {seed}, top-k gap {topk_gap(logits, k):.2e}, oracle vs reference {err:.2e}")
        assert err < 1e-5, name
        out[f"{name}/shape"] = np.array([T, H, F, E, k], dtype=np.int64)
        out[f"{name}/activation"] = np.array(act)
        out[f"{name}/x"] = bf16_bits(x)
        out[f"{name}/dy"] = dy.numpy()
        out[f"{name}/y"] = y.detach().numpy()
        out[f"{name}/router_logits"] = logits.detach().numpy()
        out[f"{name}/grad:x"] = x.grad.numpy()
        for n, prm in moe.named_parameters():
            out[f"{name}/{n}"] = bf16_bits(sd[n])
            out[f"{name}/grad:{n}"] = PV.subsample(prm.grad).numpy() if prm.dim() == 3 else prm.grad.numpy()
    return out


def pin_model(R, O, act: str) -> dict:
    import pin_vocab as PV

    cfg = O.OracleConfig(activation_function=act, **MODEL_KW)
    tokens, ids, pos, cu, labels = PV.packed_batch(O, cfg.vocab_size)
    ptok, mask, pids, ppos, pcu, plabels = PV.padded_batch(cfg.vocab_size)
    batches = (("packed", (ids, pos, cu, labels)), ("padded", (pids, ppos, pcu, plabels)))
    seen = []
    orig = O.sparse_moe

    def recording(x, p, prefix, c, bf16=False):
        y, logits = orig(x, p, prefix, c, bf16)
        seen.append(topk_gap(logits, c.num_experts_per_tok))
        return y, logits

    for seed in range(42, 62):
        params = biased(O.init_params(cfg, seed=seed), seed + 1000)
        seen.clear()
        O.sparse_moe = recording
        try:
            for _, args in batches:
                O.forward_logits(params, cfg, args[0], args[1], args[2])
        finally:
            O.sparse_moe = orig
        if min(seen) > MODEL_GAP:
            break
    else:
        raise SystemExit(f"{act}: no seed without near-tied router logits")
    fx = {"seed": np.int64(seed), "packed_tokens": tokens, "padded_tokens": ptok, "padded_mask": mask}
    fx.update({f"bias:{k}": v.numpy() for k, v in params.items() if k.endswith(".bias")})
    for batch, args in batches:
        loss, logits, grads = PV.reference_run(R, cfg, params, *args)
        loss_o, logits_o, grads_o = PV.oracle_run(O, cfg, params, *args)
        assert set(grads) == set(grads_o), sorted(set(grads) ^ set(grads_o))
        dl = (logits - logits_o).abs().max().item()
        dg = max(((grads_o[k] - v).abs().max() / (v.abs().max() + 1e-30)).item() for k, v in grads.items())
        print(f"model {act} {batch}: seed {seed}, top-k gap {min(seen):.2e}, loss {loss.item():.6f} vs oracle "
              f"{loss_o.item():.6f}, logits {dl:.2e}, grads (relative to each absmax) {dg:.2e}")
        assert abs(loss.item() - loss_o.item()) <= 1e-5 and dl <= 2e-5 and dg <= 1e-4, (act, batch)
        fx[f"{batch}_loss"] = loss.numpy()
        fx[f"{batch}_logits"] = logits[:: PV.LOGIT_ROW_STRIDE].numpy()
        for k, v in grads.items():
            fx[f"{batch}_grad:{k}"] = PV.subsample(v).numpy()
    return fx


def main() -> None:
    from oracle.validate_against_reference import import_reference

    import oracle.dolomite_oracle as O

    R = import_reference()
    np.savez_compressed(os.path.join(GOLDEN, "moe_bias_layer.npz"), **pin_layer(R, O))
    for act in MODEL_ACTS:
        np.savez_compressed(os.path.join(GOLDEN, f"moe_bias_model_{act}.npz"), **pin_model(R, O, act))
    print("MoE bias fixtures written to", GOLDEN)


if __name__ == "__main__":
    main()
