"""Pin MoE blocks of any expert count and width against the reference and write tests/golden/moe_shapes_*.npz (CPU, fp32).

    python tools/pin_moe_shapes.py

Imports the reference read-only (oracle/validate_against_reference.py) and writes:

  moe_shapes_layer.npz  the reference's eager SparseMoE (moe/base.py) for LAYER_CASES, per case "<case>/...": expert
                        counts that are not multiples of 8 (3, 20 and the single expert) and widths that are multiples of
                        8 but not of 64.  Input x, parameters, output y, router logits, and the gradients of x and every
                        parameter for the upstream gradient dy.  x and the parameters are bf16 values drawn from the case's
                        seed by tests/moe_shapes_inputs.py, so only the seed is stored; the expert weight gradients are
                        sampled by moe_shapes_inputs.subsample (every 61st element).
  moe_shapes_model_<name>.npz
                        two-layer MoEDolomite models of MODELS run through the reference's SparseMoEBlock with eager
                        experts as tools/pin_vocab.py does, on a packed ragged batch and on a padded batch: loss, logits of
                        every 8th real position, every parameter's gradient (moe_shapes_inputs.subsample), the non-zero
                        biases, and for the padded batch each layer's router logits over the real tokens and the
                        load-balancing loss of transformers' `load_balancing_loss_func` on them (the value the reference's
                        `get_moe_loss` forms when no padding is passed).

Seeds are chosen as in tools/pin_moe_bias.py: no router logit row has its k-th and (k+1)-th largest values within
LAYER_GAP (layers; wide enough for bf16 router logits) or MODEL_GAP (models; bf16 comparisons pin the routing).  The
oracle (oracle/dolomite_oracle.py) is checked against the reference before anything is written.
"""

from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from moe_shapes_inputs import subsample  # noqa: E402
from pin_moe_bias import BIAS_STD, LAYER_GAP, MODEL_GAP, topk_gap  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
# name -> (tokens, hidden, n_inner, experts, top-k, activation, add_bias).  Hidden widths have a valid head dim (16), so
# the same shapes also run as one-layer models on the GPU.
LAYER_CASES = {
    "e3_k2": (96, 80, 40, 3, 2, "swiglu", True),
    "e20_k4": (80, 144, 200, 20, 4, "gelu_pytorch_tanh", False),
    "e1_k1": (64, 48, 24, 1, 1, "gelu_pytorch_tanh", True),
}
MODELS = {
    "e6_swiglu": dict(vocab_size=512, n_positions=256, n_embd=160, n_layer=2, n_head=5, n_inner=424,
                      attention_head_type="mha", activation_function="swiglu", add_bias=False, num_experts=6,
                      num_experts_per_tok=2, normalization_function="rmsnorm", position_embedding_type="rope"),
    "e12_gelu": dict(vocab_size=512, n_positions=256, n_embd=96, n_layer=2, n_head=3, n_inner=200,
                     attention_head_type="mha", activation_function="gelu_pytorch_tanh", add_bias=True, num_experts=12,
                     num_experts_per_tok=8, normalization_function="rmsnorm", position_embedding_type="learned_absolute"),
}


def pin_layer(R, O) -> dict:
    from oracle.validate_against_reference import ref_config

    from moe_shapes_inputs import layer_inputs

    out = {}
    for ci, (name, (T, H, F, E, k, act, bias)) in enumerate(LAYER_CASES.items()):
        cfg = O.OracleConfig(vocab_size=256, n_embd=H, n_layer=1, n_head=H // 16, n_inner=F, num_experts=E,
                             num_experts_per_tok=k, add_bias=bias, activation_function=act)
        moe = R.SparseMoE(ref_config(cfg), use_padding_free_transformer=True, layer_idx=0)
        for seed in range(1000 * (ci + 1), 1000 * (ci + 1) + 500):
            x, params = layer_inputs(T, H, F, E, act, bias, seed)
            moe.load_state_dict(params)
            moe.zero_grad(set_to_none=True)
            x = x.requires_grad_(True)
            y, logits = moe(x)
            if topk_gap(logits, k) > LAYER_GAP:
                break
        else:
            raise SystemExit(f"{name}: no seed without near-tied router logits")
        dy = torch.randn(T, H, generator=torch.Generator().manual_seed(seed + 1))
        y.backward(dy)
        sd = {n: prm.detach().clone() for n, prm in moe.named_parameters()}
        p_req = {"m." + n: v.clone().requires_grad_(True) for n, v in sd.items()}
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
        out[f"{name}/add_bias"] = np.int64(bias)
        out[f"{name}/seed"] = np.int64(seed)  # tests/moe_shapes_inputs.layer_inputs draws x and the parameters from it
        out[f"{name}/dy"] = dy.numpy()
        out[f"{name}/y"] = y.detach().numpy()
        out[f"{name}/router_logits"] = logits.detach().numpy()
        out[f"{name}/grad:x"] = x.grad.numpy()
        for n, prm in moe.named_parameters():
            out[f"{name}/grad:{n}"] = subsample(prm.grad).numpy() if prm.dim() == 3 else prm.grad.numpy()
    return out


def _recording_block_class(router: list):
    """the reference's SparseMoEBlock with eager experts, returning its hidden states and appending its router logits"""
    from dolomite_engine.hf_models.models.moe_dolomite.layer import SparseMoEBlock

    class MoEBlock(SparseMoEBlock):
        def __init__(self, rc, normalization_implementation, attention_implementation, padding_free, layer_idx):
            super().__init__(rc, normalization_implementation, attention_implementation, padding_free, "eager", layer_idx)
            self.layer_idx_ = layer_idx

        def forward(self, h, attention_mask=None, rope_cos_sin=None):
            out = super().forward(h, attention_mask=attention_mask, rope_cos_sin=rope_cos_sin, output_router_logits=True)
            router.append((self.layer_idx_, out[1].detach()))
            return out[0]

    return MoEBlock


def reference_router_logits(R, cfg, params, ids, pos, cu) -> list[torch.Tensor]:
    """per layer [real tokens, E] router logits of the reference, in token order"""
    from oracle.validate_against_reference import reference_forward

    router: list = []
    Rm = types.SimpleNamespace(**{**vars(R), "GPTDolomiteBlock": _recording_block_class(router)})
    with torch.no_grad():
        reference_forward(Rm, cfg, {k: v.clone() for k, v in params.items()}, ids, pos, cu)
    return [torch.cat([lg.reshape(-1, cfg.num_experts) for i, lg in router if i == layer], 0) for layer in range(cfg.n_layer)]


def pin_model(R, O, name: str, kw: dict) -> dict:
    import pin_vocab as PV
    from transformers.models.mixtral.modeling_mixtral import load_balancing_loss_func

    cfg = O.OracleConfig(**kw)
    tokens, ids, pos, cu, labels = PV.packed_batch(O, cfg.vocab_size)
    ptok, mask, pids, ppos, pcu, plabels = PV.padded_batch(cfg.vocab_size)
    batches = (("packed", (ids, pos, cu, labels)), ("padded", (pids, ppos, pcu, plabels)))
    seen = []
    orig = O.sparse_moe

    def recording(x, p, prefix, c, bf16=False):
        y, logits = orig(x, p, prefix, c, bf16)
        seen.append(topk_gap(logits, c.num_experts_per_tok))
        return y, logits

    for seed in range(42, 142):
        params = O.init_params(cfg, seed=seed)
        if cfg.add_bias:
            g = torch.Generator().manual_seed(seed + 1000)
            params = {k: (torch.randn(v.shape, generator=g) * BIAS_STD if k.endswith(".bias") else v) for k, v in params.items()}
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
        raise SystemExit(f"{name}: no seed without near-tied router logits")
    fx = {"seed": np.int64(seed), "packed_tokens": tokens, "padded_tokens": ptok, "padded_mask": mask}
    fx.update({f"bias:{k}": v.numpy() for k, v in params.items() if k.endswith(".bias")})
    for batch, args in batches:
        loss, logits, grads = PV.reference_run(R, cfg, params, *args)
        loss_o, logits_o, grads_o = PV.oracle_run(O, cfg, params, *args)
        assert set(grads) == set(grads_o), sorted(set(grads) ^ set(grads_o))
        dl = (logits - logits_o).abs().max().item()
        dg = max(((grads_o[k] - v).abs().max() / (v.abs().max() + 1e-30)).item() for k, v in grads.items())
        print(f"model {name} {batch}: seed {seed}, top-k gap {min(seen):.2e}, loss {loss.item():.6f} vs oracle "
              f"{loss_o.item():.6f}, logits {dl:.2e}, grads (relative to each absmax) {dg:.2e}")
        assert abs(loss.item() - loss_o.item()) <= 1e-5 and dl <= 2e-5 and dg <= 1e-4, (name, batch)
        fx[f"{batch}_loss"] = loss.numpy()
        fx[f"{batch}_logits"] = logits[:: PV.LOGIT_ROW_STRIDE].numpy()
        for k, v in grads.items():
            fx[f"{batch}_grad:{k}"] = subsample(v).numpy()
    router = reference_router_logits(R, cfg, params, pids, ppos, pcu)
    _, router_o = _oracle_router(O, cfg, params, pids, ppos, pcu)
    dr = max((a - b).abs().max().item() for a, b in zip(router, router_o))
    aux = load_balancing_loss_func(tuple(r.double() for r in router), cfg.num_experts, cfg.num_experts_per_tok)
    print(f"model {name} padded: router logits vs oracle {dr:.2e}, aux {float(aux):.9f}")
    assert dr <= 2e-5, name
    for layer, r in enumerate(router):
        fx[f"padded_router_logits:{layer}"] = r.numpy()
    fx["padded_aux"] = np.float64(aux)
    return fx


def _oracle_router(O, cfg, params, ids, pos, cu):
    from moe_aux_oracle import forward_logits_with_router

    with torch.no_grad():
        return forward_logits_with_router(params, cfg, ids, pos, cu)


def main() -> None:
    from oracle.validate_against_reference import import_reference

    import oracle.dolomite_oracle as O

    R = import_reference()
    np.savez_compressed(os.path.join(GOLDEN, "moe_shapes_layer.npz"), **pin_layer(R, O))
    for name, kw in MODELS.items():
        np.savez_compressed(os.path.join(GOLDEN, f"moe_shapes_model_{name}.npz"), **pin_model(R, O, name, kw))
    print("MoE shape fixtures written to", GOLDEN)


if __name__ == "__main__":
    main()
