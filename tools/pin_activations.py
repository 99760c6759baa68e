"""Pin the MLP activations against the reference (needs the reference checkout; writes tests/golden fixtures).

    python tools/pin_activations.py

tests/golden/activations.npz, for every name of NAMES:
  status_<name>          "accepted" or the exception type get_activation_function raises
  module_<name>          the module it builds: "<Class>" or "GLUActivation(<Class>)"
  for each accepted name (PReLU / RReLU excluded: see dolomite_engine_b200/activations.py; geglu is pinned like the
  others although the engine rejects it):
  fwd32_<name>, fwd16_<name>, grad32_<name>   forward in fp32, forward of the module in eager bf16, fp32 autograd
                                              gradient of sum(y * dy)
  inputs (bf16 values): x (plain, [R, 64]), xg (GLU forms, [R, 128] = [u | x]), dy ([R, 64]); x[0, :len(kinks)] are
  the kink points of KINKS.
tests/golden/model_act_<config>.npz: logits, loss and gradients of the reference's leaf modules for MODEL_CONFIGS, in the
format of oracle/validate_against_reference.py's model fixtures, with every parameter's gradient subsampled.
"""

from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

GOLDEN = os.path.join(ROOT, "tests", "golden")

_BASE = ["celu", "elu", "gelu", "gelu_pytorch_tanh", "selu", "hard_shrink", "hard_sigmoid", "hard_swish", "hard_tanh",
         "laplace", "leaky_reLU", "log_sigmoid", "mish", "prelu", "relu", "relu2", "relu_squared", "relu6", "rrelu",
         "sigmoid", "silu", "swish", "softplus", "soft_plus", "soft_shrink", "soft_sign", "tanh", "tanh_shrink"]
NAMES = (_BASE + [b + "_glu" for b in _BASE]
         + ["glu", "sigmoid_glu", "ceglu", "eglu", "geglu", "miglu", "mishglu", "preglu", "reglu", "rreglu", "seglu", "swiglu",
            "gelu_new", "leaky_relu", "Relu", "hardswish", "foo", "foo_glu", "fooglu", "silu_glu_glu", "_glu", ""])
NAMES = list(dict.fromkeys(NAMES))

# every non-differentiable point of the functions, their thresholds and neighbours, then a bf16 sweep
KINKS = [0.0, -0.0, 0.5, -0.5, 1.0, -1.0, 3.0, -3.0, 6.0, -6.0, 20.0, 19.875, 20.125, 0.70703125, 1e-3, -1e-3]
GRAD_STRIDE = 16  # every parameter gradient is pinned at every 16th element of its flattened form
MODEL_CONFIGS = {
    # the gpt_bigcode shape with exact-erf GELU (model_conversion_families: import_config_bigcode)
    "bigcode_gelu": dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_head=8, n_inner=512,
                         attention_head_type="mqa", activation_function="gelu", add_bias=True,
                         normalization_function="layernorm", position_embedding_type="learned_absolute"),
    "gelu_tanh_glu_gqa_bias": dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_head=8,
                                   num_key_value_heads=2, n_inner=256, attention_head_type="gqa",
                                   activation_function="gelu_pytorch_tanh_glu", add_bias=True),
    "relu2": dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=1, n_head=4, n_inner=512, attention_head_type="mha",
                  activation_function="relu2", add_bias=False),
    "glu": dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=1, n_head=4, n_inner=256, attention_head_type="mha",
                activation_function="glu", add_bias=True),
}


def input_grid() -> tuple[torch.Tensor, ...]:
    sweep = torch.linspace(-8, 8, 64 * 24 - len(KINKS)).bfloat16().float()
    g = torch.Generator().manual_seed(11)
    wide = (torch.randn(64 * 8, generator=g) * 12).bfloat16().float()
    x = torch.cat([torch.tensor(KINKS), sweep, wide]).bfloat16().float().reshape(-1, 64)
    u = torch.randn(x.shape, generator=g).bfloat16().float()
    dy = torch.randn(x.shape, generator=g).bfloat16().float()
    return x, torch.cat([u, x], dim=1), dy


def describe(mod) -> str:
    if type(mod).__name__ == "GLUActivation":
        return f"GLUActivation({type(mod.base_activation).__name__})"
    return type(mod).__name__


def main():
    from oracle.validate_against_reference import import_reference, reference_forward

    import_reference()
    from dolomite_engine.hf_models.modeling_utils.activations import get_activation_function

    x, xg, dy = input_grid()
    out = {"x": x.numpy(), "xg": xg.numpy(), "dy": dy.numpy(), "kinks": torch.tensor(KINKS).bfloat16().float().numpy()}
    for name in NAMES:
        try:
            mod = get_activation_function(name)
        except Exception as e:  # noqa: BLE001 -- the exception type is what is pinned
            out[f"status_{name}"] = np.array(type(e).__name__)
            continue
        out[f"status_{name}"] = np.array("accepted")
        out[f"module_{name}"] = np.array(describe(mod))
        if any(p in describe(mod) for p in ("PReLU", "RReLU")):
            continue
        inp = xg if name.endswith("glu") else x
        xi = inp.clone().requires_grad_(True)
        y = mod(xi)
        (y * dy).sum().backward()
        out[f"fwd32_{name}"] = y.detach().numpy()
        out[f"grad32_{name}"] = xi.grad.numpy()
        out[f"fwd16_{name}"] = mod.to(torch.bfloat16)(inp.bfloat16()).float().numpy()
        print(f"{name:28s} {describe(mod)}")
    np.savez_compressed(os.path.join(GOLDEN, "activations.npz"), **out)

    import oracle.dolomite_oracle as O
    import act_oracle

    act_oracle.install()
    R = import_reference()
    for name, kw in MODEL_CONFIGS.items():
        cfg = O.OracleConfig(**kw)
        params = O.init_params(cfg, seed=42)
        if cfg.add_bias:
            g = torch.Generator().manual_seed(7)
            for k in params:
                if k.endswith(".bias"):
                    params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        rng = np.random.default_rng(1234)
        tokens = rng.integers(0, cfg.vocab_size, size=(2, 65), dtype=np.int64)
        eos = 7
        tokens[0, 20] = tokens[1, 5] = tokens[1, 40] = eos
        fixtures = {"tokens": tokens, "eos": np.int64(eos)}
        for mode, (ram, rpi) in {"uniform": (False, False), "ragged": (True, True)}.items():
            inp, labels = O.split_tokens(tokens)
            b = O.prepare_model_inputs(inp.copy(), eos, ram, rpi)
            logits, blocks, wte, wpe, ln_f_grads = reference_forward(R, cfg, params, b["input_ids"], b["position_ids"],
                                                                     b["cu_seqlens"])
            lab = torch.as_tensor(np.ascontiguousarray(labels).reshape(-1))
            loss = torch.nn.functional.cross_entropy(logits, lab)
            loss.backward()
            g_ref = {f"transformer.h.{i}.{k}": v.grad for i, blk in enumerate(blocks) for k, v in blk.named_parameters()}
            g_ref["transformer.wte.weight"] = wte.grad
            g_ref.update(ln_f_grads())
            if wpe is not None:
                g_ref["transformer.wpe.weight"] = wpe.grad
            fixtures[f"{mode}_loss"] = loss.detach().numpy()
            fixtures[f"{mode}_logits_rows"] = logits.detach()[::8].numpy()
            for k, v in g_ref.items():
                fixtures[f"{mode}_grad:{k}"] = v.flatten()[::GRAD_STRIDE].numpy()
            # the oracle reproduces the reference before anything is written
            p_req = {k: v.clone().requires_grad_(True) for k, v in params.items()}
            loss_o, logits_o = O.pretraining_loss(p_req, cfg, tokens, eos, ram, rpi)
            loss_o.backward()
            assert (logits_o.detach() - logits.detach()).abs().max() <= 2e-5, name
            for k, v in g_ref.items():
                assert (p_req[k].grad - v).abs().max() <= 5e-6 + 1e-4 * v.abs().max(), (name, k)
        np.savez_compressed(os.path.join(GOLDEN, f"model_act_{name}.npz"), **fixtures)
        print(f"model {name}: pinned")


if __name__ == "__main__":
    main()
