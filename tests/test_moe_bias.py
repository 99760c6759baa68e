"""CPU: MoE experts with biases (ParameterizedExperts with add_bias, moe_dolomite/moe/base.py:12-50).

The oracle reproduces the reference-derived fixtures of tools/pin_moe_bias.py (one eager SparseMoE layer; a two-layer
MoEDolomite with attention and expert biases), check_supported follows the reference's rules for expert biases, and the
engine lays the biases out under the reference's names and shapes, zero-initialised."""

import os

import numpy as np
import pytest
import torch

import oracle.dolomite_oracle as O
from dolomite_engine_b200.engine import DolomiteEngine, check_supported
from dolomite_engine_b200.hf_models import MoEDolomiteConfig

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
EOS = 7
GRAD_STRIDE, FULL_GRAD, LOGIT_ROW_STRIDE = 16, 4096, 8  # tools/pin_vocab.py's subsampling
MODEL_KW = dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_head=8, n_inner=192, attention_head_type="mha",
                add_bias=True, num_experts=8, num_experts_per_tok=2, normalization_function="rmsnorm",
                position_embedding_type="rope")


def bf16_from_bits(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(a.astype(np.uint16).view(np.int16)).view(torch.bfloat16).float()


def subsample(g: torch.Tensor) -> torch.Tensor:
    g = g.flatten()
    return g if g.numel() <= FULL_GRAD else g[::GRAD_STRIDE]


def layer_case(fx, name):
    """-> (oracle config, x, dy, params under prefix "m.") of one layer case of moe_bias_layer.npz"""
    T, H, F, E, k = (int(v) for v in fx[f"{name}/shape"])
    cfg = O.OracleConfig(vocab_size=256, n_embd=H, n_layer=1, n_head=4, n_inner=F, num_experts=E, num_experts_per_tok=k,
                         add_bias=True, activation_function=str(fx[f"{name}/activation"]))
    params = {f"m.{n}": bf16_from_bits(fx[f"{name}/{n}"])
              for n in ("gate.weight", "c_fc.weight", "c_fc.bias", "c_proj.weight", "c_proj.bias")}
    return cfg, bf16_from_bits(fx[f"{name}/x"]), torch.from_numpy(fx[f"{name}/dy"]), params


def model_batches(fx):
    """the packed ragged batch and the padded batch of a model fixture: name -> (ids, positions, cu_seqlens, labels)"""
    inp, labels = O.split_tokens(fx["packed_tokens"])
    b = O.prepare_model_inputs(inp.copy(), EOS, True, True)
    out = {"packed": (b["input_ids"], b["position_ids"], b["cu_seqlens"], np.ascontiguousarray(labels).reshape(-1))}
    m = fx["padded_mask"].astype(bool)
    ids = fx["padded_tokens"][m]
    lens = m.sum(1)
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    pos = np.concatenate([np.arange(n) for n in lens])
    lab = np.full(ids.shape, -100, dtype=np.int64)
    for d in range(len(lens)):
        lab[cu[d] : cu[d + 1] - 1] = ids[cu[d] + 1 : cu[d + 1]]
    out["padded"] = (ids, pos, cu, lab)
    return out


def model_params(fx, act):
    cfg = O.OracleConfig(activation_function=act, **MODEL_KW)
    params = O.init_params(cfg, seed=int(fx["seed"]))
    for k in params:
        if k.endswith(".bias"):
            params[k] = torch.from_numpy(fx[f"bias:{k}"])
    return cfg, params


@pytest.mark.parametrize("name", ["e8_k2", "e16_k4"])
def test_oracle_reproduces_the_layer_fixture(name):
    fx = np.load(os.path.join(GOLDEN, "moe_bias_layer.npz"))
    cfg, x, dy, params = layer_case(fx, name)
    assert all(params[f"m.{b}"].abs().max() > 0.1 for b in ("c_fc.bias", "c_proj.bias"))  # biases that matter
    p = {n: v.clone().requires_grad_(True) for n, v in params.items()}
    x = x.requires_grad_(True)
    y, logits = O.sparse_moe(x, p, "m.", cfg)
    y.backward(dy)
    ref_y = torch.from_numpy(fx[f"{name}/y"])
    assert (y - ref_y).abs().max() <= 1e-5 * ref_y.abs().max()
    assert (logits - torch.from_numpy(fx[f"{name}/router_logits"])).abs().max() <= 1e-5
    ref = torch.from_numpy(fx[f"{name}/grad:x"])
    assert (x.grad - ref).abs().max() <= 1e-5 * ref.abs().max()
    for n, v in p.items():
        got = subsample(v.grad) if v.dim() == 3 else v.grad
        ref = torch.from_numpy(fx[f"{name}/grad:{n[2:]}"])
        assert (got - ref).abs().max() <= 1e-5 * ref.abs().max(), n


@pytest.mark.parametrize("act", ["swiglu", "gelu_pytorch_tanh"])
def test_oracle_reproduces_the_model_fixture(act):
    fx = np.load(os.path.join(GOLDEN, f"moe_bias_model_{act}.npz"))
    cfg, params = model_params(fx, act)
    for batch, (ids, pos, cu, labels) in model_batches(fx).items():
        p = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        logits = O.forward_logits(p, cfg, ids, pos, cu)
        loss = torch.nn.functional.cross_entropy(logits, torch.as_tensor(labels), ignore_index=-100)
        loss.backward()
        assert abs(loss.item() - float(fx[f"{batch}_loss"])) <= 1e-5, batch
        assert (logits[::LOGIT_ROW_STRIDE].detach() - torch.from_numpy(fx[f"{batch}_logits"])).abs().max() <= 2e-5, batch
        names = {k.split(":", 1)[1] for k in fx.files if k.startswith(f"{batch}_grad:")}
        assert names == set(p), sorted(names ^ set(p))
        for k, v in p.items():
            ref = torch.from_numpy(fx[f"{batch}_grad:{k}"])
            assert (subsample(v.grad) - ref).abs().max() <= 1e-4 * (ref.abs().max() + 1e-30), (batch, k)


def _moe_cfg(**kw):
    base = dict(vocab_size=512, n_positions=64, n_embd=128, n_layer=2, n_head=8, n_inner=192, attention_head_type="mha",
                num_experts=8, num_experts_per_tok=2, position_embedding_type="rope", normalization_function="rmsnorm",
                activation_function="swiglu", resid_pdrop=0, embd_pdrop=0, attn_pdrop=0)
    return MoEDolomiteConfig(**{**base, **kw})


def test_check_supported_follows_the_reference_on_expert_biases():
    biased = _moe_cfg()  # add_bias left at MoEDolomiteConfig's default
    assert biased.add_bias is True
    check_supported(biased)  # the default implementation: eager experts, which carry the bias
    check_supported(biased, moe_implementation="eager")
    with pytest.raises(AssertionError, match="scattermoe doesn't support bias"):  # moe/scatter.py:22
        check_supported(biased, moe_implementation="scattermoe")
    check_supported(_moe_cfg(add_bias=False), moe_implementation="scattermoe")
    for impl in ("eager", "scattermoe"):  # MoE blocks stay RMSNorm-only, with or without biases
        with pytest.raises(NotImplementedError, match="MoE blocks are implemented with rmsnorm"):
            check_supported(_moe_cfg(normalization_function="layernorm"), moe_implementation=impl)


def test_model_defaults_to_eager_experts():
    """moe_dolomite/base.py:21: `moe_implementation` defaults to eager; scattermoe with biases is refused before any
    device is touched"""
    from dolomite_engine_b200.hf_models import MoEDolomiteForCausalLM

    with pytest.raises(AssertionError, match="scattermoe doesn't support bias"):
        MoEDolomiteForCausalLM(_moe_cfg(), moe_implementation="scattermoe", device=torch.device("cpu"))
    model = MoEDolomiteForCausalLM(_moe_cfg(), device=torch.device("cpu"), seed=1)
    assert model.moe_implementation == "eager"


@pytest.mark.parametrize("act", ["swiglu", "gelu_pytorch_tanh"])
def test_engine_parameters_match_the_reference_names_and_shapes(act):
    fx = np.load(os.path.join(GOLDEN, f"moe_bias_model_{act}.npz"))
    kw = {k: v for k, v in MODEL_KW.items()}
    eng = DolomiteEngine(MoEDolomiteConfig(activation_function=act, resid_pdrop=0, embd_pdrop=0, attn_pdrop=0, **kw), "cpu",
                         seed=1)
    shapes = {name: tuple(unit.views[name].shape) for name, unit, _ in eng.named_views()}
    ref_names = {k.split(":", 1)[1] for k in fx.files if k.startswith("packed_grad:")}  # the reference's named_parameters
    assert set(shapes) == ref_names, sorted(set(shapes) ^ ref_names)
    _, params = model_params(fx, act)
    assert shapes == {k: tuple(v.shape) for k, v in params.items()}
    for k in ("transformer.h.0.mlp.c_fc.bias", "transformer.h.1.mlp.c_proj.bias"):
        assert shapes[k] == tuple(fx[f"bias:{k}"].shape)
    for name, unit, _ in eng.named_views():
        if name.endswith(".bias"):
            assert bool((unit.views[name] == 0).all()), name  # ParameterizedExperts.reset_parameters: bias.zero_()
