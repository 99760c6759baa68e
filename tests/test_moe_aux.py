"""CPU: the MoE load-balancing loss oracle (tests/moe_aux_oracle.py) against tests/golden/moe_aux.npz, which
tools/pin_moe_aux.py wrote from transformers' Mixtral load_balancing_loss_func and the reference's get_moe_loss, and the
model-API rules that need no GPU."""

import os

import numpy as np
import pytest
import torch

from moe_aux_oracle import load_balancing_loss, moe_loss

# transformers forms the expert fractions in fp32 (one_hot(...).float()): agreement to fp32 rounding
CASES = ["e8_k2_right", "e8_k2_left", "e16_k4_none", "e40_k1_right", "e64_k8_left"]


@pytest.fixture(scope="module")
def fx(golden_dir):
    return np.load(os.path.join(golden_dir, "moe_aux.npz"))


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_transformers_and_the_reference_glue(fx, name):
    L, B, S, E, k = fx[f"{name}/shape"].tolist()
    logits = torch.from_numpy(fx[f"{name}/logits"]).double()
    mask = torch.from_numpy(fx[f"{name}/mask"])
    layers = tuple(logits[l] for l in range(L))
    aux = load_balancing_loss(layers, E, k)
    assert aux.item() == pytest.approx(float(fx[f"{name}/aux"]), rel=1e-6)
    masked = load_balancing_loss(layers, E, k, attention_mask=mask)
    assert masked.item() == pytest.approx(float(fx[f"{name}/aux_masked"]), rel=1e-6)
    # the engine's rule: the experts of the routing plan (top-k of the raw logits), statistics over the real tokens only
    keep = mask.reshape(-1).bool()
    plan = tuple(lg.topk(k, -1).indices[keep] for lg in layers)
    real = load_balancing_loss(tuple(lg[keep] for lg in layers), E, k, selected=plan)
    assert real.item() == pytest.approx(float(fx[f"{name}/aux_masked"]), rel=1e-6)
    if not (~keep).any():  # no padding: the reference's unmasked value
        assert real.item() == pytest.approx(float(fx[f"{name}/aux"]), rel=1e-6)
    coef = float(fx["coef"])
    loss, a = moe_loss(torch.tensor(float(fx[f"{name}/ce"]), dtype=torch.float64), aux, coef)
    assert loss.item() == pytest.approx(float(fx[f"{name}/glue_loss"]), rel=1e-6)
    assert a.item() == pytest.approx(float(fx[f"{name}/glue_aux"]), rel=1e-6)
    none_loss, none_aux = moe_loss(None, aux, coef)
    assert none_loss is None and none_aux.item() == pytest.approx(float(fx[f"{name}/glue_aux_no_labels"]), rel=1e-6)


def test_oracle_gradient_is_the_closed_form(fx):
    """d aux / d logits[t, e] = E / N^2 * p[t,e] * (C_e - sum_j p[t,j] C_j): what moe_router_bwd_aux computes"""
    L, B, S, E, k = fx["e8_k2_right/shape"].tolist()
    logits = torch.from_numpy(fx["e8_k2_right/logits"]).double().requires_grad_(True)
    aux = load_balancing_loss(tuple(logits[l] for l in range(L)), E, k)
    aux.backward()
    p = torch.softmax(logits.detach(), -1)
    C = torch.nn.functional.one_hot(p.topk(k, -1).indices, E).sum((0, 1, 2)).double()
    N = L * B * S
    closed = E / N**2 * p * (C - (p * C).sum(-1, keepdim=True))
    assert torch.allclose(logits.grad, closed, rtol=1e-12, atol=1e-15)


def _moe_model(**cfg_kw):
    from dolomite_engine_b200.hf_models import MoEDolomiteConfig, MoEDolomiteForCausalLM

    cfg = MoEDolomiteConfig(vocab_size=256, n_embd=64, n_layer=1, n_head=4, n_inner=128, num_experts=8, num_experts_per_tok=2,
                            attention_head_type="mha", add_bias=False, position_embedding_type="rope",
                            normalization_function="rmsnorm", activation_function="swiglu", resid_pdrop=0, embd_pdrop=0,
                            attn_pdrop=0, **cfg_kw)
    return MoEDolomiteForCausalLM(cfg, device="cpu")


def test_padding_free_with_the_flag_raises_the_reference_error():
    model = _moe_model()
    with pytest.raises(NotImplementedError, match="padding_free is not supported with load_balancing_loss_func"):
        model(input_ids=[[1, 2, 3]], labels=[[1, 2, 3]], output_router_logits=True)


def test_config_flag_alone_does_not_ask_for_the_term():
    """config.output_router_logits = True with the forward argument left at None: the reference passes the unresolved
    argument to get_moe_loss, which adds no term, so the padding-free path does not raise and runs as without the flag"""
    from dolomite_engine_b200 import _lib

    model = _moe_model(output_router_logits=True)
    calls = []
    orig = model.engine.forward

    def spy(*a, **kw):
        calls.append(kw)
        return orig(*a, **kw)

    model.engine.forward = spy
    with pytest.raises((_lib.DolomiteB200Error, AssertionError, RuntimeError)):  # no CUDA device here: the first kernel refuses
        model(input_ids=[[1, 2, 3]], labels=[[1, 2, 3]])
    assert len(calls) == 1 and not calls[0].get("router_aux", False)


def test_router_logits_need_an_moe_model():
    from dolomite_engine_b200.hf_models import GPTDolomiteConfig, GPTDolomiteForCausalLM

    cfg = GPTDolomiteConfig(vocab_size=256, n_embd=64, n_layer=1, n_head=4, n_inner=128, attention_head_type="mha",
                            position_embedding_type="rope")
    model = GPTDolomiteForCausalLM(cfg, device="cpu", use_padding_free_transformer=False)
    with pytest.raises(ValueError, match="MoE"):
        model(input_ids=torch.ones(1, 4, dtype=torch.long), output_router_logits=True)
