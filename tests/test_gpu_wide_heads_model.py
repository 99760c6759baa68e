"""GPU: models with wide attention heads (head_dim 160, 192, 256) end to end -- engine, RoPE / learned positions / ALiBi,
the padding-free and padded paths, block checkpointing, the KV cache and generation -- against the reference fixtures of
tools/pin_wide_heads.py, with the bars of the existing model-fixture tests (test_gpu_vocab.py, test_gpu_alibi.py): loss
within 1e-3 relative, every sampled gradient within rel-L2 3e-2, and the logits as _check_logits states."""

import os

import numpy as np
import pytest
import torch

import oracle.dolomite_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
EOS = 7
# tools/pin_wide_heads.py MODELS
MODELS = {
    "mqa_hd256": dict(vocab_size=256, n_positions=256, n_embd=512, n_layer=2, n_head=2, n_inner=512,
                      attention_head_type="mqa", position_embedding_type="rope", normalization_function="rmsnorm",
                      activation_function="swiglu", add_bias=True),
    "gqa_hd192": dict(vocab_size=256, n_positions=256, n_embd=768, n_layer=2, n_head=4, num_key_value_heads=2,
                      n_inner=512, attention_head_type="gqa", position_embedding_type="rope",
                      normalization_function="rmsnorm", activation_function="swiglu", add_bias=False),
    "mha_hd160_bigcode": dict(vocab_size=256, n_positions=256, n_embd=320, n_layer=2, n_head=2, n_inner=640,
                              attention_head_type="mha", position_embedding_type="learned_absolute",
                              normalization_function="layernorm", activation_function="gelu_pytorch_tanh", add_bias=True),
}
ALIBI_KW = dict(vocab_size=512, n_positions=256, n_embd=512, n_layer=2, n_head=2, n_inner=512, attention_head_type="mqa",
                position_embedding_type="alibi", activation_function="swiglu", add_bias=False)
_NO_DROPOUT = dict(resid_pdrop=0.0, embd_pdrop=0.0, attn_pdrop=0.0)


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def subsample(g):
    """the gradient samples tools/pin_wide_heads.py keeps: small tensors whole, else every 61st element"""
    g = g.flatten()
    return g if g.numel() <= 4096 else g[::61]


def _model(kw, padding_free=True, impl="sdpa", params=None, **cfg_extra):
    from dolomite_engine_b200.hf_models import GPTDolomiteConfig, GPTDolomiteForCausalLM

    cfg = GPTDolomiteConfig(**{**_NO_DROPOUT, "eos_token_id": EOS, **kw, **cfg_extra})
    model = GPTDolomiteForCausalLM(cfg, seed=None if params is not None else 42, use_padding_free_transformer=padding_free,
                                   **({} if padding_free else {"attn_implementation": impl}))
    if params is not None:
        model.load_state_dict(params)
    return model


def _fixture_params(kw, fx):
    params = O.init_params(O.OracleConfig(**kw), seed=42)
    for k in params:
        if f"bias:{k}" in fx:
            params[k] = torch.from_numpy(fx[f"bias:{k}"])
    return params


def _check_logits(got, want):
    """the bf16 engine against the fp32 reference, with the bar of test_gpu_alibi.py's MoE model: rel-L2 1e-2 and every
    logit within 4 bf16 ulps of the largest one plus 5e-3.  At these widths (512, 768) the logits reach 2-4 in magnitude,
    where one bf16 rounding of a logit alone is up to 2^-8 relative; the 5e-3 rtol / atol bar of the width-128 fixture
    models holds for 90-99 % of them here (measured on an H100), which the test prints."""
    assert got.shape == want.shape
    close = torch.isclose(got, want, rtol=5e-3, atol=5e-3).float().mean().item()
    err, rel = (got - want).abs().max().item(), rel_l2(got, want)
    print(f"\nlogits: rel-L2 {rel:.3g}, max err {err:.3g} (|logit| max {want.abs().max().item():.3g}), "
          f"within 5e-3: {close:.4f}")
    assert rel < 1e-2 and err < 4 * 2.0**-8 * want.abs().max().item() + 5e-3, (rel, err)


def _check_grads(model, fx, prefix):
    bad = []
    for pname, unit, _ in model.engine.named_views():
        g = subsample(unit.gviews[pname])
        assert torch.isfinite(g).all(), pname
        e = rel_l2(g, torch.from_numpy(fx[f"{prefix}grad:{pname}"]))
        if e > 3e-2:
            bad.append((pname, round(e, 4)))
    assert not bad, bad


@pytest.mark.parametrize("name", list(MODELS))
def test_wide_head_packed_batch_matches_reference(name):
    fx = np.load(os.path.join(GOLDEN, f"model_wide_{name}.npz"))
    model = _model(MODELS[name], params=_fixture_params(MODELS[name], fx))
    model.assume_unit_loss_grad = True
    inp, labels = O.split_tokens(fx["packed_tokens"])
    b = O.prepare_model_inputs(inp.copy(), EOS, True, True)
    ids, pos, cu = b["input_ids"], b["position_ids"], b["cu_seqlens"]
    labels = np.ascontiguousarray(labels).reshape(-1)
    args = (torch.from_numpy(ids).cuda(), torch.from_numpy(pos).cuda(), torch.from_numpy(cu).cuda(), int(np.diff(cu).max()))
    model.engine.zero_grad()
    loss = model.forward_pretraining_loss(*args, torch.from_numpy(labels).cuda())
    loss.backward()
    want = float(fx["packed_loss"])
    assert abs(loss.item() - want) / want < 1e-3, (loss.item(), want)
    _check_grads(model, fx, "packed_")
    with torch.no_grad():
        logits = model(input_ids=args[0], position_ids=args[1], cu_seqlens=args[2], max_seqlen=args[3]).logits
    _check_logits(logits.float().cpu()[::8], torch.from_numpy(fx["packed_logits"]))


@pytest.mark.parametrize("name", list(MODELS))
def test_wide_head_padded_batch_matches_reference(name):
    fx = np.load(os.path.join(GOLDEN, f"model_wide_{name}.npz"))
    model = _model(MODELS[name], padding_free=False, params=_fixture_params(MODELS[name], fx))
    tokens = torch.from_numpy(fx["padded_tokens"]).cuda()
    mask = torch.from_numpy(fx["padded_mask"]).cuda()
    model.engine.zero_grad()
    out = model(input_ids=tokens, attention_mask=mask, labels=tokens)
    out.loss.backward()
    want = float(fx["padded_loss"])
    assert abs(out.loss.item() - want) / want < 1e-3, (out.loss.item(), want)
    _check_grads(model, fx, "padded_")
    with torch.no_grad():
        logits = model(input_ids=tokens, attention_mask=mask).logits
    _check_logits(logits[mask.bool()].float().cpu()[::8], torch.from_numpy(fx["padded_logits"]))


def test_wide_head_alibi_sdpa_masked_batch_matches_reference():
    fx = np.load(os.path.join(GOLDEN, "model_wide_mqa_hd256_alibi_sdpa.npz"))
    model = _model({**ALIBI_KW, "normalization_function": "rmsnorm"}, padding_free=False, impl="sdpa",
                   params=O.init_params(O.OracleConfig(**ALIBI_KW), seed=42))
    tokens, mask = torch.from_numpy(fx["tokens"]), torch.from_numpy(fx["mask"])
    model.engine.zero_grad()
    loss = model(input_ids=tokens, attention_mask=mask, labels=tokens).loss
    loss.backward()
    ref_loss = float(fx["loss"])
    assert abs(loss.item() - ref_loss) <= 1e-3 * abs(ref_loss), (loss.item(), ref_loss)
    _check_grads(model, fx, "")
    with torch.no_grad():
        logits = model(input_ids=tokens, attention_mask=mask).logits
    _check_logits(logits[mask.bool().cuda()].float().cpu(), torch.from_numpy(fx["logits"]))


def _grads(model):
    return {pname: unit.gviews[pname].detach().float().cpu().clone() for pname, unit, _ in model.engine.named_views()}


def _step(model, tokens, mask):
    model.engine.zero_grad()
    loss = model(input_ids=tokens, attention_mask=mask, labels=tokens).loss
    loss.backward()
    return loss.detach().clone(), _grads(model)


def test_wide_head_dropout_steps_are_run_to_run_identical_and_checkpointing_keeps_gradients():
    """hd 256 with attention dropout: two steps from the same dropout seed give the same bits, and block checkpointing
    (every block re-run in backward) gives the same bits again"""
    model = _model(MODELS["mqa_hd256"], padding_free=False, impl="sdpa", attn_pdrop=0.1)
    tokens = torch.from_numpy(np.random.default_rng(6).integers(0, 256, size=(3, 200)))
    mask = torch.ones_like(tokens)
    mask[1, :37] = 0
    model.engine.dropout_seed = 11
    l1, g1 = _step(model, tokens, mask)
    model.engine.dropout_seed, model.engine._dropout_passes = 11, 0
    l2, g2 = _step(model, tokens, mask)
    model.engine.checkpoint_every = 1
    model.engine.dropout_seed, model.engine._dropout_passes = 11, 0
    l3, g3 = _step(model, tokens, mask)
    assert torch.isfinite(l1) and torch.equal(l1, l2) and torch.equal(l1, l3)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k
        assert torch.equal(g1[k], g3[k]), k


@pytest.mark.parametrize("case", ["mqa_hd256_rope", "gqa_hd192_alibi"])
def test_wide_head_cached_greedy_generation_equals_stepwise_argmax(case):
    if case == "mqa_hd256_rope":
        model = _model(MODELS["mqa_hd256"], padding_free=False, impl="sdpa")
    else:
        kw = {**MODELS["gqa_hd192"], "position_embedding_type": "alibi"}
        model = _model(kw, padding_free=False, impl="eager")
    model.eval()
    prompt = torch.from_numpy(np.random.default_rng(8).integers(0, 256, size=(2, 12)))
    mask = torch.ones_like(prompt)
    mask[0, :5] = 0
    cached = model.generate(input_ids=prompt, attention_mask=mask, max_new_tokens=24, eos_token_id=-1)
    stepwise = model.generate(input_ids=prompt, attention_mask=mask, max_new_tokens=24, eos_token_id=-1, use_cache=False)
    assert torch.equal(cached, stepwise)
