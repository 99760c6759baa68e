"""GPU: ALiBi in the attention kernels (forward, dK/dV, dQ, decode) against the fp32 oracle with the bf16 bias, and alibi
models against the reference fixtures (tools/pin_alibi.py) and the exact equalities the padded path must keep."""

import math
import os

import numpy as np
import pytest
import torch

import alibi_oracle as A
import oracle.dolomite_oracle as O
from dolomite_engine_b200.alibi import alibi_slopes

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def K():
    from dolomite_engine_b200 import kernels

    return kernels


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _inputs(lens, ng, g, hd, seed=7):
    gen = torch.Generator().manual_seed(seed)
    T = sum(lens)
    qkv = torch.randn(T, ng * (g + 2) * hd, generator=gen).bfloat16()
    dout = torch.randn(T, ng * g * hd, generator=gen).bfloat16()
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return qkv, dout, cu


def _cfg(ng, g, hd):
    return O.OracleConfig(n_embd=ng * g * hd, n_head=ng * g, num_key_value_heads=ng,
                          attention_head_type="mha" if g == 1 else ("mqa" if ng == 1 else "gqa"))


# head dims x MHA / GQA / MQA, non-power-of-two head counts (3, 5, 6, 12), ragged documents with length 1 and
# non-multiples of 128
CASES = [([128], 2, 1, 16), ([100, 37, 300, 1, 129], 3, 1, 32), ([200, 130, 515], 5, 1, 64), ([300, 77, 260], 2, 3, 80),
         ([150, 250, 1], 1, 6, 96), ([333, 64], 2, 2, 128), ([1], 1, 1, 64),
         # a document of 8192 next to short ones; 16 heads put the first slope at 2^-0.5, so the biased logits reach ~5800
         # (~8400 in log2 units), where fp32 keeps 2^-10 of them: the worst case of the backward's recomputed P
         ([8192, 37, 300], 4, 4, 64)]


@pytest.mark.parametrize("lens,ng,g,hd", CASES)
@pytest.mark.parametrize("dropout", [0.0, 0.1])
def test_alibi_attention_fwd_bwd_vs_oracle(lens, ng, g, hd, dropout):
    qkv, dout, cu = _inputs(lens, ng, g, hd)
    scale = 1.0 / math.sqrt(hd)
    cfg = _cfg(ng, g, hd)
    slopes = alibi_slopes(ng * g)
    keys = (12345, 678)
    # the [heads, L, L] scores of the 8192-token document are computed on the GPU (fp32, no TF32)
    dev = "cuda" if max(lens) > 4096 else "cpu"
    x = qkv.float().to(dev).requires_grad_(True)
    q, k, v = O.split_qkv_activations(x, cfg)
    if dropout:
        O.DROPOUT = _FixedKeys(keys)
    try:
        ref = A.packed_causal_attention(q, k, v, cu, scale, slopes, bias_bf16=True, dropout_site=0, dropout_p=dropout)
    finally:
        O.DROPOUT = None
    ref.backward(dout.float().to(dev))
    cu_d, sl = torch.from_numpy(cu).cuda(), slopes.cuda()
    out, lse = K().attn_varlen_fwd(qkv.cuda(), cu_d, max(lens), ng, g, hd, scale, dropout_p=dropout, dropout_keys=keys,
                                   alibi_slopes=sl)
    assert rel_l2(out, ref) < 6e-3
    dqkv = K().attn_varlen_bwd(dout.cuda(), qkv.cuda(), out, lse, cu_d, max(lens), ng, g, hd, scale, dropout_p=dropout,
                               dropout_keys=keys, alibi_slopes=sl)
    assert rel_l2(dqkv, x.grad) < 1.2e-2
    # the plain kernels on the same input differ: the bias is applied
    out0, _ = K().attn_varlen_fwd(qkv.cuda(), cu_d, max(lens), ng, g, hd, scale, dropout_p=dropout, dropout_keys=keys)
    if max(lens) > 1:
        assert not torch.equal(out0, out)


class _FixedKeys(O.DropoutOracle):
    """the oracle's attention dropout with explicit kernel keys (the kernels get `keys` directly)"""

    def __init__(self, keys):
        self._k = keys

    def keys(self, site):
        return self._k


def test_alibi_long_document_and_lse():
    """one document of 8192 tokens next to short ones; LSE against the oracle's biased logits"""
    lens, ng, g, hd = [8192, 5, 131], 2, 2, 64
    qkv, dout, cu = _inputs(lens, ng, g, hd, seed=3)
    scale = hd**-0.5
    slopes = alibi_slopes(ng * g)
    out, lse = K().attn_varlen_fwd(qkv.cuda(), torch.from_numpy(cu).cuda(), max(lens), ng, g, hd, scale,
                                   alibi_slopes=slopes.cuda())
    q, k, v = O.split_qkv_activations(qkv.float(), _cfg(ng, g, hd))
    ref = A.packed_causal_attention(q, k, v, cu, scale, slopes, bias_bf16=True)
    assert rel_l2(out, ref) < 6e-3
    # LSE rows of the long document, every 97th query
    rows = torch.arange(0, 8192, 97)
    kk = k.repeat_interleave(g, dim=1)
    bias = A.alibi_bias(slopes, torch.arange(8192).unsqueeze(0), True)[0]
    for h in range(ng * g):
        sc = (q[rows, h] @ kk[:8192, h].T) * scale + bias[h]
        sc = sc.masked_fill(torch.arange(8192)[None, :] > rows[:, None], float("-inf"))
        torch.testing.assert_close(lse[h, rows].cpu(), torch.logsumexp(sc, -1), atol=2e-3, rtol=1e-4)


def test_zero_query_probe_pins_the_bf16_rounding_point():
    """q = 0: every logit is the bias alone, so the last row's LSE is logsumexp of the bias row.  With one head the slope
    is 2^-8, so slope * k is not a bf16 value for most k < 8192 and an fp32 bias would miss the bar by far."""
    L, hd = 8192, 64
    qkv = torch.randn(L, 3 * hd, generator=torch.Generator().manual_seed(1)).bfloat16()
    qkv[:, :hd] = 0
    slopes = alibi_slopes(1)
    cu = torch.tensor([0, L], dtype=torch.int32).cuda()
    _, lse = K().attn_varlen_fwd(qkv.cuda(), cu, L, 1, 1, hd, hd**-0.5, alibi_slopes=slopes.cuda())
    kpos = torch.arange(L).unsqueeze(0)
    b16 = A.alibi_bias(slopes, kpos, True)[0, 0].double()
    b32 = A.alibi_bias(slopes, kpos, False)[0, 0].double()
    want, fp32_lse = torch.logsumexp(b16, 0).item(), torch.logsumexp(b32, 0).item()
    assert abs(fp32_lse - want) / abs(want) > 1e-5  # 3.8e-5: the probe tells the two rounding points apart
    assert abs(lse[0, L - 1].item() - want) / abs(want) <= 1e-6


@pytest.mark.parametrize("hd,ng,g", [(16, 1, 1), (64, 3, 1), (80, 2, 4), (128, 1, 5)])
def test_alibi_decode_vs_fp32_softmax(hd, ng, g):
    B, L_max = 3, 700
    lens = torch.tensor([1, 257, 700], dtype=torch.int32)
    gen = torch.Generator().manual_seed(5)
    kc = torch.randn(B, L_max, ng * hd, generator=gen).bfloat16()
    vc = torch.randn(B, L_max, ng * hd, generator=gen).bfloat16()
    qkv = torch.randn(B, ng * (g + 2) * hd, generator=gen).bfloat16()
    slopes = alibi_slopes(ng * g)
    scale = hd**-0.5
    out = K().attn_decode(qkv.cuda(), kc.cuda(), vc.cuda(), lens.cuda(), ng, g, hd, scale, alibi_slopes=slopes.cuda())
    q = qkv.float().view(B, ng, g + 2, hd)[:, :, :g].reshape(B, ng * g, hd)
    for b in range(B):
        n = int(lens[b])
        kk = kc[b, :n].float().view(n, ng, hd).repeat_interleave(g, dim=1)
        vv = vc[b, :n].float().view(n, ng, hd).repeat_interleave(g, dim=1)
        bias = A.alibi_bias(slopes, torch.arange(n).unsqueeze(0), True)[0]  # [nh, n]
        p = torch.softmax(torch.einsum("hd,khd->hk", q[b], kk) * scale + bias, -1)
        ref = torch.einsum("hk,khd->hd", p, vv).reshape(-1)
        assert rel_l2(out[b], ref) < 6e-3, b


def test_null_slopes_are_an_error():
    from dolomite_engine_b200 import _lib

    qkv, _, cu = _inputs([16], 1, 1, 64)
    qkv, lse = qkv.cuda(), torch.empty(1, 16, device="cuda")
    out = torch.empty(16, 64, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(_lib.DolomiteB200Error, match="alibi_slopes is null"):
        _lib.call("dolomite_b200_attn_varlen_fwd_alibi", qkv.data_ptr(), qkv.stride(0), out.data_ptr(), lse.data_ptr(),
                  torch.from_numpy(cu).cuda().data_ptr(), 1, 16, 16, 1, 1, 64, 0.125, 0.0, 0, 0, None, None)


# ------------------------------------------------------------------------------------------------
# models
# ------------------------------------------------------------------------------------------------
_BASE = dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_inner=256, activation_function="swiglu",
             position_embedding_type="alibi", add_bias=False)
# the engine-side configs: the oracle's defaults (rmsnorm, no dropout) spelled out
_ENGINE = dict(normalization_function="rmsnorm", resid_pdrop=0.0, embd_pdrop=0.0, attn_pdrop=0.0)
FIXTURES = {
    "mha_eager_nomask": (dict(n_head=8, attention_head_type="mha"), "eager"),
    "gqa_eager_left": (dict(n_head=8, num_key_value_heads=2, attention_head_type="gqa"), "eager"),
    "mqa_sdpa_mask": (dict(n_head=8, attention_head_type="mqa"), "sdpa"),
    "mha_sdpa_nomask": (dict(n_head=8, attention_head_type="mha"), "sdpa"),
}


def _model(kw, impl, params=None, cls="gpt_dolomite", **extra):
    from dolomite_engine_b200.hf_models.config import GPTDolomiteConfig, MoEDolomiteConfig
    from dolomite_engine_b200.hf_models.modeling import GPTDolomiteForCausalLM, MoEDolomiteForCausalLM

    Cfg, M = (GPTDolomiteConfig, GPTDolomiteForCausalLM) if cls == "gpt_dolomite" else (MoEDolomiteConfig, MoEDolomiteForCausalLM)
    model = M(Cfg(**{**_ENGINE, **kw}), attn_implementation=impl, use_padding_free_transformer=False, seed=None if params else 42, **extra)
    if params is not None:
        model.load_state_dict(params)
    return model


def _grads(model):
    return {s.name: u.gviews[s.name].detach().float().cpu().clone() for name, u, s in model.engine.named_views()}


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_alibi_models_vs_reference_fixtures(name):
    kw, impl = FIXTURES[name]
    fx = np.load(os.path.join(GOLDEN, f"alibi_model_{name}.npz"))
    kw = {**_BASE, **kw}
    params = O.init_params(O.OracleConfig(**kw), seed=42)
    model = _model(kw, impl, params)
    tokens = torch.from_numpy(fx["tokens"])
    mask = torch.from_numpy(fx["mask"]) if "mask" in fx else None
    model.engine.zero_grad()
    loss = model(input_ids=tokens, attention_mask=mask, labels=tokens).loss
    loss.backward()
    ref_loss = float(fx["loss"])
    assert abs(loss.item() - ref_loss) <= 1e-3 * abs(ref_loss)
    grads = _grads(model)
    for key in fx.files:
        if key.startswith("grad:"):
            g = grads[key[5:]].flatten()[::16]
            assert rel_l2(g, torch.from_numpy(fx[key])) <= 3e-2, key
    with torch.no_grad():
        logits = model(input_ids=tokens, attention_mask=mask).logits
    real = torch.ones_like(tokens, dtype=torch.bool) if mask is None else mask.bool()
    # the bf16 engine against the reference in fp32: rtol / atol 5e-3 for 99 % of the logits (as for the activations'
    # models; measured: 2 of 73728 logits miss it, by up to 6.0e-3), every one within 1e-2
    got, want = logits[real.cuda()].float().cpu(), torch.from_numpy(fx["logits"])
    assert torch.isclose(got, want, rtol=5e-3, atol=5e-3).float().mean().item() >= 0.99
    assert (got - want).abs().max().item() <= 1e-2 and rel_l2(got, want) <= 1e-2


def test_alibi_moe_eager_vs_oracle():
    """MoE eager alibi model against the bf16-emulating oracle with the bias, every gradient and the logits.  The oracle
    takes the engine's expert choices (O.FORCED_ROUTING, as in test_gpu_moe.py): a bf16 router picks another expert than
    an fp32 one for near-tied logits, which is a property of the precision, not of the kernels."""
    kw = dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_head=4, n_inner=128, num_experts=8,
              num_experts_per_tok=2, attention_head_type="mha", position_embedding_type="alibi", add_bias=False,
              activation_function="swiglu")
    ocfg = O.OracleConfig(**kw)
    params = O.init_params(ocfg, seed=42)
    model = _model(kw, "eager", params, cls="moe_dolomite")
    tokens = torch.from_numpy(np.random.default_rng(3).integers(0, 512, size=(2, 64)))
    model.engine.zero_grad()
    loss = model(input_ids=tokens, labels=tokens).loss
    routing = {f"transformer.h.{i}.mlp.": layer[-1][0].sel_idx.long().cpu()
               for i, layer in enumerate(model.engine._saved["layers"])}
    loss.backward()
    grads = _grads(model)
    with torch.no_grad():
        logits = model(input_ids=tokens).logits.reshape(128, -1).float().cpu()
    ids = tokens.numpy().reshape(-1)
    lab = np.full(128, -100)
    lab[:63], lab[64:127] = ids[1:64], ids[65:]
    p = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    O.FORCED_ROUTING.clear()
    O.FORCED_ROUTING.update(routing)
    try:
        with A.install(alibi_slopes(4), bias_bf16=True):
            ref_logits = O.forward_logits(p, ocfg, ids, np.tile(np.arange(64), 2), np.array([0, 64, 128], dtype=np.int32),
                                          bf16=True)
        ref = torch.nn.functional.cross_entropy(ref_logits.float(), torch.as_tensor(lab), ignore_index=-100)
        ref.backward()
    finally:
        O.FORCED_ROUTING.clear()
    assert abs(loss.item() - ref.item()) <= 1e-3 * ref.item()
    assert rel_l2(logits, ref_logits.detach()) < 1e-2
    assert (logits - ref_logits.detach()).abs().max() < 4 * 2.0**-8 * ref_logits.detach().abs().max() + 5e-3
    for k, v in p.items():
        assert rel_l2(grads[k], v.grad) <= 3e-2, k


def test_sdpa_without_mask_is_nope_bit_for_bit():
    kw = {**_BASE, "n_head": 8, "attention_head_type": "mha"}
    params = O.init_params(O.OracleConfig(**kw), seed=42)
    tokens = torch.from_numpy(np.random.default_rng(4).integers(0, 512, size=(2, 40)))
    with torch.no_grad():
        a = _model(kw, "sdpa", params)(input_ids=tokens).logits
        b = _model({**kw, "position_embedding_type": "nope"}, "sdpa", params)(input_ids=tokens).logits
        c = _model(kw, "eager", params)(input_ids=tokens).logits
    assert torch.equal(a, b)
    assert not torch.equal(a, c)


def test_left_padded_eager_batch_equals_unpadded_documents():
    kw = {**_BASE, "n_head": 8, "num_key_value_heads": 2, "attention_head_type": "gqa"}
    model = _model(kw, "eager")
    rng = np.random.default_rng(5)
    docs = [rng.integers(0, 512, size=n) for n in (40, 23, 7)]
    S = 40
    tokens = torch.zeros(3, S, dtype=torch.long)
    mask = torch.zeros(3, S, dtype=torch.long)
    for b, d in enumerate(docs):
        tokens[b, S - len(d):] = torch.from_numpy(d)
        mask[b, S - len(d):] = 1
    with torch.no_grad():
        padded = model(input_ids=tokens, attention_mask=mask).logits
        for b, d in enumerate(docs):
            alone = model(input_ids=torch.from_numpy(d)[None]).logits[0]
            assert torch.equal(padded[b, S - len(d):], alone), b


def _step(model, tokens, mask):
    model.engine.zero_grad()
    loss = model(input_ids=tokens, attention_mask=mask, labels=tokens).loss
    loss.backward()
    return loss.detach().clone(), _grads(model)


def test_alibi_steps_are_run_to_run_identical_and_checkpointing_keeps_gradients():
    kw = {**_BASE, "n_head": 8, "attention_head_type": "mha", "attn_pdrop": 0.1}
    model = _model(kw, "eager")
    tokens = torch.from_numpy(np.random.default_rng(6).integers(0, 512, size=(3, 200)))
    mask = torch.ones_like(tokens)
    mask[1, :37] = 0
    model.engine.dropout_seed = 11
    l1, g1 = _step(model, tokens, mask)
    model.engine.dropout_seed, model.engine._dropout_passes = 11, 0
    l2, g2 = _step(model, tokens, mask)
    model.engine.checkpoint_every = 1
    model.engine.dropout_seed, model.engine._dropout_passes = 11, 0
    l3, g3 = _step(model, tokens, mask)
    assert torch.equal(l1, l2) and torch.equal(l1, l3)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k
        assert torch.equal(g1[k], g3[k]), k


@pytest.mark.parametrize("impl", ["eager", "sdpa"])
def test_cached_greedy_generation_equals_stepwise_argmax(impl):
    kw = {**_BASE, "n_head": 6, "n_embd": 96, "attention_head_type": "mha"}
    model = _model(kw, impl)
    model.eval()
    prompt = torch.from_numpy(np.random.default_rng(8).integers(0, 512, size=(2, 12)))
    mask = torch.ones_like(prompt)
    mask[0, :5] = 0
    cached = model.generate(input_ids=prompt, attention_mask=mask, max_new_tokens=24, eos_token_id=-1)
    stepwise = model.generate(input_ids=prompt, attention_mask=mask, max_new_tokens=24, eos_token_id=-1, use_cache=False)
    assert torch.equal(cached, stepwise)


def test_padded_pretraining_rope_loss_is_bit_identical_to_padding_free():
    kw = {**_BASE, "position_embedding_type": "rope", "n_head": 8, "attention_head_type": "mha"}
    from dolomite_engine_b200.hf_models.config import GPTDolomiteConfig

    tokens = torch.from_numpy(np.random.default_rng(9).integers(0, 512, size=(2, 129)))
    losses = []
    for padding_free, impl in ((True, "flash_attention_2"), (False, "sdpa"), (False, "eager")):
        losses.append(_wrapper_loss(GPTDolomiteConfig(**{**_ENGINE, **kw}), padding_free, impl, tokens))
    assert torch.equal(losses[0], losses[1]) and torch.equal(losses[0], losses[2])


def _wrapper_loss(config, padding_free, impl, tokens):
    from dolomite_engine_b200.model_wrapper import ModelWrapperForPretraining

    w = ModelWrapperForPretraining(mode="training", model_name=None, pretrained_config=config.to_dict(),
                                   model_class="AutoModelForCausalLM", dtype=torch.bfloat16, efficient_initialization=False,
                                   attention_implementation=impl, use_padding_free_transformer=padding_free, random_seed=42,
                                   micro_batch_size=2, sequence_length=128, device="cuda")
    return w({"text": tokens}).detach().clone()


def test_padded_pretraining_rejects_reset_attention_mask():
    from dolomite_engine_b200.hf_models.config import GPTDolomiteConfig
    from dolomite_engine_b200.model_wrapper import ModelWrapperForPretraining

    cfg = GPTDolomiteConfig(**{**_ENGINE, **_BASE, "n_head": 8, "attention_head_type": "mha"})
    with pytest.raises(AssertionError, match="reset_attention_mask"):
        ModelWrapperForPretraining(mode="training", model_name=None, pretrained_config=cfg.to_dict(),
                                   model_class="AutoModelForCausalLM", dtype=torch.bfloat16, efficient_initialization=False,
                                   attention_implementation="eager", use_padding_free_transformer=False, random_seed=42,
                                   micro_batch_size=2, sequence_length=64, reset_attention_mask=True, device="cuda")


def _pretraining_wrapper(impl, tokens, position_embedding_type="alibi"):
    from dolomite_engine_b200.hf_models.config import GPTDolomiteConfig
    from dolomite_engine_b200.model_wrapper import ModelWrapperForPretraining

    cfg = GPTDolomiteConfig(**{**_ENGINE, **_BASE, "n_head": 8, "attention_head_type": "mha",
                               "position_embedding_type": position_embedding_type})
    S = tokens.shape[1] - 1
    return ModelWrapperForPretraining(mode="training", model_name=None, pretrained_config=cfg.to_dict(),
                                      model_class="AutoModelForCausalLM", dtype=torch.bfloat16,
                                      efficient_initialization=False, attention_implementation=impl,
                                      use_padding_free_transformer=False, random_seed=42,
                                      micro_batch_size=tokens.shape[0], sequence_length=S, device="cuda")


def test_padded_pretraining_adds_the_bias_for_eager_and_drops_it_for_sdpa():
    """the padded pretraining wrapper passes no attention mask: an eager alibi model trains with the bias (its loss is that
    of the model's own padded forward, which the reference fixtures pin), an sdpa alibi model as NoPE, bit for bit"""
    tokens = torch.from_numpy(np.random.default_rng(10).integers(0, 512, size=(2, 161)))
    with torch.no_grad():
        eager_w = _pretraining_wrapper("eager", tokens)
        eager = eager_w({"text": tokens}).float().cpu()
        sdpa = _pretraining_wrapper("sdpa", tokens)({"text": tokens}).float().cpu()
        nope = _pretraining_wrapper("sdpa", tokens, "nope")({"text": tokens}).float().cpu()
        nope_eager = _pretraining_wrapper("eager", tokens, "nope")({"text": tokens}).float().cpu()
        logits = eager_w.model(input_ids=tokens[:, :-1]).logits.float().cpu()
    want = torch.nn.functional.cross_entropy(logits.reshape(-1, logits.shape[-1]), tokens[:, 1:].reshape(-1))
    assert torch.equal(sdpa, nope) and torch.equal(nope, nope_eager)
    assert not torch.equal(eager, nope)
    assert abs(eager.item() - want.item()) <= 1e-5 * want.item()


def test_pretrain_yaml_trains_an_eager_alibi_model(tmp_path):
    """`python -m dolomite_engine_b200.pretrain` with an alibi YAML: eager attention, padded batches"""
    import subprocess
    import sys

    import yaml

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "configs", "c1_tiny.yml")) as f:
        cfg = yaml.safe_load(f)
    cfg["model_args"]["pretrained_config"]["position_embedding_type"] = "alibi"
    cfg["model_args"]["attention_implementation"] = "eager"
    cfg["model_args"]["use_padding_free_transformer"] = False
    cfg["save_args"]["save_path"] = str(tmp_path / "ckpt")
    cfg["training_parameters"]["num_training_steps"] = 10
    path = tmp_path / "alibi.yml"
    path.write_text(yaml.safe_dump(cfg))
    proc = subprocess.run([sys.executable, "-m", "dolomite_engine_b200.pretrain", "--config", str(path)], cwd=root,
                          capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stderr[-3000:]
    losses = [float(line.split("loss ")[1].split()[0]) for line in proc.stdout.splitlines() if line.startswith("step ")]
    assert len(losses) == 10 and all(math.isfinite(x) for x in losses), proc.stdout[-2000:]
