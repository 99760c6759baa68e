"""CPU: vocabularies that are not a multiple of 8 -- the configurations the engine accepts, the [rows, V] buffer layout,
the parameter shapes, the FP8 head rule, and the oracle against the reference fixtures of tools/pin_vocab.py."""

import os

import numpy as np
import pytest
import torch

import oracle.dolomite_oracle as O
from dolomite_engine_b200 import kernels as K
from dolomite_engine_b200.engine import _root_specs, check_supported
from dolomite_engine_b200.fp8 import fp8_weight_names
from dolomite_engine_b200.hf_models.config import GPTDolomiteConfig

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
VOCABS = [2049, 2050, 2051, 2052, 2053, 2054, 2055, 49155, 50257]
# tools/pin_vocab.py MODELS
MODELS = {
    "bigcode_2053": dict(vocab_size=2053, n_positions=256, n_embd=128, n_layer=2, n_head=8, n_inner=512,
                         attention_head_type="mqa", activation_function="gelu_pytorch_tanh", add_bias=True,
                         normalization_function="layernorm", position_embedding_type="learned_absolute",
                         tie_word_embeddings=False),
    "gqa_rope_2051": dict(vocab_size=2051, n_positions=256, n_embd=128, n_layer=2, n_head=8, num_key_value_heads=2,
                          n_inner=256, attention_head_type="gqa", activation_function="swiglu", add_bias=False),
    "moe_2055": dict(vocab_size=2055, n_positions=256, n_embd=128, n_layer=2, n_head=8, n_inner=128,
                     attention_head_type="mha", activation_function="swiglu", add_bias=False, num_experts=8,
                     num_experts_per_tok=2),
}
EOS = 7


def subsample(g):
    """the gradient samples tools/pin_vocab.py keeps: small tensors whole, else every 16th element"""
    g = g.flatten()
    return g if g.numel() <= 4096 else g[::16]


def _cfg(**kw):
    base = dict(n_embd=256, n_head=4, attention_head_type="mha", position_embedding_type="rope",
                activation_function="swiglu", normalization_function="rmsnorm", resid_pdrop=0, embd_pdrop=0, attn_pdrop=0,
                vocab_size=2048)
    base.update(kw)
    return GPTDolomiteConfig(**base)


@pytest.mark.parametrize("V", VOCABS)
def test_any_vocabulary_is_accepted(V):
    check_supported(_cfg(vocab_size=V))
    check_supported(_cfg(vocab_size=V, tie_word_embeddings=False))


@pytest.mark.parametrize("kw", [dict(n_embd=1028, n_head=16), dict(n_inner=1020)])
def test_hidden_widths_still_need_multiples_of_8(kw):
    with pytest.raises(NotImplementedError, match="n_embd and n_inner"):
        check_supported(_cfg(vocab_size=50257, **kw))


def test_reference_pretraining_example_model_is_accepted():
    """the model block of the reference's configs/pretraining-examples/pretrain-2.yml, with its real vocabulary"""
    block = dict(model_type="gpt_dolomite", vocab_size=50257, n_positions=2048, n_embd=768, n_layer=12, n_head=12,
                 num_key_value_heads=None, n_inner=None, activation_function="gelu_pytorch_tanh",
                 attention_head_type="mqa", resid_pdrop=0.1, embd_pdrop=0.1, attn_pdrop=0.1,
                 normalization_function="layernorm", layer_norm_epsilon=1e-5, initializer_range=0.02,
                 scale_attn_weights=True, use_cache=True, bos_token_id=50256, eos_token_id=50256, pad_token_id=50256,
                 attention_softmax_in_fp32=True, add_bias=True, position_embedding_type="learned_absolute",
                 rope_theta=10000)
    cfg = GPTDolomiteConfig.from_dict(block)
    assert cfg.vocab_size == 50257
    check_supported(cfg)


@pytest.mark.parametrize("tied", [True, False])
def test_vocabulary_parameters_keep_their_exact_shape(tied):
    specs = {name: shape for name, shape, _ in _root_specs(_cfg(vocab_size=50257, tie_word_embeddings=tied))}
    assert specs["transformer.wte.weight"] == (50257, 256)
    assert specs.get("lm_head.weight") == (None if tied else (50257, 256))


def test_fp8_keeps_an_odd_vocabulary_head_in_bf16():
    assert "lm_head.weight" not in fp8_weight_names(_cfg(vocab_size=2053, tie_word_embeddings=False))
    assert "lm_head.weight" not in fp8_weight_names(_cfg(vocab_size=2056, tie_word_embeddings=False))  # TE: V % 16
    assert "lm_head.weight" in fp8_weight_names(_cfg(vocab_size=2064, tie_word_embeddings=False))


@pytest.mark.parametrize("cols", [1, 7, 8, 9, 2051, 2056, 50257])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_row_buffers_keep_16_byte_strides(cols, dtype):
    t = K.rows_empty(5, cols, dtype)
    per = 16 // t.element_size()
    assert t.shape == (5, cols) and t.stride(1) == 1 and t.stride(0) == -(-cols // per) * per
    assert t.is_contiguous() == (cols % per == 0)
    x = torch.randn(5, cols).to(dtype)
    y = K.rows_aligned(x)
    assert torch.equal(y, x) and y.stride(0) == t.stride(0)
    assert (y is x) == (cols % per == 0)


def _fixture_params(cfg, fx):
    params = O.init_params(cfg, seed=42)
    for k in params:
        if f"bias:{k}" in fx:
            params[k] = torch.from_numpy(fx[f"bias:{k}"])
    return params


def _packed_inputs(fx):
    inp, labels = O.split_tokens(fx["packed_tokens"])
    b = O.prepare_model_inputs(inp.copy(), EOS, True, True)
    return b["input_ids"], b["position_ids"], b["cu_seqlens"], np.ascontiguousarray(labels).reshape(-1)


def _padded_inputs(fx):
    m = fx["padded_mask"].astype(bool)
    ids = fx["padded_tokens"][m]
    lens = m.sum(1)
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    pos = np.concatenate([np.arange(n) for n in lens])
    labels = np.full(ids.shape, -100, dtype=np.int64)
    for d in range(len(lens)):
        labels[cu[d] : cu[d + 1] - 1] = ids[cu[d] + 1 : cu[d + 1]]
    return ids, pos, cu, labels


@pytest.mark.parametrize("name", list(MODELS))
@pytest.mark.parametrize("batch", ["packed", "padded"])
def test_oracle_matches_the_reference_fixtures(name, batch):
    fx = np.load(os.path.join(GOLDEN, f"model_vocab_{name}.npz"))
    cfg = O.OracleConfig(**MODELS[name])
    params = _fixture_params(cfg, fx)
    ids, pos, cu, labels = (_packed_inputs if batch == "packed" else _padded_inputs)(fx)
    p = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    logits = O.forward_logits(p, cfg, ids, pos, cu)
    assert logits.shape[-1] == cfg.vocab_size
    loss = torch.nn.functional.cross_entropy(logits, torch.as_tensor(labels), ignore_index=-100)
    loss.backward()
    assert abs(loss.item() - float(fx[f"{batch}_loss"])) <= 1e-5
    want = torch.from_numpy(fx[f"{batch}_logits"])
    assert (logits.detach()[::8] - want).abs().max().item() <= 2e-5
    names = [k[len(f"{batch}_grad:"):] for k in fx.files if k.startswith(f"{batch}_grad:")]
    assert sorted(names) == sorted(params)
    for k in names:
        ref = torch.from_numpy(fx[f"{batch}_grad:{k}"])
        got = subsample(p[k].grad)
        assert (got - ref).abs().max().item() <= 1e-4 * ref.abs().max().item() + 1e-9, k
