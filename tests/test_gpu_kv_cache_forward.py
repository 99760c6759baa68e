"""GPU: the model's forward with a KV cache (`use_cache=True` / `past_key_values` on padded batches, engine.extend and the
attn_cache kernel) against one uncached padded forward over the whole sequence, greedy decoding through it against
`model.generate`, and its output layout, labels and errors."""

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
_COMMON = dict(vocab_size=512, n_positions=512, n_layer=2, resid_pdrop=0.0, embd_pdrop=0.0, attn_pdrop=0.0, eos_token_id=3,
               bos_token_id=3, pad_token_id=3)
MODELS = {
    "gqa_rope_swiglu": (dict(n_embd=256, n_head=8, num_key_value_heads=2, attention_head_type="gqa", n_inner=512,
                             position_embedding_type="rope", activation_function="swiglu", normalization_function="rmsnorm",
                             add_bias=False), "sdpa", "gpt_dolomite"),
    "bigcode": (dict(n_embd=256, n_head=4, attention_head_type="mqa", n_inner=1024, position_embedding_type="learned_absolute",
                     activation_function="gelu_pytorch_tanh", normalization_function="layernorm", add_bias=True),
                "sdpa", "gpt_dolomite"),
    "alibi_eager": (dict(n_embd=320, n_head=4, attention_head_type="mha", n_inner=640, position_embedding_type="alibi",
                         activation_function="swiglu", normalization_function="rmsnorm", add_bias=False), "eager",
                    "gpt_dolomite"),
    "alibi_sdpa": (dict(n_embd=320, n_head=4, attention_head_type="mha", n_inner=640, position_embedding_type="alibi",
                        activation_function="swiglu", normalization_function="rmsnorm", add_bias=False), "sdpa",
                   "gpt_dolomite"),
    "mqa_hd256": (dict(n_embd=512, n_head=2, attention_head_type="mqa", n_inner=1024, position_embedding_type="rope",
                       activation_function="swiglu", normalization_function="rmsnorm", add_bias=False), "sdpa",
                  "gpt_dolomite"),
    "moe": (dict(n_embd=256, n_head=4, num_key_value_heads=2, attention_head_type="gqa", n_inner=256, num_experts=4,
                 num_experts_per_tok=2, position_embedding_type="rope", activation_function="swiglu",
                 normalization_function="rmsnorm", add_bias=False), "sdpa", "moe_dolomite"),
}
CHUNKS = (1, 3, 17, 64, 130)


def _model(name, padding_free=False):
    from dolomite_engine_b200.hf_models.config import GPTDolomiteConfig, MoEDolomiteConfig
    from dolomite_engine_b200.hf_models.modeling import GPTDolomiteForCausalLM, MoEDolomiteForCausalLM

    kw, impl, mt = MODELS[name]
    Cfg, M = (GPTDolomiteConfig, GPTDolomiteForCausalLM) if mt == "gpt_dolomite" else (MoEDolomiteConfig, MoEDolomiteForCausalLM)
    model = M(Cfg(**{**_COMMON, **kw}), attn_implementation=impl, use_padding_free_transformer=padding_free, seed=42,
              device=DEV)
    model.eval()
    return model


def _prompt(seed=5, lens=(20, 7, 13)):
    """left padded ragged prompt"""
    g = torch.Generator().manual_seed(seed)
    W = max(lens)
    ids = torch.full((len(lens), W), 3, dtype=torch.long)
    mask = torch.zeros(len(lens), W, dtype=torch.long)
    for r, n in enumerate(lens):
        ids[r, W - n:] = torch.randint(4, 512, (n,), generator=g)
        mask[r, W - n:] = 1
    return ids, mask


def _chunk(S, seed):
    """[3, S] new tokens: row 0 all real, row 1 right padded, row 2 with its first token masked (no real token at S = 1)"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(4, 512, (3, S), generator=g)
    mask = torch.ones(3, S, dtype=torch.long)
    mask[1, S - S // 3:] = 0
    mask[2, 0] = 0
    return ids, mask


def _close(got, ref, what):
    """the bar test_zzz_generation puts on cached against recomputed logits"""
    err = (got.float() - ref.float()).abs().max().item()
    assert err < 4e-2 * max(1.0, ref.float().abs().max().item()), (what, err)


@pytest.mark.parametrize("name", sorted(MODELS))
def test_chunks_through_the_cache_match_one_uncached_forward(name):
    model = _model(name)
    ids, mask = _prompt()
    parts = [(ids, mask)] + [_chunk(S, 100 + S) for S in CHUNKS]
    full_ids = torch.cat([p[0] for p in parts], 1)
    full_mask = torch.cat([p[1] for p in parts], 1)
    with torch.no_grad():
        ref = model(input_ids=full_ids, attention_mask=full_mask).logits
        out = model(input_ids=ids, attention_mask=mask, use_cache=True)
        cache = out.past_key_values
        cap0 = cache.max_len
        got = [out.logits]
        width = ids.shape[1]
        for k, (cid, cmask) in enumerate(parts[1:]):
            width += cid.shape[1]
            # the HuggingFace mask (past and new columns) and the new columns alone, alternately
            am = full_mask[:, :width] if k % 2 == 0 else cmask
            out = model(input_ids=cid, attention_mask=am, past_key_values=cache, use_cache=True)
            assert out.past_key_values is cache and cache.get_seq_length() == width
            got.append(out.logits)
    got = torch.cat(got, 1)
    real = full_mask.bool().to(DEV)
    assert torch.equal(cache.lens.cpu(), full_mask.sum(1).int())
    assert cache.max_len > cap0  # the cache grew past its first capacity
    assert bool((got[~real] == 0).all())
    col = 0
    for k, (cid, _) in enumerate(parts):
        S = cid.shape[1]
        sel = real[:, col:col + S]
        _close(got[:, col:col + S][sel], ref[:, col:col + S][sel], (name, k))
        col += S


@pytest.mark.parametrize("name", ["gqa_rope_swiglu", "bigcode", "alibi_eager", "alibi_sdpa", "moe"])
def test_greedy_loop_through_the_cache_is_generate(name):
    """one token per step through model(..., past_key_values=..., use_cache=True) gives exactly model.generate's tokens"""
    model = _model(name)
    ids, mask = _prompt(seed=8)
    N = 12
    want = model.generate(input_ids=ids, attention_mask=mask, max_new_tokens=N, eos_token_id=-1)[:, ids.shape[1]:]
    with torch.no_grad():
        out = model(input_ids=ids, attention_mask=mask, use_cache=True)
        am = mask.to(DEV)
        toks = [out.logits[:, -1].float().argmax(-1)]
        for _ in range(N - 1):
            am = torch.cat([am, torch.ones_like(am[:, :1])], 1)
            out = model(input_ids=toks[-1][:, None], attention_mask=am, past_key_values=out.past_key_values, use_cache=True)
            toks.append(out.logits[:, -1].float().argmax(-1))
    assert torch.equal(torch.stack(toks, 1), want)


def test_tuple_layout_and_labels():
    model = _model("gqa_rope_swiglu")
    ids, mask = _prompt()
    labels = torch.where(mask.bool(), ids, torch.full_like(ids, -100))
    with torch.no_grad():
        ref = model(input_ids=ids, attention_mask=mask, labels=labels)
        out = model(input_ids=ids, attention_mask=mask, labels=labels, use_cache=True)
        tup = model(input_ids=ids, attention_mask=mask, labels=labels, use_cache=True, return_dict=False)
        assert len(tup) == 3 and torch.equal(tup[0], out.loss) and torch.equal(tup[1], out.logits)
        assert tup[2].get_seq_length() == ids.shape[1]
        no_lab = model(input_ids=ids, attention_mask=mask, use_cache=True, return_dict=False)
        assert len(no_lab) == 2 and torch.equal(no_lab[0], out.logits)
        # the chunk's loss is the padded path's loss of the same tokens
        assert torch.allclose(out.loss.float(), ref.loss.float(), rtol=1e-3, atol=1e-4), (out.loss, ref.loss)
        cid, cmask = _chunk(17, 1)
        clab = torch.where(cmask.bool(), cid, torch.full_like(cid, -100))
        step = model(input_ids=cid, attention_mask=cmask, labels=clab, past_key_values=out.past_key_values)
    lg = step.logits[:, :-1].float()
    tgt = clab.to(DEV)[:, 1:].clone()
    tgt[~(cmask.bool().to(DEV)[:, :-1] & cmask.bool().to(DEV)[:, 1:])] = -100
    want = F.cross_entropy(lg.reshape(-1, lg.shape[-1]), tgt.reshape(-1), ignore_index=-100)
    assert torch.allclose(step.loss.float(), want, rtol=1e-3, atol=1e-4), (step.loss, want)


def test_errors():
    from transformers import DynamicCache

    model = _model("moe")
    ids, mask = _prompt()
    with torch.no_grad():
        cache = model(input_ids=ids, attention_mask=mask, use_cache=True).past_key_values
        with pytest.raises(TypeError, match="past_key_values must be the KVCache"):
            model(input_ids=ids[:, :1], past_key_values=((torch.zeros(1), torch.zeros(1)),))
        with pytest.raises(TypeError, match="past_key_values must be the KVCache"):
            model(input_ids=ids[:, :1], past_key_values=DynamicCache())
        with pytest.raises(NotImplementedError, match="output_router_logits"):
            model(input_ids=ids[:, :1], past_key_values=cache, output_router_logits=True)
        with pytest.raises(ValueError, match="attention_mask must be"):
            model(input_ids=ids[:, :2], attention_mask=mask[:, :5], past_key_values=cache)
    model.train()
    with pytest.raises(NotImplementedError, match="training through a KV cache"):
        model(input_ids=ids, attention_mask=mask, use_cache=True)
    free = _model("gqa_rope_swiglu", padding_free=True)
    with pytest.raises(NotImplementedError, match="KV caching is not supported with padding_free transformer"):
        free(input_ids=[[5, 6, 7]], use_cache=True)
    # use_cache=None keeps the uncached padded forward: no cache is made
    with torch.no_grad():
        assert _model("gqa_rope_swiglu")(input_ids=ids, attention_mask=mask).past_key_values is None
