"""Autoregressive decoding on top of the packed training engine (reference surface: `model.generate(**batch,
**generate_kwargs, eos_token_id=...)` as called by model_wrapper/base.py:110-136 with the GenerationParameters of
arguments.py: max_new_tokens, do_sample, temperature, top_k, top_p).

`use_cache=True` (default, like HuggingFace): the prompts are packed as documents and run ONCE through the training
forward, which also fills a KV cache (`engine.prefill`); every further token is one `engine.decode_step` -- the training
kernels at T = batch rows plus the single-query cache attention kernel (csrc/attention_decode.cu) -- i.e. O(L) work per token.
`use_cache=False` re-runs the packed forward over the whole prefix for every token (exact by construction, O(L^2) per sequence;
the cached path is checked against it on the GPU).
"""

from __future__ import annotations

import torch


def _filter_logits(logits: torch.Tensor, temperature: float | None, top_k: int | None, top_p: float | None) -> torch.Tensor:
    """temperature -> top-k -> nucleus, the order HuggingFace's logits warpers apply"""
    if temperature is not None and temperature != 1.0:
        logits = logits / float(temperature)
    if top_k is not None and 0 < top_k < logits.shape[-1]:
        kth = logits.topk(int(top_k), dim=-1).values[..., -1:]
        logits = logits.masked_fill(logits < kth, float("-inf"))
    if top_p is not None and 0.0 < top_p < 1.0:
        srt, idx = logits.sort(dim=-1, descending=False)
        cum = srt.softmax(-1).cumsum(-1)
        drop = cum <= (1.0 - float(top_p))
        drop[..., -1] = False  # always keep the most likely token
        logits = logits.masked_fill(drop.scatter(-1, idx, drop), float("-inf"))
    return logits


@torch.no_grad()
def last_token_logits(model, input_ids: torch.Tensor, attention_mask: torch.Tensor) -> torch.Tensor:
    """fp32 [B, V] logits of every row's last real token; rows are packed as documents (empty rows are not allowed)"""
    from .modeling import _EngineFunction, _pad_packed_stream

    dev = model.engine.device
    mask = attention_mask.to(dev).bool()
    lens = mask.sum(1)
    lens_host = lens.tolist()
    if min(lens_host) < 1:
        raise ValueError("generate: every prompt needs at least one token")
    keep = mask.reshape(-1).nonzero(as_tuple=True)[0]
    ids = input_ids.to(dev).long().reshape(-1)[keep].contiguous()
    pos = (mask.long().cumsum(-1) - 1).clamp_(min=0).reshape(-1)[keep].contiguous()
    cu = torch.zeros(len(lens_host) + 1, dtype=torch.int32, device=dev)
    cu[1:] = lens.cumsum(0)
    last = (cu[1:] - 1).long()
    ids, pos, cu_p, _, _ = _pad_packed_stream(ids, pos, cu, None)
    # the reference's `generate` always passes an attention mask, so eager and SDPA both add the ALiBi bias
    logits = _EngineFunction.apply(model._anchor, model, ids, pos, cu_p, int(max(lens_host)), None, -100, False,
                                   model._alibi_pass(True))
    return logits[last].float()


@torch.no_grad()
def _prefill(model, input_ids: torch.Tensor, attention_mask: torch.Tensor, max_new_tokens: int):
    """packed forward over the (left padded) prompts that fills a KV cache -> (fp32 [B, V] logits of the last prompt tokens, cache)"""
    from ..engine import KVCache
    from .modeling import _pad_packed_stream

    eng = model.engine
    dev = eng.device
    mask = attention_mask.to(dev).bool()
    lens = mask.sum(1)
    lens_host = lens.tolist()
    if min(lens_host) < 1:
        raise ValueError("generate: every prompt needs at least one token")
    keep = mask.reshape(-1).nonzero(as_tuple=True)[0]
    ids = input_ids.to(dev).long().reshape(-1)[keep].contiguous()
    pos = (mask.long().cumsum(-1) - 1).clamp_(min=0).reshape(-1)[keep].contiguous()
    cu = torch.zeros(len(lens_host) + 1, dtype=torch.int32, device=dev)
    cu[1:] = lens.cumsum(0)
    last = (cu[1:] - 1).long()
    B = len(lens_host)
    cache = KVCache(eng, B, max(lens_host) + max_new_tokens + 8)
    # (the packed stream may carry a trailing dummy document that rounds the token count up to 8: it is not cached)
    ids_p, pos_p, cu_p, _, _ = _pad_packed_stream(ids, pos, cu, None)
    logits = eng.prefill(ids_p, pos_p, cu_p, int(max(lens_host)), cache, n_sequences=B, alibi=model._alibi_pass(True))
    return logits[last].float(), cache


@torch.no_grad()
def generate(model, input_ids: torch.Tensor, attention_mask: torch.Tensor | None = None, max_new_tokens: int = 20,
             do_sample: bool = False, temperature: float | None = None, top_k: int | None = None, top_p: float | None = None,
             eos_token_id: int | None = None, pad_token_id: int | None = None, generator: torch.Generator | None = None,
             **unused) -> torch.Tensor:
    """-> LongTensor [B, L + n] (prompt included, like HuggingFace's decoder-only `generate`): rows that emitted
    `eos_token_id` are filled with `pad_token_id` (default: eos); stops early once every row is finished."""
    unsupported = {k: v for k, v in unused.items() if v not in (None, False, 1, 1.0) and k not in ("use_cache",)}
    if unsupported:
        raise NotImplementedError(f"generate: unsupported options {sorted(unsupported)}")
    dev = model.engine.device
    ids = torch.as_tensor(input_ids).to(dev).long()
    assert ids.dim() == 2, "generate takes a [batch, sequence] prompt (left padded when ragged)"
    mask = torch.ones_like(ids, dtype=torch.bool) if attention_mask is None else torch.as_tensor(attention_mask).to(dev).bool()
    eos = model.config.eos_token_id if eos_token_id is None else eos_token_id
    pad = eos if pad_token_id is None else pad_token_id
    B = ids.shape[0]
    finished = torch.zeros(B, dtype=torch.bool, device=dev)
    limit = getattr(model.config, "n_positions", None)
    use_cache = unused.get("use_cache", True) is not False and model.engine.comm is None
    cache = None
    for step in range(int(max_new_tokens)):
        if limit is not None and model.engine.learned_positions and int(mask.sum(1).max()) >= limit:
            break  # learned absolute positions end at n_positions
        if not use_cache:
            logits = last_token_logits(model, ids, mask)
        elif cache is None:
            logits, cache = _prefill(model, ids, mask, int(max_new_tokens))
        else:
            logits = model.engine.decode_step(ids[:, -1].contiguous(), cache, active=~was_finished,
                                              alibi=model._alibi_pass(True)).float()
        was_finished = finished.clone()
        if do_sample:
            probs = _filter_logits(logits, temperature, top_k, top_p).softmax(-1)
            nxt = torch.multinomial(probs, 1, generator=generator).squeeze(1)
        else:
            nxt = logits.argmax(-1)
        nxt = torch.where(finished, torch.full_like(nxt, pad), nxt)
        ids = torch.cat([ids, nxt[:, None]], dim=1)
        # finished rows keep their length: their fill tokens are not part of the packed stream
        mask = torch.cat([mask, (~finished)[:, None]], dim=1)
        finished = finished | (nxt == eos)
        if bool(finished.all()):
            break
    return ids
