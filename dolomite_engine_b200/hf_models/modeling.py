"""GPTDolomiteForCausalLM / MoEDolomiteForCausalLM behind the reference's construction + forward contract
(hf_models/models/gpt_dolomite/{base,main}.py, hf_models/models/moe_dolomite/{base,main}.py).

The module keeps the reference kwargs (`attn_implementation`, `use_padding_free_transformer`,
`normalization_implementation`, `moe_implementation`, `torch_dtype`), input validation and state-dict names, but the
computation is the explicit B200 engine (engine.py) -- there is no eager PyTorch path to fall back to.
"""

from __future__ import annotations

import json
import os
from dataclasses import dataclass

import torch
import torch.nn as nn

from ..engine import DolomiteEngine
from .config import CommonConfig, GPTDolomiteConfig, MoEDolomiteConfig, config_class_for
from .utils import convert_padding_free_lists_to_tensors


@dataclass
class CausalLMOutputWithPast:
    loss: torch.Tensor | None = None
    logits: torch.Tensor | None = None
    past_key_values: object | None = None  # engine.KVCache of a call with use_cache=True or past_key_values
    hidden_states: None = None
    attentions: None = None
    router_logits: None = None

    def to_tuple(self) -> tuple:
        return tuple(v for v in (self.loss, self.logits, self.past_key_values) if v is not None)

    def __getitem__(self, i):
        return self.to_tuple()[i]


@dataclass
class MoeCausalLMOutputWithPast:
    """transformers' MoeCausalLMOutputWithPast, returned by MoEDolomiteForCausalLM with output_router_logits=True
    (moe_dolomite/main.py:123-131)"""

    loss: torch.Tensor | None = None
    aux_loss: torch.Tensor | None = None
    logits: torch.Tensor | None = None
    past_key_values: None = None
    hidden_states: None = None
    attentions: None = None
    router_logits: tuple | None = None

    def to_tuple(self) -> tuple:
        """the return_dict=False order of the reference (main.py:117-121): (loss, aux_loss, logits, router_logits)"""
        return tuple(v for v in (self.loss, self.aux_loss, self.logits, self.router_logits) if v is not None)

    def __getitem__(self, i):
        return self.to_tuple()[i]


class _EngineFunction(torch.autograd.Function):
    """Bridges autograd to the explicit engine: the only differentiable input is a dummy anchor; parameter gradients
    are accumulated by the engine into its flat fp32 gradient buffers (exactly where FSDP would leave them)."""

    @staticmethod
    def forward(ctx, anchor, model, input_ids, position_ids, cu_seqlens, max_seqlen, labels, ignore_index, save=True,
                alibi=False, router_aux=None, neft_numel=None):
        # `save`: the caller's torch.is_grad_enabled() (always False in here); under no_grad (evaluation) no activation is kept
        # `alibi`: the pass adds the ALiBi bias (DolomitePreTrainedModel._alibi_pass)
        # `router_aux`: None, or (T_real, coef) of the MoE load-balancing loss.  The outputs are then (loss or logits,
        # aux_loss, router logits of every layer); the router logits are not differentiable
        # `neft_numel`: element count of the reference's wte output (NEFTune bound); None = the packed stream's T * n_embd
        engine = model.engine
        ctx.model = model
        ctx.loss_mode = labels is not None
        ctx.router_aux = router_aux
        if router_aux is not None:
            T_real, coef = router_aux
            logits, loss, aux, router_logits = engine.forward(
                input_ids, position_ids, cu_seqlens, max_seqlen, labels=labels, ignore_index=ignore_index,
                save_for_backward=bool(save), alibi=bool(alibi), router_aux=True, T_real=T_real, coef=coef,
                neft_numel=neft_numel)
            ctx.mark_non_differentiable(*router_logits)
            return (loss.reshape(()) if ctx.loss_mode else logits, aux.reshape(())) + tuple(router_logits)
        # `assume_unit_loss_grad` (set by the training wrappers: train_step calls loss.backward() on the raw loss) lets the
        # engine run the LM head's backward chunk-wise inside the loss computation without ever materialising [T, V]
        logits, loss = engine.forward(input_ids, position_ids, cu_seqlens, max_seqlen, labels=labels,
                                      ignore_index=ignore_index, save_for_backward=bool(save),
                                      fuse_head_loss=bool(save) and labels is not None and model.assume_unit_loss_grad,
                                      alibi=bool(alibi), neft_numel=neft_numel)
        return loss.reshape(()) if ctx.loss_mode else logits

    @staticmethod
    def backward(ctx, grad_out, *more):
        model = ctx.model
        engine = model.engine
        if ctx.router_aux is not None:
            # loss = CE + coef * aux: the router's load-balancing gradient is scaled by s = coef * dL/dloss + dL/daux,
            # formed on the device (no host sync); both upstream gradients are general here (no unit-gradient shortcut)
            g_aux = more[0].reshape(1).float()
            if ctx.loss_mode:
                g_loss = grad_out.reshape(1).float()
                engine.backward(grad_scale_dev=g_loss, aux_grad_dev=ctx.router_aux[1] * g_loss + g_aux)
            else:
                engine.backward(dlogits=grad_out.contiguous(), aux_grad_dev=g_aux)
        elif ctx.loss_mode:
            # d(loss)/d(loss) arrives as a 0-d device tensor; it is 1 for `loss.backward()` (the only thing
            # train_utils.train_step does).  Anything else is applied on the device, without a host sync.
            scale = None if model.assume_unit_loss_grad else grad_out.reshape(1).float()
            engine.backward(grad_scale_dev=scale)
        else:
            engine.backward(dlogits=grad_out.contiguous())
        return (None,) * 12


def _pad_packed_stream(input_ids, position_ids, cu_seqlens, shift_labels, multiple: int = 8):
    """The token count is the contraction length of every weight-gradient GEMM and must be a multiple of 8 (16-byte rows of
    the MN-major operands).  Pretraining streams are (mbs * seq); finetuning streams are not, so a trailing dummy document
    of < 8 tokens is appended: it attends only to itself and its labels are ignore_index, i.e. it adds nothing to the loss
    or to any gradient.  Returns the padded tensors and the number of real tokens."""
    T = int(input_ids.numel())
    pad = (-T) % multiple
    if pad == 0:
        return input_ids, position_ids, cu_seqlens, shift_labels, T
    dev = input_ids.device
    input_ids = torch.cat([input_ids, torch.zeros(pad, dtype=input_ids.dtype, device=dev)])
    position_ids = torch.cat([position_ids, torch.arange(pad, dtype=position_ids.dtype, device=dev)])
    cu_seqlens = torch.cat([cu_seqlens, torch.tensor([T + pad], dtype=cu_seqlens.dtype, device=dev)])
    if shift_labels is not None:
        shift_labels = torch.cat([shift_labels, torch.full((pad,), -100, dtype=shift_labels.dtype, device=dev)])
    return input_ids, position_ids, cu_seqlens, shift_labels, T


class DolomitePreTrainedModel(nn.Module):
    config_class = CommonConfig
    base_model_prefix = "transformer"
    _no_split_modules = ["GPTDolomiteBlock"]
    _tied_weights_keys = ["lm_head.weight"]

    def __init__(self, config: CommonConfig, **kwargs) -> None:
        super().__init__()
        self.config = config
        # ---- reference kwargs (gpt_dolomite/base.py:30-62, moe_dolomite/base.py:18-22) ----
        self.attention_implementation = kwargs.pop("attn_implementation", "flash_attention_2")
        self._use_padding_free_transformer = kwargs.pop("use_padding_free_transformer", True)
        self.normalization_implementation = kwargs.pop("normalization_implementation", "torch")
        self.moe_implementation = kwargs.pop("moe_implementation", "eager")  # moe_dolomite/base.py:21
        kwargs.pop("torch_dtype", None)
        kwargs.pop("trust_remote_code", None)
        device = kwargs.pop("device", None)
        world_size = kwargs.pop("world_size", 1)
        rank = kwargs.pop("rank", 0)
        seed = kwargs.pop("seed", 42)
        init_on_device = kwargs.pop("init_on_device", False)
        resize_vocab_to = kwargs.pop("resize_vocab_to", None)  # resize_token_embeddings before sharding (DolomiteEngine)
        if kwargs.pop("tensor_parallel_word_embeddings", False) or kwargs.pop("sequence_parallel", False):
            raise NotImplementedError("tensor / sequence parallelism is out of scope of the data-parallel B200 path")
        if kwargs:
            raise TypeError(f"unexpected keyword arguments: {sorted(kwargs)}")
        if self.attention_implementation not in ("flash_attention_2", "eager", "sdpa"):
            raise ValueError(f"unexpected `attn_implementation` {self.attention_implementation}")
        # use_padding_free_transformer=False (padded [B, S] batches + attention_mask, attention/flash.py:72-129): the reference
        # unpads around flash attention inside every layer; here the batch is unpadded ONCE in `forward`, the packed engine
        # runs on the valid tokens only, and the logits are scattered back to [B, S, V]
        if self.moe_implementation not in ("eager", "scattermoe"):
            raise ValueError(f"unexpected `moe_implementation` {self.moe_implementation}")
        if device is None:
            if not torch.cuda.is_available():
                raise RuntimeError(
                    "dolomite_engine_b200 needs a CUDA device (sm_90a); there is no CPU path. "
                    "Use oracle/ for CPU reference computations in tests."
                )
            device = torch.device("cuda", torch.cuda.current_device())
        self.engine = DolomiteEngine(config, device, world_size=world_size, rank=rank, seed=seed, init_on_device=init_on_device,
                                     attention_implementation=self.attention_implementation,
                                     use_padding_free_transformer=self._use_padding_free_transformer,
                                     moe_implementation=self.moe_implementation, resize_vocab_to=resize_vocab_to)
        self.flat_params = nn.ParameterList([u.master for u in self.engine.units])
        self._anchor = torch.zeros(1, device=device, requires_grad=True)
        self.assume_unit_loss_grad = False
        self.upcast_logits_for_loss = config.upcast_logits_for_loss
        self.m_width = config.m_width

    # ------------------------------------------------------------------------------------------
    def prepare_inputs_for_model(self, input_ids, inputs_embeds, position_ids, token_type_ids, labels, cu_seqlens,
                                 max_seqlen, past_key_values, attention_mask, use_cache, output_attentions):
        """gpt_dolomite/base.py:68-115 (padding-free branch)"""
        if isinstance(input_ids, list) or isinstance(inputs_embeds, list):
            error_message = "{variable} should not be passed for flash attention when using List[List[int]] input types for input_ids"
            assert cu_seqlens is None, error_message.format(variable="cu_seqlens")
            assert max_seqlen is None, error_message.format(variable="max_seqlen")
            assert attention_mask is None, error_message.format(variable="attention_mask")
            input_ids, position_ids, token_type_ids, labels, cu_seqlens, max_seqlen = convert_padding_free_lists_to_tensors(
                input_ids=input_ids, inputs_embeds=inputs_embeds, position_ids=position_ids,
                token_type_ids=token_type_ids, labels=labels, device=self.engine.device,
            )
        else:
            assert cu_seqlens is not None, "cu_seqlens needs to be specified when using tensor inputs with padding_free transformer"
            assert position_ids is not None, "max_seqlen needs to be specified when specifying cu_seqlens"
            assert max_seqlen is not None, "max_seqlen needs to be specified when specifying cu_seqlens"
            assert attention_mask is None, "attention_mask should not be passed when specifying cu_seqlens"
        if use_cache or past_key_values is not None:
            raise NotImplementedError("KV caching is not supported with padding_free transformer")
        assert not output_attentions
        if inputs_embeds is not None:
            raise NotImplementedError("inputs_embeds is not supported on the B200 padding-free path")
        if token_type_ids is not None:
            raise NotImplementedError("token_type_ids is not supported on the B200 padding-free path")
        return input_ids, position_ids, token_type_ids, labels, cu_seqlens, max_seqlen

    def forward(self, input_ids=None, past_key_values=None, attention_mask=None, token_type_ids=None, position_ids=None,
                inputs_embeds=None, labels=None, use_cache=None, output_attentions=None, output_hidden_states=None,
                return_dict=True, cu_seqlens=None, max_seqlen=None, output_router_logits=None):
        if output_router_logits and self._use_padding_free_transformer:
            # moe_dolomite/main.py:47-48
            raise NotImplementedError("padding_free is not supported with load_balancing_loss_func currently")
        assert not output_hidden_states, "output_hidden_states is not supported on the B200 path"
        if not self._use_padding_free_transformer:
            return self._forward_padded(input_ids, attention_mask, position_ids, labels, return_dict, past_key_values,
                                        use_cache, inputs_embeds, token_type_ids, cu_seqlens,
                                        output_router_logits=bool(output_router_logits))
        input_ids, position_ids, token_type_ids, labels, cu_seqlens, max_seqlen = self.prepare_inputs_for_model(
            input_ids, inputs_embeds, position_ids, token_type_ids, labels, cu_seqlens, max_seqlen, past_key_values,
            attention_mask, use_cache, output_attentions,
        )
        dev = self.engine.device
        input_ids = input_ids.to(dev).reshape(-1).long().contiguous()
        position_ids = position_ids.to(dev).reshape(-1).contiguous()
        if position_ids.dtype not in (torch.int32, torch.int64):
            position_ids = position_ids.long()
        cu_seqlens = cu_seqlens.to(dev, torch.int32).contiguous()
        if isinstance(max_seqlen, torch.Tensor):
            max_seqlen = int(max_seqlen.item())  # the reference syncs here too (flash-attn takes a python int)
        shift_labels = None
        if labels is not None:
            # gpt_dolomite/main.py:185-191 : logits[:-1] vs labels[1:], document-final positions dropped
            labels = labels.to(dev).reshape(-1).long()
            shift_labels = torch.full_like(labels, -100)
            shift_labels[:-1] = labels[1:]
            drop = (cu_seqlens[1:-1] - 1).long()
            shift_labels[drop] = -100
        input_ids, position_ids, cu_seqlens, shift_labels, T_real = _pad_packed_stream(input_ids, position_ids, cu_seqlens,
                                                                                       shift_labels, self._token_multiple())
        # NEFTune's bound uses the reference's wte output, the T_real tokens of the lists (not the multiple-of-8 pad)
        out = _EngineFunction.apply(self._anchor, self, input_ids, position_ids, cu_seqlens, int(max_seqlen), shift_labels, -100,
                                    torch.is_grad_enabled(), False, None, T_real * self.config.n_embd)
        if shift_labels is not None:
            result = CausalLMOutputWithPast(loss=out, logits=None)
        else:
            result = CausalLMOutputWithPast(loss=None, logits=out[:T_real])
        if not return_dict:
            return tuple(v for v in (result.loss, result.logits) if v is not None)
        return result

    def _alibi_pass(self, has_attention_mask: bool) -> bool:
        """Whether a padded-batch pass adds the ALiBi bias (gpt_dolomite/base.py:559-598 `_get_maybe_causal_mask`): eager
        attention always adds it through its mask; SDPA only when an attention_mask is passed -- without one it runs
        `is_causal=True` and the bias is dropped (attention/sdpa.py:56-64), so an sdpa + alibi model runs as NoPE."""
        if self.engine.alibi_slopes is None:
            return False
        return self.attention_implementation == "eager" or has_attention_mask

    def _token_multiple(self) -> int:
        """FP8 training forward: the token count is also the row length of the transposed fp8 operands of the weight
        gradients, which the FP8 GEMM wants in multiples of 16.  Evaluation and generation run bf16 and pack as bf16 does."""
        e = self.engine
        return 16 if e.fp8 is not None and e.fp8_autocast and e.training and torch.is_grad_enabled() else 8

    def _forward_padded(self, input_ids, attention_mask, position_ids, labels, return_dict, past_key_values, use_cache,
                        inputs_embeds, token_type_ids, cu_seqlens, output_router_logits: bool = False):
        """Padded batch path (gpt_dolomite/base.py:374-522 non-padding-free branch + attention/flash.py unpad/pad):
        input_ids [B, S], attention_mask [B, S] (1 = token, left or right padding), labels [B, S] (-100 at padding).
        position_ids default to `cumsum(mask) - 1` (base.py:524-534); loss = CE(logits[:, :-1], labels[:, 1:]) over the
        non-ignored positions (main.py:179-202).  Every row becomes one document of the packed stream.
        `output_router_logits` (MoE, moe_dolomite/main.py:30-130): also the load-balancing loss over the real tokens
        (`aux_loss`; `loss` = CE + router_aux_loss_coef * aux_loss) and every layer's router logits as [B*S, E], zero at
        padding."""
        if output_router_logits and not self.engine.is_moe:
            raise ValueError("output_router_logits needs an MoE model (MoEDolomiteForCausalLM)")
        if use_cache or past_key_values is not None:
            return self._forward_cached(input_ids, attention_mask, position_ids, labels, return_dict, past_key_values,
                                        inputs_embeds, token_type_ids, cu_seqlens, output_router_logits)
        if inputs_embeds is not None or token_type_ids is not None:
            raise NotImplementedError("inputs_embeds / token_type_ids are not supported on the B200 path")
        assert cu_seqlens is None, "cu_seqlens belongs to the padding-free transformer"
        dev = self.engine.device
        input_ids = torch.as_tensor(input_ids).to(dev).long()
        assert input_ids.dim() == 2, "padded batches are [batch, sequence]"
        B, S = input_ids.shape
        mask = torch.ones(B, S, dtype=torch.bool, device=dev) if attention_mask is None else attention_mask.to(dev).bool()
        if position_ids is None:
            position_ids = (mask.long().cumsum(-1) - 1).clamp_(min=0)
        position_ids = position_ids.to(dev).long()
        lens = mask.sum(1)
        keep = mask.reshape(-1).nonzero(as_tuple=True)[0]
        lens_host = lens.tolist()  # one host sync, like the reference's unpad (`max_seqlen_in_batch.item()`)
        ends, total = [0], 0
        for n in lens_host:  # empty rows contribute no document
            if n > 0:
                total += int(n)
                ends.append(total)
        cu = torch.tensor(ends, dtype=torch.int32, device=dev)
        max_seqlen = max(lens_host) if lens_host else 0
        ids_p = input_ids.reshape(-1)[keep].contiguous()
        pos_p = position_ids.reshape(-1)[keep].contiguous()
        shift_labels = None
        if labels is not None:
            lab = torch.as_tensor(labels).to(dev).long()
            nxt = torch.full_like(lab, -100)
            nxt[:, :-1] = lab[:, 1:]
            # the successor must be a real token of the same row: drop targets that sit on padding
            nxt_valid = torch.zeros_like(mask)
            nxt_valid[:, :-1] = mask[:, 1:]
            nxt = torch.where(nxt_valid & mask, nxt, torch.full_like(nxt, -100))
            shift_labels = nxt.reshape(-1)[keep].contiguous()
        ids_p, pos_p, cu, shift_labels, T_real = _pad_packed_stream(ids_p, pos_p, cu, shift_labels, self._token_multiple())
        router_aux = (T_real, float(self.config.router_aux_loss_coef)) if output_router_logits else None
        out = _EngineFunction.apply(self._anchor, self, ids_p, pos_p, cu, int(max(max_seqlen, 1)), shift_labels, -100,
                                    torch.is_grad_enabled(), self._alibi_pass(attention_mask is not None), router_aux,
                                    B * S * self.config.n_embd)  # NEFTune: the reference's wte sees [B, S], padding included
        aux_loss = router_logits = None
        if router_aux is not None:
            out, aux_loss, packed_router = out[0], out[1], out[2:]
            router_logits = []
            for lg in packed_router:  # [T, E] of the packed stream -> [B*S, E] rows of the batch, zeros at padding
                full = lg.new_zeros(B * S, lg.shape[-1])
                full[keep] = lg[:T_real]
                router_logits.append(full)
            router_logits = tuple(router_logits)
        if shift_labels is not None:
            loss, logits = out, None
        else:
            full = out.new_zeros(B * S, out.shape[-1])
            full[keep] = out[:T_real]
            loss, logits = None, full.view(B, S, -1)
        if router_aux is not None:
            result = MoeCausalLMOutputWithPast(loss=loss, aux_loss=aux_loss, logits=logits, router_logits=router_logits)
            return result if return_dict else result.to_tuple()
        result = CausalLMOutputWithPast(loss=loss, logits=logits)
        if not return_dict:
            return tuple(v for v in (result.loss, result.logits) if v is not None)
        return result

    def _forward_cached(self, input_ids, attention_mask, position_ids, labels, return_dict, past_key_values, inputs_embeds,
                        token_type_ids, cu_seqlens, output_router_logits: bool):
        """Padded batch with a KV cache (gpt_dolomite/base.py:173-257): `use_cache=True` without `past_key_values` runs the
        prompt through engine.prefill and returns the filled cache; with `past_key_values` (the KVCache of an earlier call),
        input_ids [B, S] are the new tokens and engine.extend appends them.  attention_mask is [B, past + S] (HuggingFace:
        the cache's get_seq_length() columns, then the new ones) or [B, S]; its last S columns decide which new tokens are
        real, and masked tokens are neither cached nor attended to.  position_ids default to the reference's
        `cumsum(mask) - 1`, the number of real tokens before each one (base.py:247-257); given ones are used for the new
        tokens.  ALiBi biases by cache position, under the rule of _alibi_pass.  Logits are [B, S, V], 0 at masked
        positions; labels give the loss of the chunk as _forward_padded computes it."""
        from ..engine import KVCache
        from .. import kernels as K

        if past_key_values is not None and not isinstance(past_key_values, KVCache):
            raise TypeError(f"past_key_values must be the KVCache an earlier call of this model returned, got "
                            f"{type(past_key_values).__name__} (tuples and transformers caches are not accepted)")
        if output_router_logits:
            raise NotImplementedError("output_router_logits is not supported together with a KV cache")
        if self.training and torch.is_grad_enabled():
            raise NotImplementedError("training through a KV cache is not implemented (there is no backward through the "
                                      "cache): call model.eval() or run under torch.no_grad()")
        if inputs_embeds is not None or token_type_ids is not None:
            raise NotImplementedError("inputs_embeds / token_type_ids are not supported on the B200 path")
        assert cu_seqlens is None, "cu_seqlens belongs to the padding-free transformer"
        eng = self.engine
        if eng.comm is not None:
            raise NotImplementedError("decoding runs on an unsharded engine (world_size 1)")
        dev = eng.device
        input_ids = torch.as_tensor(input_ids).to(dev).long()
        assert input_ids.dim() == 2, "padded batches are [batch, sequence]"
        B, S = input_ids.shape
        cache = past_key_values
        past_width = 0 if cache is None else cache.get_seq_length()
        if cache is not None and cache.lens.numel() != B:
            raise ValueError(f"past_key_values holds {cache.lens.numel()} sequences, input_ids {B}")
        if attention_mask is None:
            mask = torch.ones(B, S, dtype=torch.bool, device=dev)
        else:
            am = torch.as_tensor(attention_mask).to(dev).bool()
            if am.dim() != 2 or am.shape[0] != B or am.shape[1] not in (S, past_width + S):
                raise ValueError(f"attention_mask must be [{B}, {past_width + S}] (past and new columns) or [{B}, {S}], "
                                 f"got {tuple(am.shape)}")
            mask = am[:, am.shape[1] - S:]
        n_host = mask.sum(1).tolist()  # one host sync, as _forward_padded
        keep = mask.reshape(-1).nonzero(as_tuple=True)[0]
        ids_p = input_ids.reshape(-1)[keep].contiguous()
        pos_p = None if position_ids is None else torch.as_tensor(position_ids).to(dev).long().reshape(-1)[keep].contiguous()
        alibi = self._alibi_pass(attention_mask is not None)
        if cache is None:
            cache = KVCache(eng, B, max(n_host) + 64)
            cu = torch.zeros(B + 1, dtype=torch.int32, device=dev)
            cu[1:] = torch.tensor(n_host, dtype=torch.int32, device=dev).cumsum(0)
            if pos_p is None:
                pos_p = (mask.long().cumsum(-1) - 1).reshape(-1)[keep].contiguous()
            ids_pp, pos_pp, cu_p, _, T_real = _pad_packed_stream(ids_p, pos_p, cu, None)
            out = eng.prefill(ids_pp, pos_pp, cu_p, max(max(n_host), 1), cache, n_sequences=B, alibi=alibi)[:T_real]
        else:
            out = eng.extend(ids_p, n_host, cache, position_ids=pos_p, alibi=alibi)
        cache.seen = past_width + S
        loss = None
        if labels is not None:  # CE(logits[:, :-1], labels[:, 1:]) over the chunk's real positions, as _forward_padded
            lab = torch.as_tensor(labels).to(dev).long()
            nxt = torch.full_like(lab, -100)
            nxt[:, :-1] = lab[:, 1:]
            nxt_valid = torch.zeros_like(mask)
            nxt_valid[:, :-1] = mask[:, 1:]
            nxt = torch.where(nxt_valid & mask, nxt, torch.full_like(nxt, -100))
            loss = K.cross_entropy_fwd_bwd(out, nxt.reshape(-1)[keep].contiguous(), ignore_index=-100,
                                           dlogits=torch.empty_like(out))[0].reshape(())
        full = out.new_zeros(B * S, out.shape[-1])
        full[keep] = out
        result = CausalLMOutputWithPast(loss=loss, logits=full.view(B, S, -1), past_key_values=cache)
        return result if return_dict else result.to_tuple()

    # ---- pretraining entry: labels already aligned with positions (model_wrapper/pretraining.py:104-127) ----
    def train(self, mode: bool = True):
        self.engine.training = bool(mode)  # dropout > 0 is only rejected in training mode (engine.forward)
        return super().train(mode)

    def generate(self, input_ids=None, attention_mask=None, **generate_kwargs) -> torch.Tensor:
        """decoder-only `generate` (model_wrapper/base.py:127): prompt + new tokens; see hf_models/generation.py"""
        from .generation import generate

        return generate(self, input_ids, attention_mask, **generate_kwargs)

    def forward_pretraining_loss(self, input_ids, position_ids, cu_seqlens, max_seqlen: int, labels, alibi: bool = False):
        return _EngineFunction.apply(self._anchor, self, input_ids, position_ids, cu_seqlens, int(max_seqlen), labels, -100,
                                     torch.is_grad_enabled(), alibi)

    # ------------------------------------------------------------------------------------------
    # state dict / (de)serialisation with the reference's names
    # ------------------------------------------------------------------------------------------
    def state_dict(self, *args, **kwargs):
        return self.engine.state_dict()

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        self.engine.load_state_dict(state_dict, strict=strict)

    def named_reference_parameters(self):
        return self.engine.state_dict().items()

    def get_input_embeddings(self):
        return self.engine.units[0].views["transformer.wte.weight"]

    def save_pretrained(self, path: str, safe_serialization: bool = True) -> None:
        from safetensors.torch import save_file

        os.makedirs(path, exist_ok=True)
        self.config.save_pretrained(path)
        sd = {k: v.contiguous().cpu() for k, v in self.engine.state_dict().items()}
        save_file(sd, os.path.join(path, "model.safetensors"), metadata={"format": "pt"})

    @classmethod
    def from_pretrained(cls, path: str, **kwargs):
        from ..utils.safetensors import SafeTensorsWeightsManager

        with open(os.path.join(path, "config.json")) as f:
            d = json.load(f)
        config = config_class_for(d["model_type"]).from_dict(d)
        sd = SafeTensorsWeightsManager(path).state_dict()
        resize_vocab_to = kwargs.pop("resize_vocab_to", None)
        if resize_vocab_to is not None and int(resize_vocab_to) != config.vocab_size:
            # resize_token_embeddings on the full host tensors, before the model (and so its root unit) is sharded
            from .utils import resize_vocab_state

            sd = resize_vocab_state({k: v.float() if k in ("transformer.wte.weight", "lm_head.weight") else v
                                     for k, v in sd.items()}, int(resize_vocab_to))
            config.vocab_size = int(resize_vocab_to)
        model = cls(config, seed=None, **kwargs)
        model.load_state_dict(sd)
        return model

    def extra_repr(self) -> str:
        return (
            f"{type(self).__name__}(PaddingFreeAttention[wgmma], RMSNorm[cuda], RoPE[cuda], "
            f"{'ScatterMoE[wgmma grouped gemm]' if self.engine.is_moe else 'MLP[wgmma gemm]'}, "
            f"params={self.engine.num_parameters():,})"
        )


class GPTDolomiteForCausalLM(DolomitePreTrainedModel):
    config_class = GPTDolomiteConfig

    def __init__(self, config: GPTDolomiteConfig, **kwargs) -> None:
        assert config.model_type == "gpt_dolomite"
        super().__init__(config, **kwargs)


class MoEDolomiteForCausalLM(DolomitePreTrainedModel):
    config_class = MoEDolomiteConfig
    _no_split_modules = ["SparseMoEBlock"]

    def __init__(self, config: MoEDolomiteConfig, **kwargs) -> None:
        assert config.model_type == "moe_dolomite"
        super().__init__(config, **kwargs)


_MODEL_CLASSES = {"gpt_dolomite": GPTDolomiteForCausalLM, "moe_dolomite": MoEDolomiteForCausalLM}


class AutoModelForCausalLM:
    """`AutoModelForCausalLM.from_config / from_pretrained` dispatch of the reference (hf_models/register_hf.py:24-44)"""

    @staticmethod
    def from_config(config: CommonConfig, **kwargs):
        return _MODEL_CLASSES[config.model_type](config, **kwargs)

    @staticmethod
    def from_pretrained(path: str, **kwargs):
        with open(os.path.join(path, "config.json")) as f:
            mt = json.load(f)["model_type"]
        return _MODEL_CLASSES[mt].from_pretrained(path, **kwargs)
