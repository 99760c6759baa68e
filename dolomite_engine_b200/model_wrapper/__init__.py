"""Model wrappers of the reference (model_wrapper/{base,pretraining,finetuning}.py) for the B200 path.

`ModelWrapperForPretraining.forward(batch: {"text": LongTensor[mbs, seq+1]}) -> scalar loss` keeps the reference
contract (model_wrapper/pretraining.py:89-127) but does the integer bookkeeping on the host, ships it with ONE
asynchronous H2D copy from pinned memory and never synchronises the device.
"""

from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from ..hf_models import AutoModelForCausalLM, config_for_model
from ..hf_models.config import CommonConfig
from ..hf_models.utils import prepare_pretraining_inputs_host


class ModelWrapper(nn.Module):
    """model_wrapper/base.py:13-266 (the parts the training path uses)"""

    def __init__(
        self,
        mode=None,
        model_name: str | None = None,
        pretrained_config: dict | None = None,
        model_class=None,
        dtype: torch.dtype = torch.bfloat16,
        efficient_initialization: bool = False,
        attention_implementation: str = "flash_attention_2",
        use_padding_free_transformer: bool = True,
        tensor_parallel_word_embeddings: bool = False,
        sequence_parallel: bool = False,
        distributed_backend=None,
        random_seed: int = 42,
        neft_alpha: float | None = None,
        trust_remote_code: bool = False,
        tokenizer_name: str | None = None,
        additional_special_tokens: list[str] | None = None,
        moe_implementation: str | None = None,
        normalization_implementation: str | None = None,
        device=None,
        world_size: int = 1,
        rank: int = 0,
        init_on_device: bool = False,
    ) -> None:
        super().__init__()
        self.mode = mode
        self.model_name = model_name
        self.pretrained_config = pretrained_config
        self.dtype = dtype
        self.efficient_initialization = efficient_initialization
        self.attention_implementation = str(getattr(attention_implementation, "value", attention_implementation))
        self.use_padding_free_transformer = use_padding_free_transformer
        self.tokenizer_name = model_name if tokenizer_name is None else tokenizer_name
        self.random_seed = random_seed
        if tensor_parallel_word_embeddings or sequence_parallel:
            raise NotImplementedError("tensor / sequence parallelism is out of scope of the data-parallel B200 path")
        if dtype not in (torch.bfloat16, "bf16"):
            raise NotImplementedError("the B200 path computes in bf16 with fp32 masters (mixed_precision_args.dtype: bf16)")
        self._setup_config()
        if self.use_padding_free_transformer:
            # model_wrapper/base.py:94-101
            assert self.attention_implementation == "flash_attention_2", "padding free transformer only works with flash attention"
        self._setup_tokenizer(required=bool(additional_special_tokens))
        kwargs = dict(attn_implementation=self.attention_implementation,
                      use_padding_free_transformer=self.use_padding_free_transformer,
                      device=device, world_size=world_size, rank=rank, seed=random_seed, init_on_device=init_on_device)
        if moe_implementation is not None:
            kwargs["moe_implementation"] = moe_implementation
        if normalization_implementation is not None:
            kwargs["normalization_implementation"] = normalization_implementation
        if additional_special_tokens:
            # model_wrapper/base.py:102-108: the model follows len(tokenizer) only when adding the tokens changed it -- which
            # also shrinks a model whose vocab_size was padded above the tokenizer's length
            original_vocab_size = len(self.tokenizer)
            self.tokenizer.add_special_tokens({"additional_special_tokens": list(additional_special_tokens)})
            if len(self.tokenizer) != original_vocab_size:
                kwargs["resize_vocab_to"] = len(self.tokenizer)
        if self.model_name is None:
            self.model = AutoModelForCausalLM.from_config(self.config, **kwargs)
        else:
            kwargs.pop("seed")
            self.model = AutoModelForCausalLM.from_pretrained(self.model_name, **kwargs)
        self.config.vocab_size = self.model.config.vocab_size
        # model_wrapper/base.py:97-100: NEFTune in training mode; the engine adds the noise in training passes only
        if str(getattr(mode, "value", mode)) not in ("inference", "unsharding") and neft_alpha is not None and neft_alpha > 0:
            self.model.engine.neft_alpha = float(neft_alpha)

    def _setup_config(self) -> None:
        """model_wrapper/base.py:151-163"""
        if self.model_name is None:
            cfg = dict(self.pretrained_config)
            self.config: CommonConfig = config_for_model(cfg.pop("model_type"), **cfg)
        else:
            self.config = CommonConfig.from_pretrained(self.model_name)

    def _setup_tokenizer(self, required: bool = False) -> None:
        """model_wrapper/base.py:165-169.  Tokenizers come from the HF hub in the reference; offline we only need the
        eos id, which the config carries -- unless tokens are to be added (`required`), which needs a local tokenizer."""
        self.tokenizer = None
        self.eos_token_id = self.config.eos_token_id
        if self.tokenizer_name is None and required:
            raise ValueError("additional_special_tokens needs a tokenizer: set tokenizer_args.tokenizer_name or model_args.model_name")
        if self.tokenizer_name is not None:
            try:
                from transformers import AutoTokenizer

                self.tokenizer = AutoTokenizer.from_pretrained(self.tokenizer_name)
                self.eos_token_id = self.tokenizer.eos_token_id
            except (OSError, ValueError, ImportError) as e:  # not a local directory and no hub access: keep the config's eos id
                if required:
                    raise ValueError(f"additional_special_tokens needs a tokenizer, and {self.tokenizer_name!r} could not be "
                                     f"loaded ({type(e).__name__}: {e})") from e
                import warnings

                warnings.warn(f"tokenizer {self.tokenizer_name!r} could not be loaded ({type(e).__name__}); continuing without "
                              "one (token-id batches only)")
                self.tokenizer = None

    def save_pretrained(self, save_path: str, state_dict: dict | None = None) -> None:
        """model_wrapper/base.py:138-149: tokenizer + either the live model or a given full state dict whose keys carry the
        wrapper prefix `model.`"""
        if self.tokenizer is not None:
            self.tokenizer.save_pretrained(save_path)
        if state_dict is None:
            self.model.save_pretrained(save_path)
            return
        from ..utils.safetensors import SafeTensorsWeightsManager

        bad = [k for k in state_dict if not k.startswith("model.")]
        assert not bad, f"state dict keys must start with 'model.': {bad[:3]}"
        self.config.save_pretrained(save_path)
        SafeTensorsWeightsManager.save_state_dict({k[len("model."):]: v for k, v in state_dict.items()}, save_path)

    def generate(self, batch: dict, generate_kwargs: dict) -> tuple[list[str] | list[list[int]], list[int]]:
        """model_wrapper/base.py:110-136: -> (generated text with the prompt trimmed, generated-token counts incl. eos).
        Without a tokenizer (offline) the first element holds the generated token ids instead of text."""
        out = self.model.generate(input_ids=batch["input_ids"], attention_mask=batch.get("attention_mask"),
                                  **generate_kwargs, eos_token_id=self.eos_token_id)
        generated = out[:, torch.as_tensor(batch["input_ids"]).shape[1] :]
        num_generated_tokens = ((generated != self.eos_token_id).sum(dim=-1) + 1).tolist()
        if self.tokenizer is None:
            return generated.tolist(), num_generated_tokens
        return self.tokenizer.batch_decode(generated, skip_special_tokens=True), num_generated_tokens


class ModelWrapperForPretraining(ModelWrapper):
    """model_wrapper/pretraining.py:16-236"""

    def __init__(self, *args, micro_batch_size: int, sequence_length: int, reset_attention_mask: bool = False,
                 reset_position_ids: bool = False, **kwargs) -> None:
        self.micro_batch_size = micro_batch_size
        self.sequence_length = sequence_length
        self.reset_attention_mask = reset_attention_mask
        self.reset_position_ids = reset_position_ids
        super().__init__(*args, **kwargs)
        if not self.use_padding_free_transformer:
            # padded pretraining (model_wrapper/pretraining.py:129-194 without cu_seqlens): every row of the batch is one
            # document of `sequence_length` tokens and no attention mask is passed -- which is the same packed stream as
            # the padding-free path without reset_attention_mask, so both stage and run it the same way
            assert not self.reset_attention_mask, (
                "currently reset_attention_mask is only implemented for padding free transformer")
            assert not self.reset_position_ids, "currently reset_position_ids is only implemented for padding free transformer"
        if self.reset_position_ids:
            assert self.reset_attention_mask, "reset_attention_mask should be specified with reset_position_ids"
        self.model.assume_unit_loss_grad = True  # train_step calls loss.backward() on the raw loss
        dev = self.model.engine.device
        T = micro_batch_size * sequence_length
        # one pinned staging buffer + one device buffer: tokens ids/labels/position ids/cu_seqlens travel in one copy
        self._n_words = 3 * T + (T + 2) // 2 + 2  # int64 words: ids, labels, pos, cu (int32 packed)
        self._host = torch.empty(self._n_words, dtype=torch.int64).pin_memory() if dev.type == "cuda" else torch.empty(self._n_words, dtype=torch.int64)
        self._dev = torch.empty(self._n_words, dtype=torch.int64, device=dev)
        self._host_np = self._host.numpy()
        self._copy_done: torch.cuda.Event | None = None
        self.h2d_bytes_per_step = 0

    def _stage(self, tokens: torch.Tensor):
        """host bookkeeping (bit-exact with model_wrapper/pretraining.py:129-194) + one async H2D copy"""
        tk = tokens.numpy() if tokens.device.type == "cpu" else tokens.cpu().numpy()
        b = prepare_pretraining_inputs_host(tk, self.eos_token_id, self.reset_attention_mask, self.reset_position_ids)
        T = b["input_ids"].shape[0]
        nb = b["cu_seqlens"].shape[0]
        if self._copy_done is not None:
            self._copy_done.synchronize()  # previous step's copy has left the pinned buffer (normally long done)
        h = self._host_np
        h[0:T] = b["input_ids"]
        h[T : 2 * T] = b["labels"]
        h[2 * T : 3 * T] = b["position_ids"]
        cu_words = (nb + 1) // 2
        assert 3 * T + cu_words <= self._n_words, "more documents than the staging buffer was sized for"
        h[3 * T : 3 * T + cu_words].view(np.int32)[:nb] = b["cu_seqlens"]
        n_used = 3 * T + cu_words
        self._dev[:n_used].copy_(self._host[:n_used], non_blocking=True)
        self._copy_done = torch.cuda.Event()
        self._copy_done.record()
        self.h2d_bytes_per_step = n_used * 8
        d = self._dev
        ids, labels, pos = d[0:T], d[T : 2 * T], d[2 * T : 3 * T]
        cu = d[3 * T : 3 * T + cu_words].view(torch.int32)[:nb]
        return ids, labels, pos, cu, b["max_seqlen"]

    def forward(self, batch: dict) -> torch.Tensor:
        tokens: torch.Tensor = batch["text"]
        assert tokens.dtype == torch.int64 and tokens.dim() == 2
        assert tokens.shape[0] * (tokens.shape[1] - 1) <= self.micro_batch_size * self.sequence_length
        ids, labels, pos, cu, max_seqlen = self._stage(tokens)
        # padded batches pass no attention mask: eager alibi models add the bias, sdpa ones run as NoPE
        alibi = not self.use_padding_free_transformer and self.model._alibi_pass(has_attention_mask=False)
        return self.model.forward_pretraining_loss(ids, pos, cu, max_seqlen, labels, alibi=alibi)


class ModelWrapperForFinetuning(ModelWrapper):
    """model_wrapper/finetuning.py:10-99.  Padding-free collate (data/utils.py:8-92): batch = {"input_ids":
    list[list[int]], "labels": list[list[int]]}; padded collate: [B, S] tensors + "attention_mask".  The loss is computed
    inside the model (gpt_dolomite/main.py:179-202)."""

    def __init__(self, *args, **kwargs) -> None:
        super().__init__(*args, **kwargs)
        self.model.assume_unit_loss_grad = True  # train_step calls loss.backward() on the raw loss (train_utils.py:61-90)

    def forward(self, batch: dict) -> torch.Tensor:
        if "attention_mask" in batch and batch["attention_mask"] is not None:
            # padded collate (use_padding_free_transformer: false, data/utils.py:8-92): [B, S] tensors + attention_mask
            out = self.model(input_ids=batch["input_ids"], attention_mask=batch["attention_mask"], labels=batch["labels"],
                             position_ids=batch.get("position_ids"))
        else:
            out = self.model(input_ids=batch["input_ids"], labels=batch["labels"], position_ids=batch.get("position_ids"))
        return out.loss


def get_model(args, mode=None, device=None, world_size: int = 1, rank: int = 0) -> ModelWrapper:
    """model_wrapper/__init__.py:20-52"""
    margs = args.model_args
    kwargs = dict(
        mode=mode,
        model_name=margs.model_name,
        pretrained_config=margs.pretrained_config,
        model_class=margs.model_class,
        dtype=torch.bfloat16,
        efficient_initialization=margs.efficient_initialization,
        attention_implementation=margs.attention_implementation or "flash_attention_2",
        use_padding_free_transformer=margs.use_padding_free_transformer,
        random_seed=args.random_args.seed,
        neft_alpha=args.research_args.neft_alpha,
        tokenizer_name=args.tokenizer_args.tokenizer_name,
        additional_special_tokens=args.tokenizer_args.additional_special_tokens,
        moe_implementation=getattr(margs, "moe_implementation", None),
        normalization_implementation=getattr(margs, "normalization_implementation", None),
        device=device,
        world_size=world_size,
        rank=rank,
    )
    tuning = str(getattr(args.tuning_args.tuning_method, "value", args.tuning_args.tuning_method))
    if tuning == "pretraining":
        seq_len = args.datasets[0].class_args.get("sequence_length")
        return ModelWrapperForPretraining(
            **kwargs,
            micro_batch_size=args.training_parameters.micro_batch_size,
            sequence_length=seq_len,
            reset_attention_mask=margs.reset_attention_mask,
            reset_position_ids=margs.reset_position_ids,
        )
    if tuning == "full_finetuning":
        return ModelWrapperForFinetuning(**kwargs)
    raise NotImplementedError(f"tuning_method={tuning}: PEFT is out of scope of the B200 hot path")
