"""`python -m dolomite_engine_b200.finetune --config <yaml>` -- the reference's finetune.py for decoder-only full
finetuning (tuning_method: full_finetuning): JSON-lines {"input", "output"} examples -> collate (padding-free lists or
left-padded tensors) -> `ModelWrapperForFinetuning` -> the same `train_step`, sharded wrap, optimizer, scheduler and
checkpoints as pretraining.

datasets:
  - class_name: JSONLinesDataset            # data/instruction_tuning: one JSON object per line
    data_name: my_sft_data
    class_args: {data_path: /path/to/dir_or_file}
    input_format: "Q: __input__\\nA:"         # optional wrappers (data/base.py:56-82)
    output_format: " __output__"
    max_input_tokens: 4096
    max_output_tokens: 1024
The tokenizer comes from `tokenizer_args.tokenizer_name` (or `model_args.model_name`) through transformers.AutoTokenizer
(local directory; there is no hub access here).
"""

from __future__ import annotations

from contextlib import nullcontext

import time

import torch.distributed as dist

from .arguments import TrainingArgs, get_args
from .checkpointing import load_checkpoint_for_training, save_checkpoint
from .data.finetuning import JSONLinesSFTDataset, batches
from .distributed import wrap_model_for_distributed_training
from .model_wrapper import get_model
from .optimization import get_optimizer, get_scheduler
from .pretrain import init_distributed
from .train_utils import train_step


def make_sft_dataloader(args: TrainingArgs, tokenize, eos_token_id: int, rank: int, world: int):
    ds_args = args.datasets[0]
    if ds_args.class_name not in ("JSONLinesDataset", "SlimOrcaDataset", "AlpacaDataset") and "data_path" not in ds_args.class_args:
        raise NotImplementedError(f"dataset class {ds_args.class_name}: the B200 finetuning feed reads JSON-lines files "
                                  "(class_name: JSONLinesDataset, class_args.data_path)")
    ds = JSONLinesSFTDataset(ds_args.class_args["data_path"], tokenize, eos_token_id, ds_args.input_format,
                             ds_args.output_format, ds_args.max_input_tokens, ds_args.max_output_tokens, split="train")
    tp = args.training_parameters
    return batches(ds, tp.micro_batch_size, eos_token_id, bool(args.model_args.use_padding_free_transformer), rank=rank,
                   world_size=world, seed=args.random_args.seed, loss_mask=str(getattr(tp.loss_mask, "value", tp.loss_mask)))


def make_sft_val_batches(args: TrainingArgs, tokenize, eos_token_id: int, rank: int, world: int):
    """-> factory of a one-pass, rank-sharded iterator over the validation split, or None when there is none"""
    ds_args, tp = args.datasets[0], args.training_parameters
    if not tp.eval_during_training or "data_path" not in ds_args.class_args:
        return None
    ds = JSONLinesSFTDataset(ds_args.class_args["data_path"], tokenize, eos_token_id, ds_args.input_format,
                             ds_args.output_format, ds_args.max_input_tokens, ds_args.max_output_tokens, split="val")
    if len(ds) < tp.micro_batch_size * world:
        return None
    return lambda: batches(ds, tp.micro_batch_size, eos_token_id, bool(args.model_args.use_padding_free_transformer), rank=rank,
                           world_size=world, seed=args.random_args.seed,
                           loss_mask=str(getattr(tp.loss_mask, "value", tp.loss_mask)), infinite=False)


def evaluate(val_batches, model) -> float | None:
    """finetune.py:156-219: mean loss over one pass of the validation batches (no activations kept), averaged over ranks"""
    if val_batches is None:
        return None
    import torch

    model.eval()
    total, n = None, 0
    with torch.no_grad():
        for batch in val_batches():
            loss = model(batch).detach().float()
            total = loss if total is None else total + loss
            n += 1
    model.train()
    if n == 0:
        return None
    mean = total / n
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(mean, op=dist.ReduceOp.AVG)
    return float(mean.item())


def train(args: TrainingArgs, model, optimizer, scheduler, dataloader, rank: int, starting_iteration: int = 0,
          val_batches=None) -> list[float]:
    tp = args.training_parameters
    losses, t0 = [], time.perf_counter()

    def run_eval(at_step: int) -> None:
        v = evaluate(val_batches, model)
        if v is not None and rank == 0:
            print(f"step {at_step}: val loss {v:.4f}", flush=True)

    if val_batches is not None:
        run_eval(starting_iteration)  # finetune.py:98-99: evaluate before the first step
    for step in range(starting_iteration + 1, tp.num_training_steps + 1):
        loss, grad_norm = train_step(model, optimizer, scheduler, train_dataloader=dataloader,
                                     gradient_accumulation_steps=tp.gradient_accumulation_steps,
                                     gradient_clipping=tp.gradient_clipping,
                                     forward_context=getattr(model, "forward_context", nullcontext))
        losses.append(loss)
        if rank == 0 and step % args.logging_args.log_interval == 0:
            dt = (time.perf_counter() - t0) / (step - starting_iteration)
            print(f"step {step}: loss {loss:.4f} grad_norm {grad_norm:.4f} lr {scheduler.get_last_lr()[0]:.3e} "
                  f"step_time {dt:.3f}s", flush=True)
        if val_batches is not None and tp.eval_interval and step % tp.eval_interval == 0:
            run_eval(step)
        if args.save_args is not None and (step % args.save_args.save_interval == 0 or step == tp.num_training_steps):
            save_checkpoint(args, model, optimizer, scheduler, dataloader, None, step, metadata={"iteration": step})
    return losses


def main() -> None:
    args = get_args()
    rank, world, local = init_distributed()
    import torch

    torch.manual_seed(args.random_args.seed)
    from .distributed import shard_world_and_rank

    shard_world, shard_rank = shard_world_and_rank(args, world, rank)
    wrapper = get_model(args, device=torch.device("cuda", local), world_size=shard_world, rank=shard_rank)
    if wrapper.tokenizer is None:
        raise ValueError("finetuning needs a tokenizer: set tokenizer_args.tokenizer_name (or model_args.model_name) to a local directory")
    model = wrap_model_for_distributed_training(args, wrapper)
    from .fp8 import setup_training

    model.forward_context = setup_training(args, wrapper)
    optimizer = get_optimizer(args.optimizer_args.class_name, args.optimizer_args.class_args, model,
                              args.optimizer_args.params_group_method)
    ls = args.lr_scheduler_args
    scheduler = get_scheduler(optimizer, ls.num_warmup_steps, ls.num_constant_steps, ls.num_decay_steps,
                              args.training_parameters.num_training_steps, ls.lr_decay_style, ls.lr_decay_factor,
                              ls.extra_lr_scheduler_args)
    tokenize = lambda text: wrapper.tokenizer(text, add_special_tokens=False)["input_ids"]  # noqa: E731
    dl = make_sft_dataloader(args, tokenize, wrapper.eos_token_id, rank, world)
    start = 0
    loaded = load_checkpoint_for_training(args, model, optimizer, scheduler, dl)  # restores the feed position as well
    if loaded is not None:
        start = loaded[0]
    val = make_sft_val_batches(args, tokenize, wrapper.eos_token_id, rank, world)
    train(args, model, optimizer, scheduler, dl, rank, start, val_batches=val)
    if dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
