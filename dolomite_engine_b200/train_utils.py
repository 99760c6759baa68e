"""train_step of the reference (train_utils.py:18-116) on the B200 runtime, plus its FLOP model (:197-236).

Same control flow: zero_grad, (grad_accum-1) micro-steps under no_sync, last micro-step with gradient sync
(reduce-scatter), clip, optimizer + scheduler step, loss /= grad_accum, loss AVG all-reduce.  Differences, all
for throughput: the loss / grad-norm stay on the device (`return_tensors=True`) so that the host never stalls the
launch queue -- `.item()` is only paid when the caller asks for floats, like the reference does every step."""

from __future__ import annotations

from contextlib import nullcontext

import torch
import torch.distributed as dist


def get_next_batch(dataloader):
    """data/utils.py:116-130"""
    if dataloader is None:
        return None
    return next(dataloader)


def train_step(model, optimizer, lr_scheduler, distributed_backend=None, train_dataloader=None,
               gradient_accumulation_steps: int = 1, gradient_clipping: float | None = 1.0, forward_context=nullcontext,
               backward_context=nullcontext, return_tensors: bool = False):
    no_sync = model.no_sync if hasattr(model, "no_sync") else nullcontext
    loss = 0
    grad_norm = None
    if hasattr(model, "zero_grad"):
        model.zero_grad()
    else:
        optimizer.zero_grad()
    with no_sync():
        for _ in range(gradient_accumulation_steps - 1):
            batch = get_next_batch(train_dataloader)
            with forward_context():
                loss_micro_step = model(batch)
            loss = loss + loss_micro_step.detach()
            with backward_context():
                loss_micro_step.backward()
    batch = get_next_batch(train_dataloader)
    with forward_context():
        loss_micro_step = model(batch)
    loss = loss + loss_micro_step.detach()
    with backward_context():
        loss_micro_step.backward()
    if gradient_clipping is not None:
        fused = type(optimizer).__name__ == "DolomiteFusedAdamW"
        grad_norm = model.clip_grad_norm_(gradient_clipping, fuse_into_optimizer=fused)
    optimizer.step()
    if hasattr(model, "mark_parameters_updated") and type(optimizer).__name__ != "DolomiteFusedAdamW":
        model.mark_parameters_updated()
    if lr_scheduler is not None:
        lr_scheduler.step()
    loss = loss / gradient_accumulation_steps
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(loss, op=dist.ReduceOp.AVG)
    if return_tensors:
        return loss, grad_norm
    loss = loss.item()
    grad_norm = 0 if grad_norm is None else grad_norm.item()
    return loss, grad_norm


def get_model_tflops(config, batch_size: int, sequence_length: int, checkpointed_fraction: float = 0.0) -> float:
    """train_utils.py:197-236 -- TFLOP per step of `batch_size` sequences (full SxS attention, no causal discount)"""
    b, s, h, f = batch_size, sequence_length, config.n_embd, config.n_inner
    n, k, l, v = config.n_head, config.num_key_value_heads, config.n_layer, config.vocab_size
    mlp_flops = 4 * b * s * h * f
    if config.activation_function.endswith("glu"):
        mlp_flops += 2 * b * s * h * f
    attention_flops = 4 * b * s * h * (h * (1 + k / n) + s)
    forward_flops = attention_flops + mlp_flops
    backward_flops = (2 + checkpointed_fraction) * forward_flops
    model_flops = l * (forward_flops + backward_flops)
    model_flops += 6 * b * s * h * v
    return model_flops / 10**12


def get_torch_profiler(trace_path: str | None, rank: int = 0, wait: int = 5, warmup: int = 5):
    """`logging_args.torch_profiler_trace_path` (train_utils.py:182-194): one traced step on rank 0 after `wait + warmup`
    steps, written as a TensorBoard trace; other ranks never reach their window.  This is the reference's timeline view of
    the loop."""
    if trace_path is None:
        return None
    acts = [torch.profiler.ProfilerActivity.CPU]
    if torch.cuda.is_available():
        acts.append(torch.profiler.ProfilerActivity.CUDA)
    return torch.profiler.profile(
        activities=acts,
        schedule=torch.profiler.schedule(wait=wait if rank == 0 else 150000, warmup=warmup, active=1, repeat=1),
        on_trace_ready=torch.profiler.tensorboard_trace_handler(trace_path), record_shapes=True)


def billion_tokens_per_day(tokens_per_step: int, step_seconds: float) -> float:
    """`throughput (B tokens/day)` of track_train_metrics (train_utils.py:119-179)"""
    return tokens_per_step * 86400.0 / step_seconds / 1e9
