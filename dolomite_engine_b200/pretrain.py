"""`python -m dolomite_engine_b200.pretrain --config <yaml>` -- the reference's pretraining entry point
(pretrain.py:60-371) for the data-parallel hot path: args -> process group -> model wrapper -> sharded wrap ->
optimizer / scheduler -> train loop over `train_step`.

The loop consumes any iterator of `{"text": LongTensor[mbs, seq+1]}` batches -- exactly what `GPTDataset` emits
(gpt_dataset.py:83-98).  `class_name: MegatronDataset` reads Megatron .bin/.idx token stores through `data/` (SURVEY.md
section 8f rank 2); `class_name: SyntheticPackedDataset` fabricates batches with the seeds of SURVEY section 8d.
"""

from __future__ import annotations

from contextlib import nullcontext

import os
import time

import torch
import torch.distributed as dist

from .arguments import TrainingArgs, get_args
from .distributed import wrap_model_for_distributed_training
from .model_wrapper import get_model
from .optimization import get_optimizer, get_scheduler
from .train_utils import billion_tokens_per_day, get_model_tflops, get_torch_profiler, train_step


class SyntheticPackedDataset:
    """batch b = randint(0, V, (mbs, S+1), manual_seed(1234 + rank + 1000003 * b)), optionally with EOS injected at seeded
    log-uniform positions (ragged packing, SURVEY.md section 8d).  One generator per batch index makes the feed resumable
    in O(1): `state_dict()` / `load_state_dict()` carry the number of batches drawn (`consumed_samples` / micro batch)."""

    def __init__(self, vocab_size: int, micro_batch_size: int, sequence_length: int, rank: int = 0, eos_token_id: int | None = None,
                 ragged: bool = False, pin: bool = True):
        self.V, self.mbs, self.S = vocab_size, micro_batch_size, sequence_length
        self.rank = rank
        self.index = 0  # batches drawn so far
        self.eos = eos_token_id
        self.ragged = ragged
        self.pin = pin and torch.cuda.is_available()

    def __iter__(self):
        return self

    def state_dict(self) -> dict:
        return {"consumed_samples": self.index * self.mbs, "batches": self.index}

    def load_state_dict(self, state: dict) -> None:
        self.index = int(state["batches"]) if "batches" in state else int(state.get("consumed_samples", 0)) // self.mbs

    def __next__(self) -> dict:
        self.gen = torch.Generator().manual_seed(1234 + self.rank + 1000003 * self.index)
        self.index += 1
        t = torch.randint(0, self.V, (self.mbs, self.S + 1), generator=self.gen, dtype=torch.int64)
        if self.ragged and self.eos is not None:
            t[t == self.eos] = (self.eos + 1) % self.V
            for r in range(self.mbs):
                pos = 0
                while True:
                    u = torch.rand(1, generator=self.gen).item()
                    step = int(64 * (self.S / 64) ** u)  # log-uniform in [64, S]
                    pos += step
                    if pos >= self.S:
                        break
                    t[r, pos] = self.eos
        if self.pin:
            t = t.pin_memory()
        return {"text": t}


def init_distributed() -> tuple[int, int, int]:
    """utils/__init__.py:28-58 / utils/parallel.py:46-79 (DP group only)"""
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    if world > 1 and not dist.is_initialized():
        from .distributed import configure_comm_ctas

        configure_comm_ctas()
        dist.init_process_group(backend="nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    return rank, world, local


def build(args: TrainingArgs):
    rank, world, local = init_distributed()
    torch.manual_seed(args.random_args.seed)
    device = torch.device("cuda", local)
    # HSDP (zero_topology): the engine shards over `data_parallel_sharding_world_size` consecutive ranks; the data feed and
    # the loss average keep using the global (rank, world)
    from .distributed import shard_world_and_rank

    shard_world, shard_rank = shard_world_and_rank(args, world, rank)
    wrapper = get_model(args, device=device, world_size=shard_world, rank=shard_rank)
    model = wrap_model_for_distributed_training(args, wrapper)
    from .fp8 import setup_training

    model.forward_context = setup_training(args, wrapper)
    optimizer = get_optimizer(args.optimizer_args.class_name, args.optimizer_args.class_args, model,
                              args.optimizer_args.params_group_method)
    ls = args.lr_scheduler_args
    scheduler = get_scheduler(optimizer, ls.num_warmup_steps, ls.num_constant_steps, ls.num_decay_steps,
                              args.training_parameters.num_training_steps, ls.lr_decay_style, ls.lr_decay_factor,
                              ls.extra_lr_scheduler_args)
    return model, optimizer, scheduler, (rank, world, local)


def _fim_spec(args: TrainingArgs, tokenizer=None):
    """class_args.fim_rate / fim_spm_rate (data/megatron/__init__.py:87-88); needs the tokenizer's <fim_*> ids"""
    ca = args.datasets[0].class_args
    rate = float(ca.get("fim_rate", 0) or 0)
    if rate == 0:
        return None
    from .data import FIMSpec, HFTokenizerCodec

    if tokenizer is None:
        from transformers import AutoTokenizer

        name = args.tokenizer_args.tokenizer_name or args.model_args.model_name
        if name is None:
            raise ValueError("fim_rate != 0 needs tokenizer_args.tokenizer_name (a tokenizer holding the <fim_*> tokens)")
        tokenizer = AutoTokenizer.from_pretrained(name)
    codec = tokenizer if hasattr(tokenizer, "detokenize") else HFTokenizerCodec(tokenizer)
    return FIMSpec.from_tokenizer(codec, rate, float(ca.get("fim_spm_rate", 0.5)))


def _blend_per_split(class_args: dict):
    """option 3 of data/megatron/__init__.py:78-84, 93-101: `train_data_path` / `val_data_path` / `test_data_path` (each one prefix or
    [w1, prefix1, w2, prefix2, ...]) instead of `data_path` + `split`"""
    per_split = [class_args.get("train_data_path"), class_args.get("val_data_path"), class_args.get("test_data_path")]
    if not any(per_split):
        return None
    if class_args.get("data_path") is not None:
        raise ValueError("MegatronDataset: data_path and train_data_path / val_data_path / test_data_path are incompatible")
    return per_split


def _data_sources(class_args: dict) -> tuple:
    """(data_path, split) of options 1 / 2; (None, None) when the splits name their own stores"""
    if _blend_per_split(class_args) is not None:
        return None, None
    if class_args.get("data_path") is None:
        raise ValueError("MegatronDataset: class_args needs data_path (+ split) or train_data_path [/ val_data_path / test_data_path]")
    return class_args["data_path"], class_args.get("split", "100,0,0")


def _index_cache_args(class_args: dict) -> dict:
    """`data_cache_path` / `node_uses_local_storage` of the reference's MegatronDataset class_args (data/megatron/__init__.py:85-89).
    With a cache path the document / sample / shuffle indices are stored there under the reference's file names (rank 0 builds, the
    others memory-map the same files); without one, indices the reference stored in its default place next to the data
    (`<prefix>/cache/GPTDataset_indices`) are used when they exist and nothing is written (the reference would write there)."""
    if class_args.get("data_cache_path"):
        return dict(data_cache_path=class_args["data_cache_path"], cache="build",
                    node_uses_local_storage=bool(class_args.get("node_uses_local_storage", False)))
    return dict(cache="load")


def make_megatron_dataloader(args: TrainingArgs, rank: int, world: int, consumed_samples: int = 0, tokenizer=None):
    """get_megatron_gpt_dataloaders (data/megatron/__init__.py:18-213), train split: Megatron .bin/.idx stores named by
    `class_args.data_path` (one prefix or [w1, prefix1, w2, prefix2, ...]) + `split`, cut into S+1-token samples, global
    batches of mbs * world consecutive samples with rank r taking rows [r*mbs, (r+1)*mbs); resumes at `consumed_samples`."""
    from .data import MegatronBatchSampler, PackedBatchLoader, build_gpt_datasets, get_train_val_test_samples

    ds, tp = args.datasets[0], args.training_parameters
    ca = ds.class_args
    sizes = get_train_val_test_samples(tp.num_training_steps, tp.micro_batch_size, tp.gradient_accumulation_steps,
                                       getattr(tp, "eval_interval", None), ca.get("eval_steps"), world)
    train, _, _ = build_gpt_datasets(*_data_sources(ca), sizes, ca["sequence_length"], ca.get("seed", args.random_args.seed),
                                     fim=_fim_spec(args, tokenizer), blend_per_split=_blend_per_split(ca), **_index_cache_args(ca))
    if train is None:
        raise ValueError("MegatronDataset: no training data (data_path with a zero train split, or no train_data_path)")
    sampler = MegatronBatchSampler(len(train), consumed_samples, tp.micro_batch_size, world, rank)
    return PackedBatchLoader(train, sampler, ca["sequence_length"])


def make_megatron_val_dataloader(args: TrainingArgs, rank: int, world: int):
    """validation split of the same stores (data/megatron/__init__.py:170-190): a fresh pass from sample 0 every evaluation"""
    from .data import MegatronBatchSampler, PackedBatchLoader, build_gpt_datasets, get_train_val_test_samples

    ds, tp = args.datasets[0], args.training_parameters
    ca = ds.class_args
    if ds.class_name != "MegatronDataset" or not ca.get("eval_steps") or not tp.eval_interval:
        return None
    sizes = get_train_val_test_samples(tp.num_training_steps, tp.micro_batch_size, tp.gradient_accumulation_steps,
                                       tp.eval_interval, ca.get("eval_steps"), world)
    _, val, _ = build_gpt_datasets(*_data_sources(ca), sizes, ca["sequence_length"], ca.get("seed", args.random_args.seed),
                                   blend_per_split=_blend_per_split(ca), **_index_cache_args(ca))
    if val is None:
        return None
    return lambda: iter(PackedBatchLoader(val, MegatronBatchSampler(len(val), 0, tp.micro_batch_size, world, rank),
                                          ca["sequence_length"]))


def evaluate(val_loader_factory, model, eval_steps: int, world: int) -> float | None:
    """pretrain.py:223-296: mean loss over `eval_steps` validation micro-batches (no activations kept), averaged over ranks"""
    if val_loader_factory is None:
        return None
    model.eval()
    it = val_loader_factory()
    total, n = None, 0
    with torch.no_grad():
        for _ in range(eval_steps):
            try:
                batch = next(it)
            except StopIteration:
                break
            loss = model(batch).detach().float()
            total = loss if total is None else total + loss
            n += 1
    model.train()
    if n == 0:
        return None
    mean = total / n
    if world > 1 and dist.is_initialized():
        dist.all_reduce(mean, op=dist.ReduceOp.AVG)
    return float(mean.item())


def make_dataloader(args: TrainingArgs, model, rank: int, world: int = 1, consumed_samples: int = 0):
    ds = args.datasets[0]
    if ds.class_name == "MegatronDataset":
        return iter(make_megatron_dataloader(args, rank, world, consumed_samples))
    if ds.class_name != "SyntheticPackedDataset":
        raise NotImplementedError(
            f"dataset class {ds.class_name}: only MegatronDataset (.bin/.idx token stores) and SyntheticPackedDataset feed "
            "the pretraining hot path; pass any other iterator of {'text': LongTensor[mbs, seq+1]} batches to train()"
        )
    cfg = model.config
    feed = SyntheticPackedDataset(cfg.vocab_size, args.training_parameters.micro_batch_size,
                                  ds.class_args["sequence_length"], rank=rank, eos_token_id=cfg.eos_token_id,
                                  ragged=bool(ds.class_args.get("ragged", False)))
    # resume: skip the micro-batches this rank already drew (consumed_samples counts sequences over all ranks)
    feed.load_state_dict({"batches": consumed_samples // (args.training_parameters.micro_batch_size * max(world, 1))})
    return feed


def train(args: TrainingArgs, model, optimizer, scheduler, dataloader, rank: int, world: int, starting_iteration: int = 0) -> list[float]:
    """pretrain.py:60-205: the step loop; checkpoints every `save_args.save_interval` steps in the reference's layout"""
    from .checkpointing import save_checkpoint

    tp = args.training_parameters
    seq = args.datasets[0].class_args["sequence_length"]
    # recomputed blocks count as extra forward FLOPs, like the reference (train_utils.py:225-230)
    dargs = args.distributed_args
    fraction = 0.0
    if dargs.gradient_checkpointing_method is not None:
        every = int((dargs.gradient_checkpointing_args or {}).get("checkpoint_every", 1))
        fraction = (model.config.n_layer // every) / model.config.n_layer
    tflop_per_step = get_model_tflops(model.config, tp.micro_batch_size * tp.gradient_accumulation_steps, seq,
                                      checkpointed_fraction=fraction)
    samples_per_step = tp.micro_batch_size * tp.gradient_accumulation_steps * world
    save_args = getattr(args, "save_args", None)
    val_factory = make_megatron_val_dataloader(args, rank, world) if tp.eval_during_training else None
    eval_steps = int(args.datasets[0].class_args.get("eval_steps") or 0)

    def run_eval(at_step: int) -> None:
        v = evaluate(val_factory, model, eval_steps, world)
        if v is not None and rank == 0:
            print(f"step {at_step}: val loss {v:.4f}", flush=True)

    if val_factory is not None:
        run_eval(starting_iteration)  # pretrain.py:121-122: evaluate before the first step
    losses = []
    profiler = get_torch_profiler(args.logging_args.torch_profiler_trace_path, rank)  # pretrain.py:138-141
    if profiler is not None:
        profiler.__enter__()
    t0 = time.perf_counter()
    for step in range(starting_iteration + 1, tp.num_training_steps + 1):
        loss, grad_norm = train_step(model, optimizer, scheduler, train_dataloader=dataloader,
                                     gradient_accumulation_steps=tp.gradient_accumulation_steps,
                                     gradient_clipping=tp.gradient_clipping,
                                     forward_context=getattr(model, "forward_context", nullcontext))
        losses.append(loss)
        if profiler is not None:
            profiler.step()
        if rank == 0 and step % args.logging_args.log_interval == 0:
            dt = (time.perf_counter() - t0) / (step - starting_iteration)
            print(f"step {step}: loss {loss:.4f} grad_norm {grad_norm:.4f} lr {scheduler.get_last_lr()[0]:.3e} "
                  f"step_time {dt:.3f}s FLOPS {tflop_per_step / dt:.1f} TFLOP/s/GPU "
                  f"throughput {billion_tokens_per_day(samples_per_step * seq, dt):.2f} B tokens/day", flush=True)
        if val_factory is not None and step % tp.eval_interval == 0:
            run_eval(step)
        if save_args is not None and (step % save_args.save_interval == 0 or step == tp.num_training_steps):
            save_checkpoint(args, model, optimizer, scheduler, None, None, step,
                            metadata={"consumed_samples": step * samples_per_step})
    if profiler is not None:
        profiler.__exit__(None, None, None)
    return losses


def main() -> None:
    args = get_args()
    model, optimizer, scheduler, (rank, world, _) = build(args)
    # resume (pretrain.py:329-343): parameters, Adam moments, scheduler, RNG; the data feed restarts at consumed_samples
    from .checkpointing import load_checkpoint_for_training

    starting_iteration, consumed_samples = 0, 0
    loaded = load_checkpoint_for_training(args, model, optimizer, scheduler, None)
    if loaded is not None:
        starting_iteration, metadata, _ = loaded
        consumed_samples = int((metadata or {}).get("consumed_samples", 0))
    dl = make_dataloader(args, model, rank, world, consumed_samples)
    train(args, model, optimizer, scheduler, dl, rank, world, starting_iteration)
    if dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
