"""Training checkpoints in the reference's on-disk layout (SURVEY.md section 8f rank 3; checkpointing.py:50-263, FSDP-1
`FULL_STATE_DICT` branch), so a run started with this engine can be resumed / unsharded by the reference tooling and
vice versa:

    <save_path>/latest_checkpointed_iteration.json          {"latest_checkpointed_iteration": N}
    <save_path>/global_step<N>/model.pt                     full fp32 state dict, reference names under "model."
    <save_path>/global_step<N>/optimizer.pt                 {"state": {fqn: {step, exp_avg, exp_avg_sq}}, "param_groups": [...]}
    <save_path>/global_step<N>/lr_scheduler.pt              LambdaLR.state_dict()
    <save_path>/global_step<N>/rng_state/rng_state-<rank>.pt
    <save_path>/global_step<N>/dataloader/dataloader-<dp_rank>.pt   {"consumed_samples": ...}
    <save_path>/global_step<N>/metadata.json, training_config.yml

The flat fp32 shards (parameters and Adam moments) of every unit are all-gathered unit by unit, cut into the named
tensors of the unit's layout on rank 0 and written with torch.save; loading scatters them back into the shards.
"""

from __future__ import annotations

import json
import os
import random

import numpy as np
import torch
import torch.distributed as dist
import yaml

_PREFIX = "model."  # ModelWrapper.model (model_wrapper/base.py) -> FSDP / state_dict fully-qualified names


def _tag(iteration: int) -> str:
    return f"global_step{iteration}"


def _base(path: str, iteration: int) -> str:
    return os.path.join(path, _tag(iteration))


def _rank_world() -> tuple[int, int]:
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


FP8_RECIPE_FILE = "fp8_recipe.pt"  # delayed-scaling state of the FP8 linears (fp8.Fp8Recipe), written by rank 0


def _engine(model):
    return model.engine if hasattr(model, "engine") else model.model.engine


def _gather_flat(engine, unit, shard: torch.Tensor) -> torch.Tensor:
    """full flat fp32 tensor [padded] of a per-unit shard tensor (parameters or an Adam moment)"""
    if engine.world_size == 1:
        return shard.detach()
    full = torch.empty(unit.padded, dtype=shard.dtype, device=shard.device)
    dist.all_gather_into_tensor(full, shard.detach().contiguous(), group=engine.comm.group)
    return full


def _named(unit, full: torch.Tensor) -> dict[str, torch.Tensor]:
    return {_PREFIX + s.name: full[s.offset : s.offset + s.numel].view(s.shape).cpu().clone() for s in unit.specs}


def _scatter_named(unit, named: dict[str, torch.Tensor], shard: torch.Tensor, what: str) -> None:
    """inverse of _named for this rank's slice: copy the named tensors into the flat shard"""
    full = torch.zeros(unit.padded, dtype=torch.float32)
    for s in unit.specs:
        key = _PREFIX + s.name
        if key not in named:
            raise KeyError(f"{what}: missing {key}")
        t = named[key]
        if tuple(t.shape) != tuple(s.shape):
            raise ValueError(f"{what}: {key} has shape {tuple(t.shape)}, expected {tuple(s.shape)}")
        full[s.offset : s.offset + s.numel] = t.reshape(-1).float()
    lo = unit.rank * unit.shard_numel
    with torch.no_grad():
        shard.copy_(full[lo : lo + unit.shard_numel])


def model_state_dict(model) -> dict[str, torch.Tensor]:
    """full fp32 state dict with the reference's fully-qualified names (collective: every rank must call it)"""
    engine = _engine(model)
    out: dict[str, torch.Tensor] = {}
    for u in engine.units:
        out.update(_named(u, _gather_flat(engine, u, u.master.data)))
    return out


def optimizer_state_dict(model, optimizer) -> dict:
    """FSDP.optim_state_dict-style full optimizer state: moments keyed by parameter name (collective)"""
    engine = _engine(model)
    step = int(getattr(optimizer, "_step", 0))
    state: dict[str, dict] = {}
    for u in engine.units:
        st = optimizer.state.get(u.master, {})
        moments = {}
        if "step" in st:  # torch.optim.AdamW keeps a per-parameter step tensor
            step = int(float(st["step"]))
        for k in ("exp_avg", "exp_avg_sq"):
            shard = st[k] if k in st else torch.zeros_like(u.master.data)
            moments[k] = _named(u, _gather_flat(engine, u, shard))
        for s in u.specs:
            key = _PREFIX + s.name
            state[key] = {"step": torch.tensor(float(step)), "exp_avg": moments["exp_avg"][key],
                          "exp_avg_sq": moments["exp_avg_sq"][key]}
    groups = []
    for g in optimizer.param_groups:
        d = {k: v for k, v in g.items() if k != "params"}
        d["params"] = [_PREFIX + s.name for u in engine.units for s in u.specs]
        groups.append(d)
    return {"state": state, "param_groups": groups}


def save_checkpoint(args, model, optimizer, lr_scheduler, train_dataloader, experiments_tracker, iteration: int,
                    metadata: dict | None = None) -> None:
    """checkpointing.py:50-146 (distributed_backend torch, fsdp_algorithm 1)"""
    rank, _ = _rank_world()
    save_root = args.save_args.save_path
    save_path = _base(save_root, iteration)
    os.makedirs(save_path, exist_ok=True)
    save_opt = getattr(args.save_args, "save_optimizer", True) and optimizer is not None
    if int(getattr(getattr(args, "distributed_args", None), "fsdp_algorithm", 1) or 1) == 2:
        # torch.distributed.checkpoint directories `model/`, `optimizer/` (checkpointing.py:108-113)
        from . import checkpointing_dcp as D

        D.save_model(model, os.path.join(save_path, "model"))
        if save_opt:
            D.save_optimizer(model, optimizer, os.path.join(save_path, "optimizer"))
    else:
        sd = model_state_dict(model)
        if rank == 0:
            torch.save(sd, os.path.join(save_path, "model.pt"))
        del sd
        if save_opt:
            osd = optimizer_state_dict(model, optimizer)
            if rank == 0:
                torch.save(osd, os.path.join(save_path, "optimizer.pt"))
            del osd
    if rank == 0 and lr_scheduler is not None:
        torch.save(lr_scheduler.state_dict(), os.path.join(save_path, "lr_scheduler.pt"))
    rng = {"random_rng_state": random.getstate(), "np_rng_state": np.random.get_state(), "torch_rng_state": torch.get_rng_state(),
           "cuda_rng_state": torch.cuda.get_rng_state() if torch.cuda.is_available() else None}
    eng = _engine(model)
    # counter-based dropout masks and NEFTune noise: (seed, passes so far) is the whole generator state
    if getattr(eng, "uses_pass_seed", False):
        rng["dolomite_b200_dropout_state"] = (eng.dropout_seed, eng._dropout_passes)
    if rank == 0 and getattr(eng, "fp8", None) is not None:  # identical on every rank (amaxes are all-reduced)
        torch.save(eng.fp8.state_dict(), os.path.join(save_path, FP8_RECIPE_FILE))
    os.makedirs(os.path.join(save_path, "rng_state"), exist_ok=True)
    torch.save(rng, os.path.join(save_path, "rng_state", f"rng_state-{rank}.pt"))
    if train_dataloader is not None:
        os.makedirs(os.path.join(save_path, "dataloader"), exist_ok=True)
        state = train_dataloader.state_dict() if hasattr(train_dataloader, "state_dict") else {
            "consumed_samples": int(getattr(train_dataloader, "consumed_samples", 0))}
        torch.save(state, os.path.join(save_path, "dataloader", f"dataloader-{rank}.pt"))
    if rank == 0:
        if experiments_tracker is not None:
            json.dump(experiments_tracker.state_dict(), open(os.path.join(save_path, "experiments_tracker.json"), "w"), indent=4)
        if metadata is not None:
            json.dump(metadata, open(os.path.join(save_path, "metadata.json"), "w"), indent=4)
        cfg = args.model_dump(mode="json") if hasattr(args, "model_dump") else dict(args)
        yaml.safe_dump(cfg, open(os.path.join(save_path, "training_config.yml"), "w"), indent=2)
    if dist.is_available() and dist.is_initialized():
        dist.barrier()
    if rank == 0:
        json.dump({"latest_checkpointed_iteration": iteration},
                  open(os.path.join(save_root, "latest_checkpointed_iteration.json"), "w"), indent=4)


def _strip_wrapper(key: str) -> str:
    """reference checkpoints written with block gradient checkpointing carry the activation-checkpoint wrapper's infix
    (`...h.3._checkpoint_wrapped_module.attn...`, checkpointing.py:41); the engine's names do not"""
    return key.replace("._checkpoint_wrapped_module", "")


def load_model_state_dict(model, sd: dict[str, torch.Tensor]) -> None:
    """every rank reads the full dict and keeps its slice (+ the full bf16 compute copy), like FULL_STATE_DICT loading"""
    engine = _engine(model)
    sd = {_strip_wrapper(k): v for k, v in sd.items()}
    bad = [k for k in sd if not k.startswith(_PREFIX)]
    if bad:
        raise KeyError(f"model checkpoint keys must start with '{_PREFIX}': {bad[:5]}")
    engine.load_state_dict({k[len(_PREFIX):]: v for k, v in sd.items()}, strict=True)


def load_optimizer_state_dict(model, optimizer, osd: dict) -> None:
    engine = _engine(model)
    state = {_strip_wrapper(k): v for k, v in osd["state"].items()}
    step = None
    for u in engine.units:
        st = optimizer.state[u.master]
        for k in ("exp_avg", "exp_avg_sq"):
            if k not in st:
                st[k] = torch.zeros_like(u.master.data)
            _scatter_named(u, {key: v[k] for key, v in state.items()}, st[k], f"optimizer checkpoint ({k})")
        any_key = _PREFIX + u.specs[0].name
        step = int(float(state[any_key]["step"])) if step is None else step
    if hasattr(optimizer, "_step"):
        optimizer._step = step or 0
    else:
        for u in engine.units:
            optimizer.state[u.master]["step"] = torch.tensor(float(step or 0))
    for g, saved in zip(optimizer.param_groups, osd["param_groups"]):
        for k, v in saved.items():
            if k != "params":
                g[k] = tuple(v) if k == "betas" else v


def resume_learning_rate(args, optimizer, lr_scheduler, iteration: int | None) -> None:
    """checkpointing.py:419-445 ("phase 2" resume, used when the stored scheduler is NOT loaded): the YAML's schedule is
    re-created at step `iteration` on top of the learning rates the loaded optimizer currently holds (they become the
    schedule's base rates), and its state replaces the live scheduler's"""
    from .optimization import get_scheduler

    groups = optimizer.param_groups
    kept = [g.get("initial_lr") for g in groups]
    for g in groups:
        g["initial_lr"] = g["lr"]
    ls, tp = args.lr_scheduler_args, args.training_parameters
    fresh = get_scheduler(optimizer, ls.num_warmup_steps, ls.num_constant_steps, ls.num_decay_steps, tp.num_training_steps,
                          ls.lr_decay_style, ls.lr_decay_factor, ls.extra_lr_scheduler_args,
                          last_epoch=-1 if iteration is None else iteration - 1)
    for g, value in zip(groups, kept):
        if value is None:
            g.pop("initial_lr", None)
        else:
            g["initial_lr"] = value
    lr_scheduler.load_state_dict(fresh.state_dict())


def load_checkpoint_for_training(args, model, optimizer, lr_scheduler, train_dataloader):
    """checkpointing.py:149-263 -> (starting iteration, metadata, experiments tracker state) or None when nothing to load"""
    la = getattr(args, "load_args", None)
    if la is None or la.load_path is None:
        return None
    rank, _ = _rank_world()
    iteration = la.iteration
    if iteration is None:
        iteration = json.load(open(os.path.join(la.load_path, "latest_checkpointed_iteration.json")))["latest_checkpointed_iteration"]
    load_path = _base(la.load_path, iteration)
    from . import checkpointing_dcp as D

    want_opt = getattr(la, "load_optimizer", True) and optimizer is not None
    if D.is_dcp_checkpoint(load_path):  # written with fsdp_algorithm: 2 (by this engine or by the reference)
        D.load_model(model, os.path.join(load_path, "model"))
        if want_opt:
            D.load_optimizer(model, optimizer, os.path.join(load_path, "optimizer"))
    else:
        load_model_state_dict(model, torch.load(os.path.join(load_path, "model.pt"), map_location="cpu"))
        if want_opt:
            load_optimizer_state_dict(model, optimizer, torch.load(os.path.join(load_path, "optimizer.pt"), map_location="cpu"))
    if getattr(la, "load_lr_scheduler", True) and lr_scheduler is not None:
        assert getattr(la, "load_optimizer", True), "load_lr_scheduler requires loading of optimizer"
        lr_scheduler.load_state_dict(torch.load(os.path.join(load_path, "lr_scheduler.pt"), weights_only=False))
    elif getattr(la, "resume_learning_rate", True) and lr_scheduler is not None and optimizer is not None:
        resume_learning_rate(args, optimizer, lr_scheduler, iteration)
    fp8_state = os.path.join(load_path, FP8_RECIPE_FILE)
    if getattr(_engine(model), "fp8", None) is not None and os.path.exists(fp8_state):
        _engine(model).fp8.load_state_dict(torch.load(fp8_state, map_location="cpu"))
    if getattr(la, "load_rng_state", True):
        p = os.path.join(load_path, "rng_state", f"rng_state-{rank}.pt")
        if os.path.exists(p):
            rng = torch.load(p, weights_only=False)
            random.setstate(rng["random_rng_state"])
            np.random.set_state(rng["np_rng_state"])
            torch.set_rng_state(rng["torch_rng_state"])
            if rng.get("cuda_rng_state") is not None and torch.cuda.is_available():
                torch.cuda.set_rng_state(rng["cuda_rng_state"])
            if rng.get("dolomite_b200_dropout_state") is not None:
                eng = _engine(model)
                eng.dropout_seed, eng._dropout_passes = rng["dolomite_b200_dropout_state"]
    metadata = None
    if os.path.isfile(os.path.join(load_path, "metadata.json")):
        metadata = json.load(open(os.path.join(load_path, "metadata.json")))
    if getattr(la, "load_dataloader_state", True) and train_dataloader is not None:
        p = os.path.join(load_path, "dataloader", f"dataloader-{rank}.pt")
        if os.path.exists(p):
            state = torch.load(p, weights_only=False)
            if hasattr(train_dataloader, "load_state_dict"):
                train_dataloader.load_state_dict(state)
    tracker = None
    if getattr(la, "load_experiments_tracker_state", True) and os.path.exists(os.path.join(load_path, "experiments_tracker.json")):
        tracker = json.load(open(os.path.join(load_path, "experiments_tracker.json")))
    if not getattr(la, "load_starting_iteration", True):
        iteration = 0
    return iteration, metadata, tracker


def load_checkpoint_for_inference(args, mode="inference", device=None):
    """checkpointing.py:266-402 (distributed_backend torch, tensor_parallel_size 1): rebuild the model from the
    `training_config.yml` stored next to the checkpoint, load `model.pt` / the DCP directory `model/` into it.
    -> (model wrapper, training args of the checkpoint, full state dict or None for DCP)"""
    from .arguments import get_args_from_dict, load_yaml
    from .model_wrapper import get_model

    la = args.load_args
    iteration = la.iteration
    if iteration is None:
        iteration = json.load(open(os.path.join(la.load_path, "latest_checkpointed_iteration.json")))["latest_checkpointed_iteration"]
    load_path = _base(la.load_path, iteration)
    args_from_checkpoint = get_args_from_dict(load_yaml(os.path.join(load_path, "training_config.yml")), "training")
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device())
    # generation runs on padded batches: the finetuning wrapper takes both layouts, the pretraining wrapper only packed text
    args_from_checkpoint.model_args.use_padding_free_transformer = False
    if str(getattr(args_from_checkpoint.tuning_args.tuning_method, "value", args_from_checkpoint.tuning_args.tuning_method)) == "pretraining":
        args_from_checkpoint.tuning_args.tuning_method = "full_finetuning"
    model = get_model(args_from_checkpoint, mode, device=device)
    from . import checkpointing_dcp as D

    state = None
    if D.is_dcp_checkpoint(load_path):
        D.load_model(model, os.path.join(load_path, "model"))
    else:
        state = torch.load(os.path.join(load_path, "model.pt"), map_location="cpu")
        state = {k.replace("._checkpoint_wrapped_module", ""): v for k, v in state.items()}
        load_model_state_dict(model, state)
    return model, args_from_checkpoint, state
