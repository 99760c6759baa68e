"""Flat-bucket sharded data parallelism for the B200 path (replaces torch FSDP as configured by
`wrap_model_for_distributed_training`, reference distributed/__init__.py:47-236).

One FlatUnit per transformer block + one root unit (same wrapping as `transformer_auto_wrap_policy` over
`_no_split_modules`).  Rank r owns slice r of every unit's fp32 master / optimizer state.  Per step and unit:

  forward   cast own fp32 shard -> bf16 into its slice of the unit's gather buffer, in-place `ncclAllGather`
            on the communication stream, prefetched one unit ahead of the compute stream (N1 of SURVEY 2.2)
  backward  wgrad GEMM epilogues accumulate into the unit's full gradient buffer; when the unit's backward is
            done (last micro-step only, i.e. outside `no_sync`) `ncclReduceScatter(AVG)` on the communication
            stream overlaps the next unit's backward (N2)

Placement choices: the gathered bf16 parameters of a 3.5 B (8 B) model are 7 GB (16 GB) of an 80 GB H100, so units
stay resident between forward and backward (`reshard_after_forward=False`; one all-gather per unit per optimizer
step instead of the reference's two per micro-step) unless stage-3 resharding is requested; gather/gradient buffers
are allocated once (no allocator churn, no record_stream); scalar collectives (loss AVG, grad-norm SUM) stay on
the device without `.item()` until the caller asks.
"""

from __future__ import annotations

import contextlib
import os

import torch
import torch.distributed as dist
import torch.nn as nn

from . import kernels as K
from .engine import DolomiteEngine, FlatUnit


def comm_cta_budget() -> int:
    """CTAs (= SMs) the NCCL collectives may occupy; DOLO_COMM_CTAS overrides (default 8)."""
    return int(os.environ.get("DOLO_COMM_CTAS", "8"))


def configure_comm_ctas() -> None:
    """Call BEFORE `init_process_group`: caps NCCL at `comm_cta_budget()` CTAs per collective (NVLink 5 needs few
    CTAs for the ~210 MB per-unit all-gather / reduce-scatter) so that the budget can be subtracted from the
    persistent GEMM grids instead of letting them queue behind the communication kernels."""
    os.environ.setdefault("NCCL_MAX_CTAS", str(comm_cta_budget()))
    os.environ.setdefault("NCCL_MIN_CTAS", "1")


def hybrid_layout(world_size: int, sharding_world_size: int | None, replication_world_size: int | None):
    """Rank lists of the 2-D data-parallel topology (`zero_topology`, reference arguments.py:283-298,
    utils/parallel.py:59-68 and :255-266).  Returns (shard_groups, replicate_groups): parameters / optimizer state are
    sharded inside a shard group and replicated across the groups; gradients are reduce-scattered inside the shard group
    and then all-reduced between the ranks that own the same slice.

    Placement: a shard group is `sharding_world_size` CONSECUTIVE ranks (one NVSwitch domain), so the large
    per-unit all-gather / reduce-scatter stay on NVLink and only the 1/S-sized shard all-reduce crosses nodes."""
    if replication_world_size is None or sharding_world_size is None:
        if replication_world_size is not None or sharding_world_size is not None:
            raise ValueError("data_parallel_replication_world_size and data_parallel_sharding_world_size go together")
        return [list(range(world_size))], [[r] for r in range(world_size)]
    S, R = int(sharding_world_size), int(replication_world_size)
    if S < 1 or R < 1 or S * R != world_size:
        raise ValueError(f"replication ({R}) x sharding ({S}) world sizes must equal the data-parallel world size ({world_size})")
    shard_groups = [[g * S + i for i in range(S)] for g in range(R)]
    replicate_groups = [[g * S + i for g in range(R)] for i in range(S)]
    return shard_groups, replicate_groups


def build_data_parallel_groups(sharding_world_size: int | None = None, replication_world_size: int | None = None):
    """-> (shard_group, replicate_group or None, shard_world_size, shard_rank).  Collective: every rank creates every
    group, in the same order (`dist.new_group` contract)."""
    world, rank = dist.get_world_size(), dist.get_rank()
    shard_groups, replicate_groups = hybrid_layout(world, sharding_world_size, replication_world_size)
    if len(shard_groups) == 1:
        return dist.group.WORLD, None, world, rank
    mine_s = mine_r = None
    for ranks in shard_groups:
        g = dist.new_group(ranks)
        if rank in ranks:
            mine_s = (g, ranks)
    for ranks in replicate_groups:
        g = dist.new_group(ranks)
        if rank in ranks:
            mine_r = g
    return mine_s[0], mine_r, len(mine_s[1]), mine_s[1].index(rank)


class _SlotTable:
    """Who owns which shared parameter buffer (stage-3 / pooled mode).  Unit 0 (root) and every unit of the resident mode
    own a private buffer (slot -1); block unit i >= 1 of the pooled mode uses slot (i - 1) mod n_slots.  Pure bookkeeping,
    no device work: `claim(i)` is called when unit i's all-gather is issued and returns the unit that loses the slot."""

    def __init__(self, pooled: list[bool], n_slots: int):
        self.pooled = list(pooled)
        self.n_slots = n_slots
        self.slot_of = [((i - 1) % n_slots if p else -1) for i, p in enumerate(pooled)]
        self.owner = [-1] * n_slots
        self.fresh = [False] * len(pooled)  # the unit's buffer holds its current parameters (once its gather is waited)

    def invalidate(self) -> None:
        self.fresh = [False] * len(self.fresh)

    def is_fresh(self, i: int) -> bool:
        return self.fresh[i] and (not self.pooled[i] or self.owner[self.slot_of[i]] == i)

    def claim(self, i: int) -> int:
        if not self.pooled[i]:
            return -1
        s = self.slot_of[i]
        prev = self.owner[s]
        self.owner[s] = i
        if prev >= 0 and prev != i:
            self.fresh[prev] = False
            return prev
        return -1


class _Comm:
    """engine hooks: all-gather prefetch in forward, reduce-scatter (+ replica all-reduce) in backward.

    Two memory modes.  resident (`reshard_after_forward=False`, FSDP SHARD_GRAD_OP-like and kept until the optimizer step):
    every unit owns its gathered bf16 parameters and its full fp32 gradient buffer; one all-gather per unit per optimizer
    step.  reshard (`reshard_after_forward=True`, what `stage: 3` means in the reference, distributed/__init__.py:205-213):
    the block units share `engine.pool_slots` parameter buffers and as many gradient buffers (engine.convert_to_pooled);
    a block's parameters are re-gathered for its backward and its gradients are reduce-scattered as soon as its backward
    ends, on EVERY micro-step (FULL_SHARD never holds unsharded gradients; under `no_sync()` the reduced shards accumulate,
    which is the same sum)."""

    def __init__(self, engine: DolomiteEngine, group, communication_dtype: torch.dtype, reshard_after_forward: bool,
                 replicate_group=None):
        self.engine = engine
        self.group = group
        self.replicate_group = replicate_group
        self.ws = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.comm_dtype = communication_dtype
        self.reshard = reshard_after_forward
        if self.reshard:
            engine.convert_to_pooled(int(os.environ.get("DOLO_POOL_SLOTS", "2")))
        self.stream = torch.cuda.Stream(device=engine.device, priority=-1)
        n = len(engine.units)
        self.ag_work: list = [None] * n
        self.rs_work: list = [None] * n
        self.sync_grads = True
        self.pooled = [u.pooled for u in engine.units]
        n_slots = getattr(engine, "pool_slots", 0) if any(self.pooled) else 0
        self.slots = _SlotTable(self.pooled, max(n_slots, 1))
        self.slot_of = self.slots.slot_of
        self.grad_slot_free = [None] * max(n_slots, 1)  # event: the slot's gradients have left for the wire
        self.first_rs = [True] * n                 # first reduce-scatter of the accumulation window overwrites the shard grad
        biggest = max(u.padded for u in engine.units)
        if communication_dtype == torch.bfloat16:
            self.rs_stage = [torch.empty(biggest, dtype=torch.bfloat16, device=engine.device) for _ in range(2)]
            self.rs_out = [torch.empty(biggest // self.ws, dtype=torch.bfloat16, device=engine.device) for _ in range(2)]
            self.rs_stage_evt = [None, None]
        elif self.reshard:
            self.rs_out32 = [torch.empty(biggest // self.ws, dtype=torch.float32, device=engine.device) for _ in range(2)]
            self.rs_stage_evt = [None, None]
        self._rs_count = 0

    # ---- all-gather ----
    def invalidate(self) -> None:
        self.slots.invalidate()

    def window_reset(self) -> None:
        """zero_grad(): the next reduce-scatter of every unit starts a new accumulation window"""
        self.first_rs = [True] * len(self.first_rs)

    def _issue_gather(self, i: int) -> None:
        if self.slots.is_fresh(i) or self.ag_work[i] is not None:
            return
        u = self.engine.units[i]
        cur = torch.cuda.current_stream()
        # previous readers of the buffer (last backward; in pooled mode the block that used the slot before) are ordered
        # before the overwrite: everything enqueued on the compute stream so far
        self.stream.wait_stream(cur)
        prev = self.slots.claim(i)
        assert prev < 0 or self.ag_work[prev] is None, "parameter slot reassigned while its gather is still pending"
        with torch.cuda.stream(self.stream):
            own = u.compute[self.rank * u.shard_numel : (self.rank + 1) * u.shard_numel]
            K.cast_f32_to_bf16(u.master.data, own)
            self.ag_work[i] = dist.all_gather_into_tensor(u.compute, own, group=self.group, async_op=True)

    def _wait_gather(self, i: int) -> None:
        if self.ag_work[i] is not None:
            self.ag_work[i].wait()  # compute stream waits (device side) for the collective
            self.ag_work[i] = None
            self.slots.fresh[i] = True

    def pre_forward_unit(self, i: int) -> None:
        self._issue_gather(i)
        if i + 1 < len(self.pooled):
            self._issue_gather(i + 1)  # prefetch depth 1
        self._wait_gather(i)

    def post_forward_unit(self, i: int) -> None:
        pass  # pooled mode: a block's parameters disappear when its slot is handed to the next block

    def pre_backward_unit(self, i: int) -> None:
        if self.pooled[i]:
            self._issue_gather(i)
            if i - 1 >= 1:
                self._issue_gather(i - 1)
            self._wait_gather(i)
            evt = self.grad_slot_free[self.slot_of[i]]
            if evt is not None:  # the block that used this gradient slot before has handed its gradients to the wire
                torch.cuda.current_stream().wait_event(evt)
                self.grad_slot_free[self.slot_of[i]] = None
            self.engine.prepare_unit_grads(i)

    # ---- reduce-scatter ----
    def post_backward_unit(self, i: int) -> None:
        if not self.sync_grads and not self.pooled[i]:
            return
        if not self.sync_grads and i == 0:
            return  # the root keeps its own gradient buffer: accumulate under no_sync like the resident mode
        u = self.engine.units[i]
        if self.pooled[i]:
            self.engine.finish_unit_grads(i)
        cur = torch.cuda.current_stream()
        self.stream.wait_stream(cur)
        self.engine.join_wgrad_stream(self.stream)  # weight gradients launched on the engine's second stream
        first = self.first_rs[i]
        self.first_rs[i] = False
        with torch.cuda.stream(self.stream):
            slot = self._rs_count % 2
            self._rs_count += 1
            if self.comm_dtype == torch.bfloat16:
                if self.rs_stage_evt[slot] is not None:
                    self.rs_stage_evt[slot].wait()
                stage = self.rs_stage[slot][: u.padded]
                out = self.rs_out[slot][: u.shard_numel]
                K.cast_f32_to_bf16(u.grad_full, stage)
                if self.pooled[i]:  # the fp32 gradient slot is free as soon as the bf16 wire copy exists
                    free = torch.cuda.Event()
                    free.record(self.stream)
                    self.grad_slot_free[self.slot_of[i]] = free
                work = dist.reduce_scatter_tensor(out, stage, op=dist.ReduceOp.AVG, group=self.group, async_op=True)
                work.wait()  # orders the comm stream after the collective
                if self.replicate_group is not None:  # HSDP: mean over the replicas of this slice, still in bf16
                    dist.all_reduce(out, op=dist.ReduceOp.AVG, group=self.replicate_group)
                if first or not self.pooled[i]:
                    u.master.grad.zero_()
                K.accum_bf16_into_f32(out, u.master.grad, 1.0)
                evt = torch.cuda.Event()
                evt.record(self.stream)
                self.rs_stage_evt[slot] = evt
                self.rs_work[i] = evt
            elif self.pooled[i]:
                if self.rs_stage_evt[slot] is not None:
                    self.rs_stage_evt[slot].wait()
                out = self.rs_out32[slot][: u.shard_numel]
                work = dist.reduce_scatter_tensor(out, u.grad_full, op=dist.ReduceOp.AVG, group=self.group, async_op=True)
                work.wait()
                free = torch.cuda.Event()
                free.record(self.stream)
                self.grad_slot_free[self.slot_of[i]] = free
                if self.replicate_group is not None:
                    dist.all_reduce(out, op=dist.ReduceOp.AVG, group=self.replicate_group)
                if first:
                    u.master.grad.copy_(out)
                else:
                    u.master.grad.add_(out)
                evt = torch.cuda.Event()
                evt.record(self.stream)
                self.rs_stage_evt[slot] = evt
                self.rs_work[i] = evt
            else:
                work = dist.reduce_scatter_tensor(u.master.grad, u.grad_full, op=dist.ReduceOp.AVG, group=self.group,
                                                  async_op=True)
                if self.replicate_group is not None:
                    work.wait()
                    work = dist.all_reduce(u.master.grad, op=dist.ReduceOp.AVG, group=self.replicate_group, async_op=True)
                self.rs_work[i] = work
        if i == 0:
            self.finish_backward()

    def finish_backward(self) -> None:
        cur = torch.cuda.current_stream()
        for i, w in enumerate(self.rs_work):
            if w is None:
                continue
            if isinstance(w, torch.cuda.Event):
                cur.wait_event(w)
            else:
                w.wait()
            self.rs_work[i] = None
        # (the full gradient buffers are zeroed by zero_grad() at the start of the next accumulation window)

    def gather_master(self, unit: FlatUnit) -> torch.Tensor:
        full = torch.empty(unit.padded, dtype=torch.float32, device=unit.master.device)
        dist.all_gather_into_tensor(full, unit.master.data, group=self.group)
        return full


class ShardedDataParallel(nn.Module):
    """What `wrap_model_for_distributed_training` returns.  Supports what train_utils.train_step needs from an
    FSDP-1 style wrapper: `.no_sync()`, `.clip_grad_norm_(max_norm)`, `.parameters()` (flat fp32 shards with
    `.grad`), `.train()/.eval()`, `.config`, `.tokenizer` and `forward(batch) -> loss`."""

    def __init__(self, model_wrapper: nn.Module, process_group=None, communication_dtype: torch.dtype | None = None,
                 reshard_after_forward: bool = True, replicate_group=None):
        super().__init__()
        self.module = model_wrapper
        self.engine: DolomiteEngine = model_wrapper.model.engine
        self.group = process_group  # the SHARD group; `replicate_group` links the owners of the same slice (HSDP)
        self.replicate_group = replicate_group
        # the engine was built for a given data-parallel degree; a world_size-1 engine stays unsharded even when a
        # process group exists (e.g. an unsharded reference copy next to a sharded model)
        self.world_size = self.engine.world_size
        if self.world_size == 1 and replicate_group is not None and dist.get_world_size(replicate_group) > 1:
            raise NotImplementedError("replication without sharding (data_parallel_sharding_world_size == 1) is not built: "
                                      "shard over the box's GPUs and replicate across boxes")
        if self.world_size > 1:
            assert dist.is_initialized() and dist.get_world_size(process_group) == self.world_size, \
                "engine must be built with world_size/rank of the (shard) DP group"
            comm_dtype = torch.bfloat16 if communication_dtype is None else communication_dtype
            self.engine.comm = _Comm(self.engine, process_group, comm_dtype, reshard_after_forward, replicate_group)
            # STATIC persistent GEMM grids (gemm_dynamic = 0) must not claim the SMs the NCCL kernels run on (see
            # configure_comm_ctas); the default cluster-launch-control grids ignore the margin: they run on whatever SMs are
            # free and pick up the ones a collective releases
            K.set_option("gemm_sm_margin", comm_cta_budget())
        self._sumsq = torch.zeros(1, dtype=torch.float32, device=self.engine.device)
        self.clip_coef = torch.ones(1, dtype=torch.float32, device=self.engine.device)
        self.grad_norm = torch.zeros(1, dtype=torch.float32, device=self.engine.device)
        self._stale = True
        self._versions = [-1] * len(self.engine.units)

    # ---- attribute passthrough ----
    @property
    def config(self):
        return self.module.config

    @property
    def tokenizer(self):
        return getattr(self.module, "tokenizer", None)

    def parameters(self, recurse: bool = True):
        for u in self.engine.units:
            yield u.master

    def named_parameters(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True):
        for u in self.engine.units:
            yield f"{prefix}flat.{u.name}", u.master

    # ---- parameter freshness ----
    def mark_parameters_updated(self) -> None:
        """call after the optimizer changed the fp32 masters (train_step does; torch optimizers are also detected
        through the tensors' version counters)"""
        self._stale = True

    def _refresh_parameters_if_needed(self) -> None:
        changed = self._stale
        for i, u in enumerate(self.engine.units):
            if u.master._version != self._versions[i]:
                changed = True
        if not changed:
            return
        if self.engine.comm is not None:
            self.engine.comm.invalidate()
        else:
            self.engine.refresh_compute_from_master()
        self._versions = [u.master._version for u in self.engine.units]
        self._stale = False

    def notify_fused_update(self) -> None:
        """the fused AdamW already wrote the bf16 copies (world_size == 1) -> nothing to refresh"""
        self._versions = [u.master._version for u in self.engine.units]
        self._stale = self.engine.comm is not None
        if self.engine.comm is not None:
            self.engine.comm.invalidate()
            self._stale = False

    # ---- forward ----
    def forward(self, batch: dict) -> torch.Tensor:
        self._refresh_parameters_if_needed()
        return self.module(batch)

    @contextlib.contextmanager
    def no_sync(self):
        comm = self.engine.comm
        if comm is None:
            yield
            return
        prev = comm.sync_grads
        comm.sync_grads = False
        try:
            yield
        finally:
            comm.sync_grads = prev

    def set_requires_gradient_sync(self, flag: bool) -> None:  # FSDP-2 style spelling
        if self.engine.comm is not None:
            self.engine.comm.sync_grads = bool(flag)

    # ---- gradient clipping (train_utils.py:99-103) ----
    def clip_grad_norm_(self, max_norm: float, fuse_into_optimizer: bool = False) -> torch.Tensor:
        """total L2 norm over all ranks' shards; returns a 0-d device tensor (no host sync).  With
        `fuse_into_optimizer` the gradients are left unscaled and the clip coefficient (device scalar
        `self.clip_coef`) is consumed by DolomiteFusedAdamW; otherwise gradients are scaled in place."""
        self._sumsq.zero_()
        for u in self.engine.units:
            K.sumsq_accum(u.master.grad, self._sumsq)
        if self.world_size > 1:
            dist.all_reduce(self._sumsq, op=dist.ReduceOp.SUM, group=self.group)
        K.clip_coef(self._sumsq, max_norm, self.clip_coef, self.grad_norm)
        if not fuse_into_optimizer:
            for u in self.engine.units:
                u.master.grad.mul_(self.clip_coef)
        return self.grad_norm.reshape(())

    def zero_grad(self, set_to_none: bool = False) -> None:
        self.engine.zero_grad()

    def state_dict(self, *args, **kwargs):
        return self.engine.state_dict()

    def load_state_dict(self, sd, strict: bool = True, assign: bool = False):
        self.engine.load_state_dict(sd, strict=strict)
        self.mark_parameters_updated()


def wrap_model_for_distributed_training(args, model: nn.Module) -> nn.Module:
    """Reference signature (distributed/__init__.py:47).  Reads the same knobs from `args.distributed_args`:
    `stage` -- 3 reshards the parameters after forward and shares the gather / gradient buffers between blocks, exactly
    what `reshard_after_forward = stage == 3` / FULL_SHARD does in the reference (distributed/__init__.py:161-176,
    :205-213); 0 / 2 keep every unit's gathered parameters and full gradients resident (SHARD_GRAD_OP-like) --,
    `communication_dtype`, `fsdp_algorithm` (both map to the same flat-bucket runtime), and rejects what is out of scope.
    The one key the reference does not have is `reshard_after_forward` (default None = follow `stage`): `false` together with
    `stage: 3` opts into the resident mode, which trades ~6 B / parameter of HBM for one all-gather per unit and step."""
    dargs = getattr(args, "distributed_args", None)
    stage = getattr(dargs, "stage", 3) if dargs is not None else 3
    comm_dtype = None
    if dargs is not None and getattr(dargs, "communication_dtype", None) is not None:
        comm_dtype = {"fp32": torch.float32, "bf16": torch.bfloat16}[str(dargs.communication_dtype).split(".")[-1]]
    if dargs is not None:
        if str(getattr(dargs, "distributed_backend", "torch")).split(".")[-1] != "torch":
            raise NotImplementedError("only distributed_backend=torch (NCCL) exists on the B200 path; no DeepSpeed dispatch")
        if getattr(dargs, "tensor_parallel_size", 1) != 1:
            raise NotImplementedError("tensor parallelism is out of scope of the data-parallel B200 path")
        if getattr(dargs, "torch_compile", False):
            raise NotImplementedError("torch.compile is not used on the B200 path (hand-written kernels + CUDA streams)")
    explicit = getattr(dargs, "reshard_after_forward", None) if dargs is not None else None
    reshard = (stage == 3) if explicit is None else bool(explicit)
    if dargs is not None and getattr(dargs, "gradient_checkpointing_method", None) is not None:
        # block_checkpointing(model, block_name, checkpoint_every=1) (distributed/__init__.py:113-121,
        # gradient_checkpointing/block.py:13-37): blocks 0, k, 2k, ... keep only their input and are re-run in backward
        every = int((getattr(dargs, "gradient_checkpointing_args", None) or {}).get("checkpoint_every", 1))
        model.model.engine.checkpoint_every = every
    group, replicate_group = (dist.group.WORLD if dist.is_initialized() else None), None
    topo = getattr(dargs, "zero_topology", None) if dargs is not None else None
    if topo is not None and getattr(topo, "data_parallel_replication_world_size", None) is not None:
        # HSDP: the engine must have been built with the SHARD group's size / rank (pretrain.build does)
        group, replicate_group, _, _ = data_parallel_groups(topo.data_parallel_sharding_world_size,
                                                            topo.data_parallel_replication_world_size)
    return ShardedDataParallel(model, group, communication_dtype=comm_dtype, reshard_after_forward=reshard,
                               replicate_group=replicate_group)


_GROUP_CACHE: dict = {}


def data_parallel_groups(sharding_world_size: int | None, replication_world_size: int | None):
    """memoised `build_data_parallel_groups` (process groups are created once per topology)"""
    key = (sharding_world_size, replication_world_size)
    if key not in _GROUP_CACHE:
        _GROUP_CACHE[key] = build_data_parallel_groups(sharding_world_size, replication_world_size)
    return _GROUP_CACHE[key]


def shard_world_and_rank(args, world: int, rank: int) -> tuple[int, int]:
    """(world_size, rank) the ENGINE must be built with: the shard group's under `zero_topology` (HSDP), else the global ones.
    The data feed and the loss average always use the global (rank, world)."""
    dargs = getattr(args, "distributed_args", None)
    topo = getattr(dargs, "zero_topology", None) if dargs is not None else None
    if world > 1 and topo is not None and getattr(topo, "data_parallel_replication_world_size", None) is not None:
        _, _, shard_world, shard_rank = data_parallel_groups(topo.data_parallel_sharding_world_size,
                                                             topo.data_parallel_replication_world_size)
        return shard_world, shard_rank
    return world, rank
