"""N-rank check of the flat-bucket sharded data-parallel runtime against an unsharded run in the same process.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29533 tools/ddp_parity.py

env: COMM_DTYPE=fp32|bf16 (wire dtype of the reduce-scatter), ACCUM=k (micro-steps per optimizer step, the first k-1
under no_sync()), RESHARD=1 (what `stage: 3` means: block units share two parameter / gradient buffers, parameters are
re-gathered in backward, gradients reduce-scattered per micro-step), CKPT=k (block activation checkpointing),
SHARD=S (HSDP: S consecutive ranks per shard group), MOE=1 (MoEDolomite blocks instead of dense ones), FP8=1 (the linears
in FP8 with delayed scaling, ACCUM=1: the ranks all-reduce their amaxes, so every rank must hold the same scales; the
unsharded copy runs every rank's micro-batch with the scales the ranks used in that step).

Every rank r feeds its own micro-batches to the sharded model (world_size = N); rank 0 additionally runs an unsharded
copy of the same model over ALL micro-batches of all ranks.  Checks per step: (1) mean loss over ranks == mean loss
of the unsharded run; (2) reduce-scattered (AVG) gradient shard == slice of (unsharded accumulated gradient / N);
(3) gathered bf16 parameters agree (bit-exact before the first update, tensor-wise afterwards: Adam's first steps
are sign-like, so an element whose tiny gradient flips sign moves by 2*lr)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

from contextlib import nullcontext

from dolomite_engine_b200.distributed import ShardedDataParallel, build_data_parallel_groups, configure_comm_ctas
from dolomite_engine_b200.fp8 import fp8_autocast
from dolomite_engine_b200.model_wrapper import ModelWrapperForPretraining
from dolomite_engine_b200.optimization import get_optimizer

CFG = dict(model_type="gpt_dolomite", vocab_size=1024, n_positions=512, n_embd=320, n_layer=3, n_head=4, n_inner=640,
           attention_head_type="mha", position_embedding_type="rope", activation_function="swiglu",
           normalization_function="rmsnorm", add_bias=True, resid_pdrop=0, embd_pdrop=0, attn_pdrop=0, eos_token_id=7)
# MOE=1: MoEDolomite blocks (8 experts, top-2, no biases): the K-grouped expert weight gradients overwrite their (pooled) buffers
MOE_CFG = dict(CFG, model_type="moe_dolomite", num_experts=8, num_experts_per_tok=2, add_bias=False)
OPT = {"lr": 1e-3, "weight_decay": 0.1, "betas": [0.9, 0.95], "eps": 1e-10}


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    configure_comm_ctas()
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    comm_dtype = torch.float32 if os.environ.get("COMM_DTYPE", "fp32") == "fp32" else torch.bfloat16
    accum = int(os.environ.get("ACCUM", "1"))
    reshard = bool(int(os.environ.get("RESHARD", "0")))
    mbs, seq = 2, 128
    # SHARD=S: HSDP with S consecutive ranks per shard group, world / S replicas (zero_topology)
    shard = int(os.environ.get("SHARD", "0")) or None
    group, rep_group, s_world, s_rank = build_data_parallel_groups(shard, world // shard if shard else None)
    moe = os.environ.get("MOE", "0") == "1"
    CFG = MOE_CFG if moe else globals()["CFG"]
    w = ModelWrapperForPretraining(pretrained_config=dict(CFG), micro_batch_size=mbs, sequence_length=seq, device=dev,
                                   world_size=s_world, rank=s_rank)
    if os.environ.get("CKPT"):
        w.model.engine.checkpoint_every = int(os.environ["CKPT"])
    sdp = ShardedDataParallel(w, group, communication_dtype=comm_dtype, reshard_after_forward=reshard,
                              replicate_group=rep_group)
    opt = get_optimizer("DolomiteFusedAdamW", OPT, sdp)
    ref = ref_sdp = ref_opt = None
    if rank == 0:
        ref = ModelWrapperForPretraining(pretrained_config=dict(CFG), micro_batch_size=mbs, sequence_length=seq, device=dev)
        ref_sdp = ShardedDataParallel(ref, None, reshard_after_forward=False)
        ref_opt = get_optimizer("DolomiteFusedAdamW", OPT, ref_sdp)
    fp8 = os.environ.get("FP8", "0") == "1"
    eng = w.model.engine
    ref_eng = ref.model.engine if rank == 0 else None
    if fp8:
        assert accum == 1, "FP8=1 runs with ACCUM=1"
        eng.enable_fp8()
        if rank == 0:
            ref_eng.enable_fp8()
            ref_eng.fp8.update = lambda all_reduce=False: None  # takes the ranks' scales before every step instead
    ctx = (lambda e: fp8_autocast(e)) if fp8 else (lambda e: nullcontext())
    rng = np.random.default_rng(0)
    ok = True
    for step in range(4):
        if fp8 and rank == 0:
            ref_eng.fp8.load_state_dict(eng.fp8.state_dict())
        # tokens[m][r]: micro-step m, rank r
        tokens = [[torch.from_numpy(rng.integers(0, 1024, size=(mbs, seq + 1), dtype=np.int64)) for _ in range(world)]
                  for _ in range(accum)]
        sdp.zero_grad()
        lsum = torch.zeros((), device=dev)
        with sdp.no_sync():
            for m in range(accum - 1):
                l = sdp({"text": tokens[m][rank]})
                l.backward()
                lsum += l.detach()
        with ctx(eng):
            l = sdp({"text": tokens[accum - 1][rank]})
        l.backward()
        lsum += l.detach()
        torch.cuda.synchronize()
        lsum /= accum
        dist.all_reduce(lsum, op=dist.ReduceOp.AVG)
        fulls = [w.model.engine.full_master(u) for u in w.model.engine.units]  # collective: every rank
        if fp8:  # the amax all-reduce gives every rank the same scales
            st = torch.cat([eng.fp8.fwd_scale, eng.fp8.bwd_scale, eng.fp8.fwd_history.flatten()])
            every = [torch.empty_like(st) for _ in range(world)]
            dist.all_gather(every, st)
            same = all(torch.equal(every[0], x) for x in every)
            if rank == 0 and not same:
                print(f"step {step}: FP8 scales differ between ranks", flush=True)
            ok = ok and same
        if rank == 0:
            ref_sdp.zero_grad()
            rl = 0.0
            for m in range(accum):
                for t in tokens[m]:
                    with ctx(ref_eng):
                        x = ref_sdp({"text": t})
                    x.backward()
                    rl += x.item()
            rl /= world * accum
            dl = abs(lsum.item() - rl) / rl
            worst, pworst = 0.0, 0.0
            for u, ru, full in zip(w.model.engine.units, ref.model.engine.units, fulls):
                # what the next all-gather will deliver (bf16 of the fp32 shards) vs the unsharded model's bf16 parameters
                a, b = full[: ru.numel].bfloat16().float(), ru.compute[: ru.numel].float()
                pworst = max(pworst, ((a - b).norm() / (b.norm() + 1e-20)).item())
                g = u.master.grad
                lo, hi = s_rank * u.shard_numel, (s_rank + 1) * u.shard_numel
                if hi <= ru.padded:
                    rg = (ru.master.grad / world)[lo:hi]
                    worst = max(worst, ((g - rg).norm() / (rg.norm() + 1e-20)).item())
            gtol = (2e-2 if comm_dtype == torch.bfloat16 else 1e-5) if step == 0 else 5e-2
            if moe and step > 0:
                # the two trajectories drift apart (wire rounding, sign-like first Adam steps) and a router logit near a tie then
                # selects another expert in one of them: a flip rate f moves the gradients by ~sqrt(2 f) (DESIGN 8.4).
                # Step 0 -- identical parameters -- keeps the strict bound.
                gtol = 1.5e-1
            ptol = 1e-6 if step == 0 else 2e-2
            good = dl < 1e-3 and worst < gtol and pworst < ptol
            print(f"step {step}: loss {lsum.item():.6f} ref {rl:.6f} rel {dl:.2e}; shard-grad rel-L2 {worst:.2e}; "
                  f"gathered-param rel-L2 {pworst:.2e} {'ok' if good else 'MISMATCH'}", flush=True)
            ok = ok and good
            # the sharded run averages gradients over ranks; give the reference the same scale before clip + AdamW
            for ru in ref.model.engine.units:
                ru.master.grad.div_(world)
            ref_sdp.clip_grad_norm_(1.0, fuse_into_optimizer=True)
            ref_opt.step()
        sdp.clip_grad_norm_(1.0, fuse_into_optimizer=True)
        opt.step()
    flag = torch.tensor([1.0 if ok else 0.0], device=dev)
    dist.broadcast(flag, 0)
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print("DDP_PARITY", "OK" if ok else "FAILED", f"(world {world}, wire {os.environ.get('COMM_DTYPE', 'fp32')}, accum {accum}, "
              f"reshard {int(reshard)}, moe {os.environ.get('MOE', '0')}, fp8 {int(fp8)})", flush=True)
    sys.exit(0 if flag.item() == 1.0 else 1)


if __name__ == "__main__":
    main()
