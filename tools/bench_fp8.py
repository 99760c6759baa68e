"""FP8 vs BF16 GEMMs at the four C2 block shapes (one 4096-token sequence), timed with CUDA events in one process.

    python tools/bench_fp8.py [--tokens 4096] [--iters 50] [--dump DIR]

First the training step: one C2 model (seq 4096, one sequence, fused AdamW, the configuration of bench.py), whose steps run
alternately in BF16 and in FP8 (the same engine with and without fp8_autocast), reporting tokens/s, step time and the peak
allocated HBM of each mode.  Then, for each C2 block shape, it times, alternating BF16 and FP8 launches, the forward GEMM (bf16: K-major x K-major; fp8: fast
accumulation) and the weight-gradient GEMM (bf16: MN-major operands into fp32; fp8: split accumulation on the transposed
casts), reports achieved TFLOP/s from the shapes, and the time of the cast kernels the FP8 linear adds (input and weight
casts of the forward; cast-transpose of the output gradient and the transposed re-casts of the backward).  Prints one JSON
line with the card name and power limit.

--dump DIR writes, as .npy files, what the FP8 GEMMs compute from seeded inputs, so that two builds can be compared
byte for byte: the output of every FP8 GEMM job it times at the C2 shapes (fresh outputs, one launch each); a grid of
small GEMMs over the four format pairs, split accumulation on / off, fp32 and bf16 D and bias / C / both, with M and N
tails, and one four-problem weight-gradient launch; and, under train/, the loss of the FP8 training steps and a fixed
sample of parameters and gradients after the last one (bench.py's dump_outputs).
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from contextlib import nullcontext

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))  # the repository root (bench.py)

from dolomite_engine_b200 import kernels as K  # noqa: E402



def c2_block_shapes() -> dict:
    """{linear: (N, K)} of a C2 block, from the flagship benchmark's model configuration"""
    import bench

    cfg = bench.model_config("c2")
    H, F, nh = cfg["n_embd"], cfg["n_inner"], cfg["n_head"]
    kv = {"mha": nh, "mqa": 1}.get(cfg["attention_head_type"], cfg.get("num_key_value_heads") or nh)
    fc = 2 * F if cfg["activation_function"].endswith("glu") else F
    return {"c_attn": (H + 2 * kv * (H // nh), H), "attn.c_proj": (H, H), "c_fc": (fc, H), "mlp.c_proj": (H, F)}


def _card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the numbers are still reported; the card line says why it is missing
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unavailable ({e})"}


def _time(fn, iters: int) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e-3


def _save(dump: str, name: str, t: torch.Tensor) -> None:
    import numpy as np

    os.makedirs(dump, exist_ok=True)
    np.save(os.path.join(dump, name + ".npy"), t.detach().contiguous().view(torch.uint8).cpu().numpy())


def dump_grid(dump: str) -> None:
    """the FP8 GEMM at M = 200, N = 272, K = 208 (tails on 128 x 128 tiles) over every format pair, accumulation mode,
    output type and epilogue input, and one weight-gradient launch of four problems, two of them accumulating"""
    g = torch.Generator(device="cuda").manual_seed(1)

    def operand(rows, cols, fmt):
        x = torch.randn(rows, cols, device="cuda", generator=g).to(torch.bfloat16)
        return K.fp8_cast(x, fmt, torch.tensor([100.0 if fmt == K.E4M3 else 5000.0], device="cuda"))[0]

    M, N, Kd = 200, 272, 208
    sa, sb = torch.tensor([0.0173], device="cuda"), torch.tensor([0.0291], device="cuda")
    bias = torch.randn(N, device="cuda", generator=g).to(torch.bfloat16)
    for fa in (K.E4M3, K.E5M2):
        for fb in (K.E4M3, K.E5M2):
            A, B = operand(M, Kd, fa), operand(N, Kd, fb)
            for split in (False, True):
                for dt in (torch.float32, torch.bfloat16):
                    for wb, wc in ((True, False), (False, True), (True, True)):
                        c = torch.randn(M, N, device="cuda", generator=g).to(dt) if wc else None
                        d = K.gemm_fp8(A, fa, sa, B, fb, sb, out_dtype=dt, c=c, alpha=0.7, beta=1.3,
                                       bias=bias if wb else None, split_accumulate=split)
                        _save(dump, f"grid_{fa}{fb}_split{int(split)}_{str(dt)[6:]}_bias{int(wb)}_c{int(wc)}", d)
    for split in (False, True):
        probs = []
        for q, (M, N) in enumerate([(200, 272), (128, 384), (384, 144), (64, 128)]):
            probs.append((operand(M, 336, K.E5M2), sa, operand(N, 336, K.E4M3), sb,
                          torch.randn(M, N, device="cuda", generator=g), 0.3 + q, q in (1, 2)))
        K.gemm_fp8_wgrad_multi(probs, split_accumulate=split)
        for q, p in enumerate(probs):
            _save(dump, f"wgrad_multi_split{int(split)}_{q}", p[4])


def train_steps(steps: int, rounds: int, dump: str | None = None) -> dict:
    """alternating blocks of `steps` BF16 and FP8 C2 training steps on one model; best block of each mode"""
    import bench  # the C2 model configuration of the flagship benchmark

    from dolomite_engine_b200.distributed import ShardedDataParallel
    from dolomite_engine_b200.fp8 import fp8_autocast
    from dolomite_engine_b200.model_wrapper import ModelWrapperForPretraining
    from dolomite_engine_b200.optimization import get_optimizer
    from dolomite_engine_b200.pretrain import SyntheticPackedDataset
    from dolomite_engine_b200.train_utils import train_step

    dev = torch.device("cuda", 0)
    cfg = bench.model_config("c2")
    seq = bench.WORKLOADS["c2"]["seq"]
    wrapper = ModelWrapperForPretraining(pretrained_config=cfg, micro_batch_size=1, sequence_length=seq, device=dev,
                                         init_on_device=True)
    engine = wrapper.model.engine
    engine.enable_fp8()
    model = ShardedDataParallel(wrapper, None)
    opt = get_optimizer("DolomiteFusedAdamW", {"lr": 1e-5, "weight_decay": 0.1, "betas": [0.9, 0.95], "eps": 1e-10}, model)
    data = SyntheticPackedDataset(cfg["vocab_size"], 1, seq, rank=0, eos_token_id=cfg["eos_token_id"])
    ctx = {"bf16": lambda: nullcontext(), "fp8": lambda: fp8_autocast(engine)}
    out = {m: {"step_ms": float("inf"), "peak_hbm_gb": 0.0} for m in ctx}
    fp8_losses = []
    for r in range(rounds + 1):  # round 0 warms both modes up
        for mode, fc in ctx.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                loss, _ = train_step(model, opt, None, train_dataloader=data, gradient_clipping=1.0, forward_context=fc,
                                     return_tensors=True)
                if mode == "fp8":
                    fp8_losses.append(loss.detach().reshape(()))
            e1.record()
            torch.cuda.synchronize()
            if r == 0:
                continue
            ms = e0.elapsed_time(e1) / steps
            o = out[mode]
            o["step_ms"] = min(o["step_ms"], round(ms, 2))
            o["tokens_per_s"] = round(seq / (o["step_ms"] / 1e3), 1)
            o["peak_hbm_gb"] = round(max(o["peak_hbm_gb"], torch.cuda.max_memory_allocated(dev) / 1e9), 2)
            o["loss"] = float(loss)
    out["fp8_speedup"] = round(out["bf16"]["step_ms"] / out["fp8"]["step_ms"], 3)
    if dump:  # the FP8 mode ran last
        bench.dump_outputs(os.path.join(dump, "train"), engine, fp8_losses, 0)
    del model, opt, wrapper, engine
    torch.cuda.empty_cache()
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--train-steps", type=int, default=5, help="steps per block of the end-to-end comparison (0: skip it)")
    ap.add_argument("--dump", default=None, metavar="DIR", help="write what the FP8 GEMMs compute under DIR (see above)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8 needs a CUDA device")
    T = a.tokens
    g = torch.Generator(device="cuda").manual_seed(0)
    one = torch.ones(1, dtype=torch.float32, device="cuda")
    amax = torch.zeros(1, dtype=torch.float32, device="cuda")
    res = {"tokens": T, **_card()}
    if a.train_steps:
        res["train_step_c2"] = train_steps(a.train_steps, a.rounds, a.dump)
    if a.dump:
        dump_grid(a.dump)
    res["shapes"] = {}
    for name, (N, Kd) in c2_block_shapes().items():
        x = torch.randn(T, Kd, device="cuda", generator=g).to(torch.bfloat16)
        w = (torch.randn(N, Kd, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
        dy = (torch.randn(T, N, device="cuda", generator=g) * 1e-3).to(torch.bfloat16)
        dw = torch.zeros(N, Kd, dtype=torch.float32, device="cuda")
        xq, xt = K.fp8_cast(x, K.E4M3, one, transpose=True)
        wq, _ = K.fp8_cast(w, K.E4M3, one)
        dyq, dyt = K.fp8_cast(dy, K.E5M2, one, transpose=True)
        y = torch.empty(T, N, dtype=torch.bfloat16, device="cuda")
        jobs = {
            "bf16_fwd": lambda: K.gemm(x, w, out=y),
            "fp8_fwd": lambda: K.gemm_fp8(xq, K.E4M3, one, wq, K.E4M3, one, out=y),
            "bf16_wgrad": lambda: K.gemm(dy, x, a_mn=True, b_mn=True, out=dw, c=dw, beta=1.0),
            "fp8_wgrad": lambda: K.gemm_fp8(dyt, K.E5M2, one, xt, K.E4M3, one, out=dw, c=dw, beta=1.0, split_accumulate=True),
            "casts": lambda: (K.fp8_cast(x, K.E4M3, one, amax=amax, out=xq), K.fp8_cast(w, K.E4M3, one, amax=amax, out=wq),
                              K.fp8_cast(dy, K.E5M2, one, transpose=True, amax=amax, out=dyq, out_t=dyt),
                              K.fp8_cast(w, K.E4M3, one, plain=False, transpose=True),
                              K.fp8_cast(x, K.E4M3, one, plain=False, transpose=True, out_t=xt)),
        }
        for fn in jobs.values():  # warm-up of every shape in the timed window
            fn()
        torch.cuda.synchronize()
        best = {k: float("inf") for k in jobs}
        for _ in range(a.rounds):  # alternate the variants; keep the best round of each
            for k, fn in jobs.items():
                best[k] = min(best[k], _time(fn, a.iters))
        flops = 2.0 * T * N * Kd
        r = {k + "_ms": round(v * 1e3, 4) for k, v in best.items()}
        for k in ("bf16_fwd", "fp8_fwd", "bf16_wgrad", "fp8_wgrad"):
            r[k + "_tflops"] = round(flops / best[k] / 1e12, 1)
        r["fwd_speedup"] = round(best["bf16_fwd"] / best["fp8_fwd"], 3)
        r["wgrad_speedup"] = round(best["bf16_wgrad"] / best["fp8_wgrad"], 3)
        if a.dump:
            dw8 = torch.randn(N, Kd, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
            K.gemm_fp8(dyt, K.E5M2, one, xt, K.E4M3, one, out=dw8, c=dw8, beta=1.0, split_accumulate=True)
            _save(a.dump, f"{name}_fp8_fwd", K.gemm_fp8(xq, K.E4M3, one, wq, K.E4M3, one))
            _save(a.dump, f"{name}_fp8_wgrad", dw8)
        res["shapes"][name] = {"M": T, "N": N, "K": Kd, **r}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
