"""Attention backward on one GPU: time of the backward call (K.attn_varlen_bwd = Delta, dK/dV and dQ kernels) per shape,
per-kernel times from torch.profiler, and byte dumps of dqkv for comparing two builds.

    python tools/bench_attention.py                      # timings (median of 50 launches after warm-up)
    python tools/bench_attention.py --profile            # per-kernel device times (one torch.profiler pass)
    python tools/bench_attention.py --dump DIR           # dqkv of a fixed seeded grid of configurations, one file each

TFLOP/s is algorithmic: 5 causal matmuls (S, dP, dV, dK, dQ) of 2 * S^2/2 * head_dim flops per head and document.
"""

from __future__ import annotations

import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# name: (document lengths, kv groups, q heads per group, head_dim, alibi, dropout p)
SHAPES = {
    "c2": ([4096], 32, 1, 80, False, 0.0),
    "c2_8x512": ([512] * 8, 32, 1, 80, False, 0.0),
    "hd128": ([4096], 16, 1, 128, False, 0.0),
    "gqa_8192": ([3000, 2048, 1900, 1244], 8, 4, 128, False, 0.0),
    "c2_alibi": ([4096], 32, 1, 80, True, 0.0),
    "c2_dropout": ([4096], 32, 1, 80, False, 0.1),
}

# --dump grid: every head dim, MHA / GQA / MQA, ALiBi, dropout, ragged documents around the 64 / 128 boundaries, an empty one
DUMP_GRID = [
    (hd, lens, ng, g, alibi, p)
    for hd in (16, 32, 64, 80, 96, 128)
    for (lens, ng, g) in (([63, 64, 65, 0, 127, 128, 129, 300], 2, 1), ([191, 0, 257, 700], 2, 2), ([2100], 1, 4))
    for (alibi, p) in ((False, 0.0), (True, 0.0), (False, 0.1))
]


def flops(lens, n_heads, hd):
    return 5 * 2 * sum(L * L / 2 for L in lens) * hd * n_heads


def make(lens, ng, g, hd, alibi, p, seed=0):
    import numpy as np
    import torch

    from dolomite_engine_b200 import kernels as K
    from dolomite_engine_b200.alibi import alibi_slopes

    gen = torch.Generator(device="cuda").manual_seed(seed)
    T = sum(lens)
    qkv = torch.randn(T, ng * (g + 2) * hd, device="cuda", generator=gen).bfloat16()
    dout = torch.randn(T, ng * g * hd, device="cuda", generator=gen).bfloat16()
    cu = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)).cuda()
    slopes = alibi_slopes(ng * g).cuda() if alibi else None
    keys = (1234, 5678)
    scale = 1.0 / math.sqrt(hd)
    out, lse = K.attn_varlen_fwd(qkv, cu, max(lens), ng, g, hd, scale, dropout_p=p, dropout_keys=keys, alibi_slopes=slopes)
    dqkv = torch.empty_like(qkv)

    def bwd():
        K.attn_varlen_bwd(dout, qkv, out, lse, cu, max(lens), ng, g, hd, scale, dqkv=dqkv, dropout_p=p, dropout_keys=keys,
                          alibi_slopes=slopes)

    return bwd, dqkv


def time_call(fn, iters=50, warmup=10):
    import torch

    for _ in range(warmup):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    t = sorted(a.elapsed_time(b) for a, b in ev)
    return t[len(t) // 2]


def gpu_info():
    import subprocess

    import torch

    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # informational only
        pl = f"unknown ({type(e).__name__})"
    return {"gpu": name, "power_limit, max_sm_clock": pl}


def flash_attn_c2():
    """flash_attn's varlen backward at the C2 shape, if the package imports (informational yardstick)"""
    try:
        import flash_attn  # noqa: F401
        from flash_attn import flash_attn_varlen_func
    except Exception:
        return None
    import torch

    S, nh, hd = 4096, 32, 80
    q, k, v = (torch.randn(S, nh, hd, device="cuda", dtype=torch.bfloat16, requires_grad=True) for _ in range(3))
    cu = torch.tensor([0, S], dtype=torch.int32, device="cuda")
    o = flash_attn_varlen_func(q, k, v, cu, cu, S, S, causal=True)
    g = torch.randn_like(o)
    ms = time_call(lambda: torch.autograd.grad(o, (q, k, v), g, retain_graph=True))
    return {"ms": ms, "tflops": flops([S], nh, hd) / ms / 1e9}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default=",".join(SHAPES), help="comma-separated subset of " + ",".join(SHAPES))
    ap.add_argument("--profile", action="store_true", help="per-kernel device times from one torch.profiler pass")
    ap.add_argument("--dump", metavar="DIR", help="write dqkv of the fixed seeded grid to DIR and exit")
    args = ap.parse_args()

    import torch

    assert torch.cuda.is_available(), "bench_attention needs a GPU"
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
        for i, (hd, lens, ng, g, alibi, p) in enumerate(DUMP_GRID):
            bwd, dqkv = make(lens, ng, g, hd, alibi, p, seed=i)
            bwd()
            torch.cuda.synchronize()
            name = f"{i:03d}_hd{hd}_ng{ng}_g{g}_alibi{int(alibi)}_p{p}.bin"
            dqkv.view(torch.int16).cpu().numpy().tofile(os.path.join(args.dump, name))
        print(json.dumps({"dumped": len(DUMP_GRID), "dir": args.dump}))
        return

    res = {"info": gpu_info(), "shapes": {}}
    for name in args.shapes.split(","):
        lens, ng, g, hd, alibi, p = SHAPES[name]
        bwd, _ = make(lens, ng, g, hd, alibi, p)
        if args.profile:
            from torch.profiler import ProfilerActivity, profile

            for _ in range(5):
                bwd()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    bwd()
                torch.cuda.synchronize()
            per = {}
            for e in prof.key_averages():
                if e.device_type.name == "CUDA" and "attn" in e.key:
                    per[e.key[:60]] = round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 10 / 1e3, 4)
            res["shapes"][name] = {"kernel_ms": per}
        else:
            ms = time_call(bwd)
            res["shapes"][name] = {"ms": round(ms, 4), "tflops": round(flops(lens, ng * g, hd) / ms / 1e9, 1)}
    if not args.profile:
        fa = flash_attn_c2()
        if fa:
            res["flash_attn_c2"] = fa
    print(json.dumps(res))


if __name__ == "__main__":
    main()
