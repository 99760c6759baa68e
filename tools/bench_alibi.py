"""Time the attention kernels with and without ALiBi at C2's attention shape (T = 4096, 32 heads, head dim 80): one
document of 4096 and eight of 512; forward, backward (dK/dV + dQ, one call) and decode.  Also head dim 128 (16 heads,
one document of 4096), whose dK/dV kernel keeps a few registers in local memory.  Median of 50 launches each, CUDA
events.  Prints one JSON line per measurement and the GPU's name and power limit.

    python tools/bench_alibi.py
"""

from __future__ import annotations

import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dolomite_engine_b200 import kernels as K  # noqa: E402
from dolomite_engine_b200.alibi import alibi_slopes  # noqa: E402

T, NH, HD, N = 4096, 32, 80, 50


def median_ms(fn) -> float:
    for _ in range(5):
        fn()
    times = []
    for _ in range(N):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}))
    g = torch.Generator(device="cuda").manual_seed(0)
    for nh, hd, docs_list in ((NH, HD, (1, 8)), (16, 128, (1,))):
        attention(g, nh, hd, docs_list)
    decode(g)


def attention(g, NH, HD, docs_list):
    qkv = torch.randn(T, NH * 3 * HD, device="cuda", generator=g).bfloat16()
    dout = torch.randn(T, NH * HD, device="cuda", generator=g).bfloat16()
    slopes = alibi_slopes(NH).cuda()
    scale = HD**-0.5
    for docs in docs_list:
        cu = torch.arange(0, T + 1, T // docs, dtype=torch.int32, device="cuda")
        L = T // docs
        res = {"heads": NH, "head_dim": HD, "docs": docs}
        for name, sl in (("plain", None), ("alibi", slopes)):
            out, lse = K.attn_varlen_fwd(qkv, cu, L, NH, 1, HD, scale, alibi_slopes=sl)
            res[f"fwd_{name}_ms"] = median_ms(lambda: K.attn_varlen_fwd(qkv, cu, L, NH, 1, HD, scale, alibi_slopes=sl))
            res[f"bwd_{name}_ms"] = median_ms(
                lambda: K.attn_varlen_bwd(dout, qkv, out, lse, cu, L, NH, 1, HD, scale, alibi_slopes=sl))
        for d in ("fwd", "bwd"):
            res[f"{d}_ratio"] = round(res[f"{d}_alibi_ms"] / res[f"{d}_plain_ms"], 3)
        print(json.dumps(res))


def decode(g):
    """8 sequences of 4096 cached positions, one new token each, C2's heads"""
    slopes = alibi_slopes(NH).cuda()
    scale = HD**-0.5
    B = 8
    kc = torch.randn(B, T, NH * HD, device="cuda", generator=g).bfloat16()
    vc = torch.randn(B, T, NH * HD, device="cuda", generator=g).bfloat16()
    q1 = torch.randn(B, NH * 3 * HD, device="cuda", generator=g).bfloat16()
    lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
    res = {"decode_batch": B, "cache": T}
    for name, sl in (("plain", None), ("alibi", slopes)):
        res[f"decode_{name}_ms"] = median_ms(lambda: K.attn_decode(q1, kc, vc, lens, NH, 1, HD, scale, alibi_slopes=sl))
    res["decode_ratio"] = round(res["decode_alibi_ms"] / res["decode_plain_ms"], 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
