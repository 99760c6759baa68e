"""Kernel time of every MLP activation, forward and backward (with the fused c_fc bias gradient), in every form.

    python tools/bench_activations.py [--T 4096] [--F 10240] [--iters 50] [--json out.json]

The default shape is C2's MLP (bench.py: T = 4096 tokens, n_inner 10240; GLU input [T, 2F]).  Each entry reports the
median CUDA-event time of one launch, the bytes the kernel must move (bf16: x and y forward; dy, x and dx backward, plus
the fp32 bias gradient) over that time, the share of 3.35 TB/s (H100 SXM HBM3 data sheet), and the time relative to the
SwiGLU (GLU forms) or tanh-GELU (plain form) kernel of the same run.  The card's name and power limit are read in the
same run.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dolomite_engine_b200 import activations as A  # noqa: E402
from dolomite_engine_b200 import kernels as K  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12
NAMES = ["celu", "elu", "gelu", "gelu_tanh", "selu", "hardshrink", "hardsigmoid", "hardswish", "hardtanh", "laplace",
         "leaky_relu", "log_sigmoid", "mish", "relu", "relu2", "relu6", "sigmoid", "silu", "softplus", "softshrink",
         "softsign", "tanh", "tanhshrink"]
FORMS = {A.PLAIN: "plain", A.GLU: "glu", A.SIGMOID_GLU: "sigmoid_glu"}


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = (s.strip() for s in out[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def time_ms(fn, iters: int) -> float:
    for _ in range(3):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    t = sorted(a.elapsed_time(b) for a, b in ev)
    return t[len(t) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=4096)
    ap.add_argument("--F", type=int, default=10240)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_activations needs a CUDA device")
    T, F = args.T, args.F
    g = torch.Generator(device="cuda").manual_seed(0)
    x2 = (torch.randn(T, 2 * F, device="cuda", generator=g) * 2).bfloat16()
    x1 = x2[:, :F].contiguous()
    dy = torch.randn(T, F, device="cuda", generator=g).bfloat16()
    y = torch.empty(T, F, device="cuda", dtype=torch.bfloat16)
    dx2, dx1 = torch.empty_like(x2), torch.empty_like(x1)
    db2, db1 = torch.zeros(2 * F, device="cuda"), torch.zeros(F, device="cuda")
    rows = []
    for act_id, name in enumerate(NAMES):
        for form in ((A.PLAIN, A.GLU, A.SIGMOID_GLU) if act_id == A.SIGMOID else (A.PLAIN, A.GLU)):
            x, dx, db = (x1, dx1, db1) if form == A.PLAIN else (x2, dx2, db2)
            fwd = time_ms(lambda: K.act_fwd(x, act_id, form, out=y), args.iters)
            bwd = time_ms(lambda: K.act_bwd(dy, x, act_id, form, out=dx, bias_grad_accum=db), args.iters)
            fwd_bytes = 2 * (x.numel() + y.numel())
            bwd_bytes = 2 * (dy.numel() + 2 * x.numel()) + 8 * db.numel()
            rows.append({"act": name, "form": FORMS[form], "fwd_ms": fwd, "bwd_ms": bwd,
                         "fwd_TBps": fwd_bytes / fwd / 1e9, "bwd_TBps": bwd_bytes / bwd / 1e9,
                         "fwd_peak_share": fwd_bytes / fwd / 1e-3 / PEAK_BYTES_PER_S,
                         "bwd_peak_share": bwd_bytes / bwd / 1e-3 / PEAK_BYTES_PER_S})
    base = {"plain": next(r for r in rows if r["act"] == "gelu_tanh" and r["form"] == "plain"),
            "glu": next(r for r in rows if r["act"] == "silu" and r["form"] == "glu")}
    base["sigmoid_glu"] = base["glu"]
    for r in rows:
        b = base[r["form"]]
        r["fwd_vs_base"] = r["fwd_ms"] / b["fwd_ms"]
        r["bwd_vs_base"] = r["bwd_ms"] / b["bwd_ms"]
    result = {"card": card(), "T": T, "F": F, "rows": rows}
    print(f"{result['card']}  T={T} F={F}")
    print(f"{'act':12s} {'form':11s} {'fwd ms':>8s} {'TB/s':>6s} {'x base':>6s} {'bwd ms':>8s} {'TB/s':>6s} {'x base':>6s}")
    for r in rows:
        print(f"{r['act']:12s} {r['form']:11s} {r['fwd_ms']:8.4f} {r['fwd_TBps']:6.2f} {r['fwd_vs_base']:6.2f} "
              f"{r['bwd_ms']:8.4f} {r['bwd_TBps']:6.2f} {r['bwd_vs_base']:6.2f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
