"""Every bf16 GEMM launch of a C2 training step at both output tile widths (128 x 128 and 128 x 256) and under the
automatic choice, timed with CUDA events.

    python tools/bench_gemm.py [--window-ms 25] [--rounds 5]

The shapes come from bench.model_config("c2") and the flagship workload's sequence length: the forward and the dgrad of
the four block linears and of the LM head, the block's four weight gradients in one gemm_bf16_wgrad_multi launch, and
the head's weight gradient.  Each launch is warmed up at every width, then timed in rounds that alternate the widths,
each round a window of back-to-back launches of at least --window-ms; the best round of each width is kept.  Per shape
it reports TFLOP/s at each width, the width the automatic choice takes, and c_256 / c_128, the time of one 128 x 256
tile over one 128 x 128 tile: time / ceil(tiles / SMs) at each width.  The median of that ratio over the shapes is the
constant of the automatic choice (TILE256_COST in csrc/gemm.cu).

The launches carry the engine's epilogue operands: a bias on every block linear's forward, the residual as C on the
two c_proj forwards, and weight gradients that overwrite their output (one micro-step per optimizer step).

A K sweep times the forward of a 4096 x 2560 output at K = 2560 .. 20480 at both widths and fits the time of one tile,
t = n_kb * a + f (n_kb 64-deep k-blocks): `a` is the mainloop's cost per k-block and `f` the fixed cost per tile
(epilogue, pipeline fill and drain).  Prints one JSON line with the card name and power limit.
"""

from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dolomite_engine_b200 import kernels as K  # noqa: E402


def _card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the numbers are still reported; the card line says why it is missing
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unavailable ({e})"}


def c2_shapes() -> tuple[int, int, dict, list]:
    """tokens, layers, {linear: (out_features, in_features)} of a C2 block and the LM head"""
    import bench

    cfg = bench.model_config("c2")
    T = bench.WORKLOADS["c2"]["seq"] * bench.WORKLOADS["c2"]["mbs"]
    H, F, nh = cfg["n_embd"], cfg["n_inner"], cfg["n_head"]
    kv = {"mha": nh, "mqa": 1}.get(cfg["attention_head_type"], cfg.get("num_key_value_heads") or nh)
    fc = 2 * F if cfg["activation_function"].endswith("glu") else F
    block = {"c_attn": (H + 2 * kv * (H // nh), H), "attn.c_proj": (H, H), "c_fc": (fc, H), "mlp.c_proj": (H, F)}
    return T, cfg["n_layer"], block, [("head", (cfg["vocab_size"], H))]


def _bf16(*shape, g, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(torch.bfloat16)


def _launches(T: int, block: dict, head: list, g) -> list[dict]:
    """(name, [(M, N) outputs], FLOPs, fn) of every bf16 GEMM launch of one C2 step"""
    out = []
    for name, (N, Kd) in list(block.items()) + head:
        x, w, dy = _bf16(T, Kd, g=g), _bf16(N, Kd, g=g, scale=0.02), _bf16(T, N, g=g, scale=1e-3)
        y, dx = torch.empty(T, N, dtype=torch.bfloat16, device="cuda"), torch.empty(T, Kd, dtype=torch.bfloat16, device="cuda")
        bias = None if name == "head" else _bf16(N, g=g, scale=0.02)
        res = _bf16(T, N, g=g) if name.endswith("c_proj") else None  # the residual stream, added by the c_proj forwards
        out.append(dict(name=f"{name}.fwd", outputs=[(T, N)], flops=2.0 * T * N * Kd,
                        fn=lambda x=x, w=w, y=y, b=bias, c=res: K.gemm(x, w, out=y, bias=b, c=c, beta=1.0)))
        out.append(dict(name=f"{name}.dgrad", outputs=[(T, Kd)], flops=2.0 * T * N * Kd,
                        fn=lambda dy=dy, w=w, dx=dx: K.gemm(dy, w, b_mn=True, out=dx)))
        if name == "head":
            dw = torch.zeros(N, Kd, dtype=torch.float32, device="cuda")
            out.append(dict(name="head.wgrad", outputs=[(N, Kd)], flops=2.0 * T * N * Kd,
                            fn=lambda dy=dy, x=x, dw=dw: K.gemm(dy, x, a_mn=True, b_mn=True, out=dw)))
    probs, outputs, flops = [], [], 0.0
    for N, Kd in block.values():
        probs.append((_bf16(T, N, g=g, scale=1e-3), _bf16(T, Kd, g=g), torch.zeros(N, Kd, dtype=torch.float32, device="cuda"),
                      1.0, False))
        outputs.append((N, Kd))
        flops += 2.0 * T * N * Kd
    out.append(dict(name="block.wgrad_multi", outputs=outputs, flops=flops, fn=lambda probs=probs: K.gemm_wgrad_multi(probs)))
    return out


def _time(fn, iters: int) -> float:
    """seconds per call over `iters` back-to-back calls"""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e-3


def k_sweep(T: int, N: int, g, window_ms: float, rounds: int, workers: int) -> dict:
    """forward of a T x N output at K = 2560 .. 20480 at both widths; least-squares fit of the per-tile time
    t = n_kb * a + f, where t = launch time / ceil(tiles / workers)"""
    res = {}
    for width in (128, 256):
        K.set_option("gemm_tile_n", width)
        waves = math.ceil(math.ceil(T / 128) * math.ceil(N / width) / workers)
        pts = []
        for Kd in (2560, 5120, 10240, 20480):
            x, w = _bf16(T, Kd, g=g), _bf16(N, Kd, g=g, scale=0.02)
            y = torch.empty(T, N, dtype=torch.bfloat16, device="cuda")
            fn = lambda x=x, w=w, y=y: K.gemm(x, w, out=y)  # noqa: E731
            fn()
            torch.cuda.synchronize()
            iters = max(5, math.ceil(window_ms * 1e-3 / _time(fn, 3)))
            best = min(_time(fn, iters) for _ in range(rounds))
            pts.append((Kd // 64, best / waves, 2.0 * T * N * Kd / best / 1e12))
        n = len(pts)
        mx, my = sum(p[0] for p in pts) / n, sum(p[1] for p in pts) / n
        a = sum((p[0] - mx) * (p[1] - my) for p in pts) / sum((p[0] - mx) ** 2 for p in pts)
        f = my - a * mx
        res[str(width)] = {"waves": waves, "tile_us": {p[0] * 64: round(p[1] * 1e6, 3) for p in pts},
                           "tflops": {p[0] * 64: round(p[2], 1) for p in pts},
                           "a_us_per_kblock": round(a * 1e6, 4), "f_us_per_tile": round(f * 1e6, 3)}
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-ms", type=float, default=25.0, help="least length of one timed window of a launch")
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm needs a CUDA device")
    g = torch.Generator(device="cuda").manual_seed(0)
    T, layers, block, head = c2_shapes()
    launches = _launches(T, block, head, g)
    workers = torch.cuda.get_device_properties(0).multi_processor_count - K.get_option("gemm_sm_margin")
    widths = {"128": 128, "256": 256, "auto": 0}
    default = K.get_option("gemm_tile_n")
    res = {"tokens": T, **_card(), "workers": workers, "shapes": {}}
    ratios = []
    totals = {k: 0.0 for k in widths}
    try:
        for L in launches:
            for w in widths.values():  # warm-up of every width
                K.set_option("gemm_tile_n", w)
                L["fn"]()
            torch.cuda.synchronize()
            iters = max(5, math.ceil(a.window_ms * 1e-3 / _time(L["fn"], 3)))
            best = {k: float("inf") for k in widths}
            for _ in range(a.rounds):
                for k, w in widths.items():
                    K.set_option("gemm_tile_n", w)
                    best[k] = min(best[k], _time(L["fn"], iters))
            K.set_option("gemm_tile_n", 0)
            auto_n, cost = K.gemm_tile_n(L["outputs"])
            waves = {n: math.ceil(sum(math.ceil(m / 128) * math.ceil(c / n) for m, c in L["outputs"]) / workers)
                     for n in (128, 256)}
            ratio = (best["256"] / waves[256]) / (best["128"] / waves[128])
            ratios.append(ratio)
            for k in widths:  # the block's launches run once per layer
                totals[k] += best[k] * (1 if L["name"].startswith("head") else layers)
            r = {f"{k}_ms": round(v * 1e3, 4) for k, v in best.items()}
            r.update({f"{k}_tflops": round(L["flops"] / v / 1e12, 1) for k, v in best.items()})
            r.update(outputs=L["outputs"], auto_tile_n=auto_n, waves_128=waves[128], waves_256=waves[256],
                     tile_cost_256_over_128=round(ratio, 3), auto_over_128=round(best["auto"] / best["128"], 4))
            res["shapes"][L["name"]] = r
        res["k_sweep_4096x2560"] = k_sweep(T, 2560, g, a.window_ms, a.rounds, workers)
    finally:
        K.set_option("gemm_tile_n", default)
    res["tile_cost_256_over_128_median"] = round(statistics.median(ratios), 3)
    res["tile_cost_256_over_128_in_library"] = round(K.gemm_tile_n([(T, T)])[1], 3)
    res["gemm_ms_per_step"] = {k: round(v * 1e3, 2) for k, v in totals.items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
