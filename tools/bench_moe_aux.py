"""Cost of the MoE load-balancing loss: one MoE layer's forward + backward with and without the term, CUDA events.

    python tools/bench_moe_aux.py [--tokens 8192] [--iters 30]

Shapes: the C4 MoE layer (configs/c4_moe_8x_top2.yml: H = 2048, n_inner = 4096, SwiGLU, E = 8, top-2) and the same widths
at E = 64, top-8.  "with" adds what forward(router_aux=True) adds per layer -- moe_aux_stats in the forward, the
moe_router_bwd_aux router backward -- plus the one finalize launch of a forward; "without" is the plain layer.  The two
modes alternate, each timed over `iters` forward + backward pairs after a warm-up; the median of 5 rounds is reported.
Prints one JSON line per shape, with the card name and power limit.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dolomite_engine_b200 import kernels as K  # noqa: E402
from dolomite_engine_b200 import moe  # noqa: E402


def _card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unavailable ({e})"}


def _layer(E: int, k: int):
    from dolomite_engine_b200.hf_models import MoEDolomiteConfig, MoEDolomiteForCausalLM

    cfg = MoEDolomiteConfig(vocab_size=256, n_positions=8192, n_embd=2048, n_layer=1, n_head=16, n_inner=4096,
                            num_experts=E, num_experts_per_tok=k, attention_head_type="mha", add_bias=False,
                            position_embedding_type="rope", normalization_function="rmsnorm", activation_function="swiglu",
                            resid_pdrop=0, embd_pdrop=0, attn_pdrop=0)
    return MoEDolomiteForCausalLM(cfg, seed=0).engine


def _step(eng, x, dh, with_aux: bool) -> None:
    u, p = eng.units[1], "transformer.h.0."
    T = x.shape[0]
    if with_aux:
        eng._aux_fwd = (K.moe_aux_acc(eng.cfg.num_experts, x.device), T, [])
    out, saved = moe.forward(eng, u, p, x, x, 1.0)
    if with_aux:
        acc = eng._aux_fwd[0]
        eng._aux_fwd = None
        _, c = K.moe_aux_finalize(acc, T, 0.01)
        eng._aux_bwd = (c, torch.full((1,), 0.01, device=x.device), T)
    moe.backward(eng, u, p, x, dh, 1.0, saved)
    eng._aux_bwd = None


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=30)
    a = ap.parse_args()
    card = _card()
    for E, k in ((8, 2), (64, 8)):
        eng = _layer(E, k)
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randn(a.tokens, 2048, device="cuda", generator=g).to(torch.bfloat16)
        dh = (torch.randn(a.tokens, 2048, device="cuda", generator=g) * 1e-2).to(torch.bfloat16)
        for mode in (False, True, False, True):
            _step(eng, x, dh, mode)
        torch.cuda.synchronize()
        times = {False: [], True: []}
        for _ in range(5):
            for mode in (False, True):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.iters):
                    _step(eng, x, dh, mode)
                e1.record()
                e1.synchronize()
                times[mode].append(e0.elapsed_time(e1) / a.iters)
        med = {m: sorted(v)[len(v) // 2] for m, v in times.items()}
        print(json.dumps({"shape": {"tokens": a.tokens, "n_embd": 2048, "n_inner": 4096, "experts": E, "top_k": k},
                          "layer_fwd_bwd_ms_without": round(med[False], 4), "layer_fwd_bwd_ms_with": round(med[True], 4),
                          "overhead_pct": round(100 * (med[True] / med[False] - 1), 2),
                          "spread_ms": {str(m): [round(min(v), 4), round(max(v), 4)] for m, v in times.items()},
                          **card}), flush=True)
        del eng


if __name__ == "__main__":
    main()
