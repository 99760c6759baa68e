"""Cost of MoE expert biases: one MoE layer's forward + backward with and without biases, CUDA events.

    python tools/bench_moe_bias.py [--tokens 8192] [--iters 30] [--dump-dir DIR] [--bias-free-only]

Shapes: those of tools/bench_moe_aux.py (H = 2048, n_inner = 4096, SwiGLU; E = 8, top-2 and E = 64, top-8).  "with" is
the layer of a model with add_bias=True (biases drawn with std 0.1): the biased grouped GEMM entry point in the forward,
the per-expert bias-gradient reductions in the backward; "without" is the same layer with add_bias=False.  The two modes
alternate, each timed over `iters` forward + backward pairs after a warm-up; the median of 5 rounds is reported.  Prints
one JSON line per shape, with the card name and power limit.

--dump-dir writes the bias-free layer's output, input gradient and parameter gradients (one forward + backward from a
fresh zero_grad, seeded inputs) as .npy files, so that builds can be compared byte for byte.  --bias-free-only skips the
biased layer (and the timing).
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dolomite_engine_b200 import moe  # noqa: E402


def _card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unavailable ({e})"}


def _layer(E: int, k: int, bias: bool):
    from dolomite_engine_b200.hf_models import MoEDolomiteConfig, MoEDolomiteForCausalLM

    cfg = MoEDolomiteConfig(vocab_size=256, n_positions=8192, n_embd=2048, n_layer=1, n_head=16, n_inner=4096,
                            num_experts=E, num_experts_per_tok=k, attention_head_type="mha", add_bias=bias,
                            position_embedding_type="rope", normalization_function="rmsnorm", activation_function="swiglu",
                            resid_pdrop=0, embd_pdrop=0, attn_pdrop=0)
    eng = MoEDolomiteForCausalLM(cfg, seed=0).engine
    if bias:
        g = torch.Generator(device="cuda").manual_seed(1)
        for name in ("transformer.h.0.mlp.c_fc.bias", "transformer.h.0.mlp.c_proj.bias"):
            v = eng.units[1].views[name]
            v.copy_(torch.randn(v.shape, device="cuda", generator=g) * 0.1)
    return eng


def _step(eng, x, dh):
    u, p = eng.units[1], "transformer.h.0."
    out, saved = moe.forward(eng, u, p, x, x, 1.0)
    return out, moe.backward(eng, u, p, x, dh, 1.0, saved)


def _dump(eng, x, dh, path: str) -> None:
    os.makedirs(path, exist_ok=True)
    eng.zero_grad()
    out, dx = _step(eng, x, dh)
    torch.cuda.synchronize()
    arrays = {"out": out, "dx": dx}
    arrays.update({n.replace("transformer.h.0.", "grad_"): eng.units[1].gviews[n] for n, _, _ in eng.named_views()
                   if n.startswith("transformer.h.0.mlp.")})
    for n, t in arrays.items():
        a = t.detach().cpu()
        a = a.view(torch.int16).numpy() if a.dtype == torch.bfloat16 else a.numpy()
        np.save(os.path.join(path, n + ".npy"), a)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--dump-dir", default=None)
    ap.add_argument("--bias-free-only", action="store_true")
    a = ap.parse_args()
    card = _card()
    for E, k in ((8, 2), (64, 8)):
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randn(a.tokens, 2048, device="cuda", generator=g).to(torch.bfloat16)
        dh = (torch.randn(a.tokens, 2048, device="cuda", generator=g) * 1e-2).to(torch.bfloat16)
        engs = {False: _layer(E, k, False)}
        if a.dump_dir:
            _dump(engs[False], x, dh, os.path.join(a.dump_dir, f"e{E}_k{k}"))
        if a.bias_free_only:
            continue
        engs[True] = _layer(E, k, True)
        for mode in (False, True, False, True):
            _step(engs[mode], x, dh)
        torch.cuda.synchronize()
        times = {False: [], True: []}
        for _ in range(5):
            for mode in (False, True):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.iters):
                    _step(engs[mode], x, dh)
                e1.record()
                e1.synchronize()
                times[mode].append(e0.elapsed_time(e1) / a.iters)
        med = {m: sorted(v)[len(v) // 2] for m, v in times.items()}
        print(json.dumps({"shape": {"tokens": a.tokens, "n_embd": 2048, "n_inner": 4096, "experts": E, "top_k": k},
                          "layer_fwd_bwd_ms_without": round(med[False], 4), "layer_fwd_bwd_ms_with": round(med[True], 4),
                          "overhead_pct": round(100 * (med[True] / med[False] - 1), 2),
                          "spread_ms": {str(m): [round(min(v), 4), round(max(v), 4)] for m, v in times.items()},
                          **card}), flush=True)
        del engs


if __name__ == "__main__":
    main()
