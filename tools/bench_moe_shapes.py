"""Cost of MoE shapes off multiples of 64 and 8: one MoE layer's forward + backward, CUDA events.

    python tools/bench_moe_shapes.py [--tokens 16384] [--iters 20] [--rounds 5] [--other-lib PATH]

Every figure is one MoE layer (moe.forward + moe.backward, SwiGLU, H 2048, no bias) at `tokens` tokens, the token count of
one C4 micro-batch (8 x 2048).  Each line compares two variants that alternate, each timed over `iters` forward + backward
pairs after a warm-up, for `rounds` rounds; the median and the spread of the rounds are printed, with the card's name
and power limit, one JSON line per comparison:

  n_inner 1376 vs 1408   an n_inner off a multiple of 64 against its on-64 neighbour (E 8, top-2)
  E 6 vs E 8             an expert count off a multiple of 8 against its neighbour (n_inner 4096, top-2)

--other-lib PATH also loads a libdolomite_b200.so built from another tree (for example the parent commit) into the same
process and compares the C4 layer (n_inner 4096; E 8 / top-2 and E 64 / top-8) run on each library: the time of both,
and whether the layer's output, input gradient and every parameter gradient are byte-identical (one forward + backward
from a fresh zero_grad on the same seeded inputs and weights).
"""

from __future__ import annotations

import argparse
import hashlib
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dolomite_engine_b200 import _lib, moe  # noqa: E402

H = 2048


def _card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unavailable ({e})"}


def _layer(E: int, k: int, F: int):
    from dolomite_engine_b200.hf_models import MoEDolomiteConfig, MoEDolomiteForCausalLM

    cfg = MoEDolomiteConfig(vocab_size=256, n_positions=8192, n_embd=H, n_layer=1, n_head=16, n_inner=F, num_experts=E,
                            num_experts_per_tok=k, attention_head_type="mha", add_bias=False,
                            position_embedding_type="rope", normalization_function="rmsnorm", activation_function="swiglu",
                            resid_pdrop=0, embd_pdrop=0, attn_pdrop=0)
    return MoEDolomiteForCausalLM(cfg, seed=0).engine


def _step(eng, x, dh):
    u, p = eng.units[1], "transformer.h.0."
    out, saved = moe.forward(eng, u, p, x, x, 1.0)
    return out, moe.backward(eng, u, p, x, dh, 1.0, saved)


def _digest(eng, x, dh) -> str:
    eng.zero_grad()
    out, dx = _step(eng, x, dh)
    torch.cuda.synchronize()
    h = hashlib.sha256()
    for t in [out, dx] + [eng.units[1].gviews[n] for n, _, _ in eng.named_views() if n.startswith("transformer.h.0.mlp.")]:
        h.update(t.detach().contiguous().view(torch.uint8).cpu().numpy().tobytes())
    return h.hexdigest()


def _inputs(tokens: int):
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(tokens, H, device="cuda", generator=g).to(torch.bfloat16)
    dh = (torch.randn(tokens, H, device="cuda", generator=g) * 1e-2).to(torch.bfloat16)
    return x, dh


def _time(variants: dict, x, dh, iters: int, rounds: int) -> dict:
    """variants: name -> (library handle, engine); alternated round by round"""
    for _ in range(2):
        for lib, eng in variants.values():
            _lib._lib = lib
            _step(eng, x, dh)
    torch.cuda.synchronize()
    times = {n: [] for n in variants}
    for _ in range(rounds):
        for n, (lib, eng) in variants.items():
            _lib._lib = lib
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                _step(eng, x, dh)
            e1.record()
            e1.synchronize()
            times[n].append(e0.elapsed_time(e1) / iters)
    return {n: {"median_ms": round(sorted(v)[len(v) // 2], 4), "spread_ms": [round(min(v), 4), round(max(v), 4)]}
            for n, v in times.items()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=16384)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--other-lib", default=None, help="libdolomite_b200.so of another tree, compared on the C4 layer")
    a = ap.parse_args()
    card = _card()
    this = _lib.load()
    x, dh = _inputs(a.tokens)
    common = {"tokens": a.tokens, "n_embd": H, **card}

    if a.other_lib:
        path = _lib.LIB_PATH
        _lib.LIB_PATH, _lib._lib = os.path.abspath(a.other_lib), None
        other = _lib.load()
        _lib.LIB_PATH, _lib._lib = path, this
        for E, k in ((8, 2), (64, 8)):
            eng = _layer(E, k, 4096)
            digests = {}
            for name, lib in (("other", other), ("this", this)):
                _lib._lib = lib
                digests[name] = _digest(eng, x, dh)
            t = _time({"other": (other, eng), "this": (this, eng)}, x, dh, a.iters, a.rounds)
            print(json.dumps({"compare": "other library vs this one, C4 layer", "experts": E, "top_k": k, "n_inner": 4096,
                              "byte_identical": digests["other"] == digests["this"], **t, **common}), flush=True)
            del eng
            torch.cuda.empty_cache()
        _lib._lib = this

    for label, (va, vb) in (("n_inner 1376 vs 1408", ((8, 2, 1376), (8, 2, 1408))),
                            ("E 6 vs E 8", ((6, 2, 4096), (8, 2, 4096)))):
        engs = {f"E{E}_k{k}_F{F}": (this, _layer(E, k, F)) for E, k, F in (va, vb)}
        t = _time(engs, x, dh, a.iters, a.rounds)
        print(json.dumps({"compare": label, **t, **common}), flush=True)
        del engs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
