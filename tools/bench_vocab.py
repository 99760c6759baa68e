"""Cost of a vocabulary that is not a multiple of 8, at C2's shape (configs/c2_granite3b_shape.yml: 32 layers, 2560 wide,
T = 2 x 4096 tokens) for V = 49152 (C2), 49155 (Granite 3.x) and 50257 (GPT-2 / the reference's pretraining examples):

  * the LM head's three GEMMs (forward [T, V], dgrad, fp32 wgrad) and the cross-entropy kernel on [T, V], median of 20
    launches each, CUDA events;
  * one training step (forward with the fused head + loss, backward; no optimizer), median of 5 after 2 warm-up steps.

Prints one JSON line per measurement and the GPU's name and power limit.

    python tools/bench_vocab.py [--layers N]
"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dolomite_engine_b200 import kernels as K  # noqa: E402

VOCABS = (49152, 49155, 50257)
T, H = 8192, 2560
C2 = dict(n_positions=4096, n_embd=H, n_layer=32, n_head=32, n_inner=10240, attention_head_type="mha",
          position_embedding_type="rope", activation_function="swiglu", normalization_function="rmsnorm",
          layer_norm_epsilon=1e-5, add_bias=True, resid_pdrop=0, embd_pdrop=0, attn_pdrop=0, eos_token_id=0)


def median_ms(fn, n: int = 20, warmup: int = 3) -> float:
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def head_kernels(V: int) -> dict:
    g = torch.Generator(device="cuda").manual_seed(0)
    hf = (torch.randn(T, H, generator=g, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(V, H, generator=g, device="cuda") * 0.02).bfloat16()
    gw = torch.zeros(V, H, device="cuda")
    labels = torch.randint(0, V, (T,), generator=g, device="cuda")
    logits = K.gemm(hf, w)
    dlogits = K.rows_empty(T, V, device="cuda")
    out = {"head_fwd_ms": median_ms(lambda: K.gemm(hf, w, out=logits)),
           "cross_entropy_ms": median_ms(lambda: K.cross_entropy_fwd_bwd(logits, labels, dlogits=dlogits)),
           "head_dgrad_ms": median_ms(lambda: K.gemm(logits, w, b_mn=True)),
           "head_wgrad_ms": median_ms(lambda: K.gemm(logits, hf, a_mn=True, b_mn=True, out=gw))}
    out["head_row_stride"] = logits.stride(0)
    return out


def step_ms(V: int, layers: int) -> float:
    from dolomite_engine_b200.engine import DolomiteEngine
    from dolomite_engine_b200.hf_models import GPTDolomiteConfig

    cfg = GPTDolomiteConfig(vocab_size=V, **{**C2, "n_layer": layers})
    eng = DolomiteEngine(cfg, "cuda", seed=1, init_on_device=True)
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(0, V, (T + 1,), generator=g, device="cuda")
    pos = torch.arange(4096, device="cuda").repeat(2)
    cu = torch.tensor([0, 4096, T], dtype=torch.int32, device="cuda")

    def step():
        eng.zero_grad()
        eng.forward(ids[:-1], pos, cu, 4096, labels=ids[1:], fuse_head_loss=True)
        eng.backward()

    ms = median_ms(step, n=5, warmup=2)
    del eng
    torch.cuda.empty_cache()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=C2["n_layer"])
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({"gpu": gpu, "T": T, "H": H, "layers": a.layers}))
    for V in VOCABS:
        r = {"V": V, **head_kernels(V)}
        torch.cuda.empty_cache()
        r["step_ms"] = step_ms(V, a.layers)
        r["step_tokens_per_s"] = T / (r["step_ms"] / 1e3)
        print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in r.items()}))


if __name__ == "__main__":
    main()
