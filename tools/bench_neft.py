"""Cost of NEFTune noise (`research_args.neft_alpha`):

  * the embedding gather with and without noise at T = 16384 tokens, H = 4096, V = 128256 (Llama-3-8B's table), median of
    50 launches each, CUDA events, as a share of 3.35 TB/s (H100 SXM HBM3) for the bytes the gather must move: T rows of
    2H bytes read, T rows written, T int64 ids;
  * a reduced C5 finetuning step (bench.py's Llama-3-8B shape with --layers blocks, seq 8192 as 4 ragged documents, block
    checkpointing every 2; forward with the fused head + loss and backward, no optimizer) with and without NEFTune,
    alternating rounds of 5 steps after 2 warm-up steps each.

Prints one JSON line per measurement, with the GPU's name and power limit.

    python tools/bench_neft.py [--layers N] [--rounds R]
"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from dolomite_engine_b200 import kernels as K  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
NEFT_SITE = -1


def median_ms(fn, n: int = 50, warmup: int = 5) -> float:
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


def gather(T: int = 16384, H: int = 4096, V: int = 128256) -> dict:
    g = torch.Generator(device="cuda").manual_seed(0)
    wte = (torch.randn(V, H, generator=g, device="cuda") * 0.02).to(torch.bfloat16)
    ids = torch.randint(0, V, (T,), generator=g, device="cuda")
    out = torch.empty(T, H, dtype=torch.bfloat16, device="cuda")
    keys, mag = K.dropout_keys(1, NEFT_SITE), K.neft_mag(5.0, T * H)
    plain = median_ms(lambda: K.embedding_fwd(ids, wte, out=out))
    neft = median_ms(lambda: K.embedding_fwd_neft(ids, wte, keys, mag, out=out))
    nbytes = 2 * T * H * 2 + T * 8
    floor_ms = nbytes / HBM_BYTES_PER_S * 1e3
    return {"measurement": "embedding_gather", "T": T, "H": H, "V": V, "bytes": nbytes,
            "plain_ms": plain, "neft_ms": neft, "plain_share_of_hbm": floor_ms / plain, "neft_share_of_hbm": floor_ms / neft,
            "neft_over_plain": neft / plain}


def step(layers: int, rounds: int) -> dict:
    import bench

    from dolomite_engine_b200.engine import DolomiteEngine
    from dolomite_engine_b200.hf_models import GPTDolomiteConfig

    cfg_d = bench.model_config("c5", layers)
    cfg_d.pop("model_type", None)
    cfg = GPTDolomiteConfig(**cfg_d)
    eng = DolomiteEngine(cfg, "cuda", seed=1, init_on_device=True)
    eng.checkpoint_every = 2
    eng.dropout_seed = 1
    lens = [3000, 2500, 1700, 992]
    T = sum(lens)
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(0, cfg.vocab_size, (T,), generator=g, device="cuda")
    labels = ids.roll(-1)
    pos = torch.cat([torch.arange(n, device="cuda") for n in lens])
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device="cuda")

    def one():
        eng.zero_grad()
        eng.forward(ids, pos, cu, max(lens), labels=labels, fuse_head_loss=True)
        eng.backward()

    times = {"off": [], "on": []}
    for _ in range(rounds):
        for mode in ("off", "on"):
            eng.neft_alpha = 5.0 if mode == "on" else None
            times[mode].append(median_ms(one, n=5, warmup=2))
    off, on = statistics.median(times["off"]), statistics.median(times["on"])
    return {"measurement": "c5_reduced_step", "layers": layers, "tokens": T, "rounds": rounds, "off_ms": off, "on_ms": on,
            "on_over_off": on / off, "off_rounds_ms": times["off"], "on_rounds_ms": times["on"]}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_neft.py measures on a CUDA device; none is available")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}))
    rnd = lambda d: {k: (round(v, 4) if isinstance(v, float) else v) for k, v in d.items()}  # noqa: E731
    print(json.dumps(rnd(gather())))
    torch.cuda.empty_cache()
    print(json.dumps(rnd(step(a.layers, a.rounds))))


if __name__ == "__main__":
    main()
