"""Cost of a forward with a KV cache (engine.extend, csrc/attention_cache.cu):

  * attention only: attn_cache for n new tokens per sequence after `past` cached ones, n in {1, 4, 16, 64, 512} and past in
    {1024, 4096, 16384}, B sequences, for the heads of C2 (32 x 80 MHA), GQA 32:8 x 128, MQA 24 x 128 and MHA 12 x 256.
    Median of CUDA-event timings; algorithmic TFLOP/s (4 hd FLOP per visible (query, key) pair and head) and GB/s of cache
    read (K and V of past + n positions per sequence, once).  Beside it, n sequential attn_decode calls (the single-query
    kernel decode_step runs, one step per new token), which is what extend runs when every sequence has exactly 1 new token.
  * model: a C2-shaped model of --layers blocks, B sequences of a 4096-token cache, appending a 512-token turn
    (model(..., past_key_values=cache)) against re-running the uncached padded forward over all 4608 tokens; alternating
    rounds after a warm-up of each.

Prints one JSON line per measurement, after one with the GPU's name, power limit and max SM clock.

    python tools/bench_kv_cache.py [--batch B] [--layers N] [--rounds R] [--skip-model]
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

HEADS = {"c2_mha_32x80": (32, 1, 80), "gqa_32:8x128": (8, 4, 128), "mqa_24x128": (1, 24, 128), "mha_12x256": (12, 1, 256)}
NEWS = (1, 4, 16, 64, 512)
PASTS = (1024, 4096, 16384)


def median_ms(fn, n: int, warmup: int = 2) -> float:
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


def attention(B: int) -> list[dict]:
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for hname, (ng, gq, hd) in HEADS.items():
        nh, W = ng * gq, ng * (gq + 2) * hd
        L = max(PASTS) + max(NEWS)
        kc = torch.randn(B, L, ng * hd, generator=g, device="cuda").bfloat16()
        vc = torch.randn(B, L, ng * hd, generator=g, device="cuda").bfloat16()
        for past in PASTS:
            for n in NEWS:
                qkv = torch.randn(B * n, W, generator=g, device="cuda").bfloat16()
                cu = torch.arange(0, B * n + 1, n, dtype=torch.int32, device="cuda")
                pa = torch.full((B,), past, dtype=torch.int32, device="cuda")
                out = torch.empty(B * n, nh * hd, dtype=torch.bfloat16, device="cuda")
                scale = hd**-0.5
                ms = median_ms(lambda: K.attn_cache(qkv, cu, pa, kc, vc, ng, gq, hd, scale, max_new=n, max_end=past + n,
                                                    out=out), n=20)
                # n sequential single-query steps: step k sees past + k + 1 keys
                lens = [torch.full((B,), past + k + 1, dtype=torch.int32, device="cuda") for k in range(n)]
                q1 = qkv[:B].contiguous()
                seq_ms = median_ms(lambda: [K.attn_decode(q1, kc, vc, ln, ng, gq, hd, scale) for ln in lens],
                                   n=5 if n >= 64 else 20)
                pairs = B * sum(past + i + 1 for i in range(n))
                flop = 4 * hd * nh * pairs
                nbytes = 2 * B * (past + n) * ng * hd * 2
                rows.append({"measurement": "attn_cache", "heads": hname, "B": B, "past": past, "n": n,
                             "attn_cache_us": ms * 1e3, "tflops": flop / ms / 1e9, "cache_read_gbs": nbytes / ms / 1e6,
                             "n_decode_calls_us": seq_ms * 1e3, "one_decode_us": seq_ms * 1e3 / n if n == 1 else None})
        del kc, vc
        torch.cuda.empty_cache()
    return rows


def model_turn(B: int, layers: int, rounds: int, past: int = 4096, turn: int = 512) -> dict:
    from dolomite_engine_b200.hf_models import GPTDolomiteConfig, GPTDolomiteForCausalLM

    cfg = GPTDolomiteConfig(vocab_size=49152, n_positions=8192, n_embd=2560, n_layer=layers, n_head=32, n_inner=10240,
                            attention_head_type="mha", position_embedding_type="rope", activation_function="swiglu",
                            normalization_function="rmsnorm", add_bias=True, resid_pdrop=0, embd_pdrop=0, attn_pdrop=0,
                            eos_token_id=0)
    model = GPTDolomiteForCausalLM(cfg, attn_implementation="flash_attention_2", use_padding_free_transformer=False,
                                   device=torch.device("cuda", 0))
    model.eval()
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(1, 49152, (B, past + turn), generator=g).cuda()
    mask = torch.ones_like(ids)
    with torch.no_grad():
        base = model(input_ids=ids[:, :past], attention_mask=mask[:, :past], use_cache=True).past_key_values
        base.reserve(past + turn)
        lens0 = base.lens.clone()

        def cached():
            base.lens.copy_(lens0)
            base.seen = past
            return model(input_ids=ids[:, past:], attention_mask=mask, past_key_values=base).logits

        def full():
            return model(input_ids=ids, attention_mask=mask).logits

        a = cached()
        b = full()[:, past:]
        diff = (a.float() - b.float()).abs().max().item()
        t_cached, t_full = [], []
        for _ in range(rounds):
            t_cached.append(median_ms(cached, n=5))
            t_full.append(median_ms(full, n=5))
    return {"measurement": "model_turn", "layers": layers, "B": B, "past": past, "turn": turn,
            "extend_ms": statistics.median(t_cached), "uncached_ms": statistics.median(t_full),
            "speedup": statistics.median(t_full) / statistics.median(t_cached), "max_abs_logit_diff": diff}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-model", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_kv_cache needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    rnd = lambda d: {k: (round(v, 3) if isinstance(v, float) else v) for k, v in d.items()}  # noqa: E731
    for r in attention(a.batch):
        print(json.dumps(rnd(r)), flush=True)
    if not a.skip_model:
        print(json.dumps(rnd(model_turn(a.batch, a.layers, a.rounds))), flush=True)
