"""Pin ALiBi against the reference (needs the reference checkout; writes tests/golden fixtures).

    python tools/pin_alibi.py

tests/golden/alibi.npz
  slopes_<n>                      Alibi(n).slopes (fp32) for n in HEADS
  bias32_<case>_<n>, bias16_<case>_<n>
                                  Alibi(n).forward(mask, B, L, dtype) for fp32 and bf16 (as fp32 values), [B, n, L] at
                                  every BIAS_STRIDE-th key (L = 8192), every key for the short case
  mask_<case>                     the attention mask of the case (absent: no mask)
tests/golden/alibi_model_<name>.npz, for MODELS: a padded [B, S] batch run through the reference's GPTDolomiteBlocks
  (eager or sdpa) with the mask `_get_maybe_causal_mask` builds from `_get_alibi_bias` (both taken from the reference's
  GPTDolomiteModel as unbound methods on a duck-typed `self`), in fp32:
  tokens, mask (absent: no mask), loss, logits of the real positions, and every parameter's gradient, subsampled.
The oracle (tests/alibi_oracle.py over oracle/dolomite_oracle.py) is checked against the reference before anything is written.
"""

from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

GOLDEN = os.path.join(ROOT, "tests", "golden")
HEADS = [1, 2, 3, 5, 6, 8, 12, 20, 24, 32, 40, 48, 64]
GRAD_STRIDE = 16
BIAS_STRIDE = 61
_BASE = dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_inner=256, activation_function="swiglu",
             position_embedding_type="alibi", add_bias=False)
MODELS = {
    "mha_eager_nomask": (dict(n_head=8, attention_head_type="mha"), "eager", None),
    "gqa_eager_left": (dict(n_head=8, num_key_value_heads=2, attention_head_type="gqa"), "eager", "left"),
    "mqa_sdpa_mask": (dict(n_head=8, attention_head_type="mqa"), "sdpa", "right"),
    "mha_sdpa_nomask": (dict(n_head=8, attention_head_type="mha"), "sdpa", None),
}


def _mask(kind: str | None, B: int, S: int) -> np.ndarray | None:
    if kind is None:
        return None
    lens = [S, S - 5, 1, S - 17][:B]
    m = np.zeros((B, S), dtype=np.int64)
    for b, n in enumerate(lens):
        if kind == "left":
            m[b, S - n :] = 1
        else:
            m[b, :n] = 1
    return m


def _model_ns(R, n_heads: int, impl: str):
    """duck-typed GPTDolomiteModel carrying what _get_alibi_bias / _get_maybe_causal_mask read"""
    M = R.GPTDolomiteModel
    ns = types.SimpleNamespace(position_embedding_type=R.PositionEmbeddingType.alibi, alibi=R.Alibi(n_heads),
                               _use_sdpa=impl == "sdpa", _use_eager_attention=impl == "eager", mask_value=None)
    ns._prepare_causal_attention_mask = types.MethodType(M._prepare_causal_attention_mask, ns)
    ns._get_mask_value = types.MethodType(M._get_mask_value, ns)
    return ns, M


def reference_padded(R, cfg, impl: str, params: dict, tokens: np.ndarray, mask: np.ndarray | None):
    from oracle.validate_against_reference import ref_config

    rc = ref_config(cfg)
    B, S = tokens.shape
    blocks = []
    for i in range(cfg.n_layer):
        b = R.GPTDolomiteBlock(rc, "torch", impl, False, i)
        b.load_state_dict({k[len(f"transformer.h.{i}."):]: v for k, v in params.items() if k.startswith(f"transformer.h.{i}.")})
        blocks.append(b)
    ln_f = R.get_normalization_function(cfg.normalization_function, cfg.n_embd, eps=cfg.layer_norm_epsilon)
    ln_f.load_state_dict({"weight": params["transformer.ln_f.weight"]})
    wte = params["transformer.wte.weight"].clone().requires_grad_(True)
    am = None if mask is None else torch.as_tensor(mask)
    ns, M = _model_ns(R, cfg.n_head, impl)
    bias = M._get_alibi_bias(ns, am, B, S, S, None, torch.float32)
    attn_mask = M._get_maybe_causal_mask(ns, am, bias, B, S, S, torch.float32, None)
    h = torch.nn.functional.embedding(torch.as_tensor(tokens), wte)
    for b in blocks:
        h = b(h, attention_mask=attn_mask, rope_cos_sin=None)
    logits = torch.nn.functional.linear(ln_f(h), wte)
    # targets of real positions only (a padding position's successor is not a target, as in the engine's padded path)
    labels = torch.as_tensor(tokens)[:, 1:].clone()
    if am is not None:
        labels[(am[:, 1:] == 0) | (am[:, :-1] == 0)] = -100
    loss = torch.nn.functional.cross_entropy(logits[:, :-1].reshape(-1, logits.shape[-1]), labels.reshape(-1))
    loss.backward()
    grads = {f"transformer.h.{i}.{k}": v.grad for i, blk in enumerate(blocks) for k, v in blk.named_parameters()}
    grads["transformer.wte.weight"] = wte.grad
    grads["transformer.ln_f.weight"] = ln_f.weight.grad
    return loss.detach(), logits.detach(), grads


def oracle_padded(cfg, impl: str, params: dict, tokens: np.ndarray, mask: np.ndarray | None):
    """the oracle's packed form of the padded batch: every row's real tokens are one document"""
    import alibi_oracle as A
    import oracle.dolomite_oracle as O
    from dolomite_engine_b200.alibi import alibi_slopes

    B, S = tokens.shape
    m = np.ones((B, S), dtype=bool) if mask is None else mask.astype(bool)
    ids = tokens[m]
    cu = np.concatenate([[0], np.cumsum(m.sum(1))]).astype(np.int32)
    pos = np.concatenate([np.arange(n) for n in m.sum(1)])
    p = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    with_bias = impl == "eager" or mask is not None
    if with_bias:
        with A.install(alibi_slopes(cfg.n_head), bias_bf16=False):
            logits = O.forward_logits(p, cfg, ids, pos, cu)
    else:
        logits = O.forward_logits(p, cfg, ids, pos, cu)
    labels = np.full(ids.shape, -100, dtype=np.int64)
    for d in range(B):
        s, e = cu[d], cu[d + 1]
        labels[s : e - 1] = ids[s + 1 : e]
    loss = torch.nn.functional.cross_entropy(logits, torch.as_tensor(labels), ignore_index=-100)
    loss.backward()
    return loss.detach(), logits.detach(), {k: v.grad for k, v in p.items()}, m


def main():
    from oracle.validate_against_reference import import_reference

    import_reference()
    from dolomite_engine.hf_models.enums import PositionEmbeddingType as PET
    from dolomite_engine.hf_models.modeling_utils.position_embedding.alibi import Alibi
    from dolomite_engine.hf_models.models.gpt_dolomite.base import GPTDolomiteModel

    R = import_reference()
    R.Alibi, R.GPTDolomiteModel, R.PositionEmbeddingType = Alibi, GPTDolomiteModel, PET

    out = {}
    for n in HEADS:
        out[f"slopes_{n}"] = Alibi(n).slopes.numpy()
    # long cases keep every BIAS_STRIDE-th key (the file stays small); the short one keeps every key
    cases = {"nomask": (None, 2, 8192, BIAS_STRIDE), "left": ("left", 4, 8192, BIAS_STRIDE),
             "right": ("right", 4, 8192, BIAS_STRIDE), "short": ("left", 3, 37, 1)}
    for name, (kind, B, L, stride) in cases.items():
        mask = _mask(kind, B, L)
        am = None if mask is None else torch.as_tensor(mask)
        for n in (5, 32):
            a = Alibi(n)
            out[f"bias32_{name}_{n}"] = a(am, B, L, None, torch.float32)[..., ::stride].numpy()
            out[f"bias16_{name}_{n}"] = a(am, B, L, None, torch.bfloat16)[..., ::stride].float().numpy()
        if mask is not None:
            out[f"mask_{name}"] = mask
    np.savez_compressed(os.path.join(GOLDEN, "alibi.npz"), **out)
    print("alibi.npz: pinned")

    import oracle.dolomite_oracle as O

    for name, (kw, impl, kind) in MODELS.items():
        cfg = O.OracleConfig(**_BASE, **kw)
        params = O.init_params(cfg, seed=42)
        rng = np.random.default_rng(99)
        tokens = rng.integers(0, cfg.vocab_size, size=(3, 48), dtype=np.int64)
        mask = _mask(kind, 3, 48)
        loss, logits, grads = reference_padded(R, cfg, impl, params, tokens, mask)
        loss_o, logits_o, grads_o, m = oracle_padded(cfg, impl, params, tokens, mask)
        real = torch.as_tensor(m)
        dl = (logits[real] - logits_o).abs().max().item()
        dg = max((grads_o[k] - v).abs().max().item() for k, v in grads.items())
        print(f"model {name}: loss {loss.item():.6f} vs oracle {loss_o.item():.6f}, logits {dl:.2e}, grads {dg:.2e}")
        # eager: the existing pins; SDPA sums in another order (measured up to 1.4e-6 / 2.2e-8)
        tol_l, tol_g = (4e-7, 2e-9) if impl == "eager" else (2e-6, 5e-8)
        assert abs(loss.item() - loss_o.item()) <= 1e-5 and dl <= tol_l and dg <= tol_g, name
        fx = {"tokens": tokens, "loss": loss.numpy(), "logits": logits[real].numpy()}
        if mask is not None:
            fx["mask"] = mask
        for k, v in grads.items():
            fx[f"grad:{k}"] = v.flatten()[::GRAD_STRIDE].numpy()
        np.savez_compressed(os.path.join(GOLDEN, f"alibi_model_{name}.npz"), **fx)


if __name__ == "__main__":
    main()
