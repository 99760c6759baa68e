"""Pin models with vocabularies that are not a multiple of 8 against the reference (needs the reference checkout; writes
tests/golden fixtures).

    python tools/pin_vocab.py

tests/golden/model_vocab_<name>.npz, for MODELS, each with two batches run through the reference's GPTDolomiteBlock /
SparseMoEBlock (eager, fp32) glued as oracle/validate_against_reference.py does (one document per batch row):
  <batch>_tokens                  packed: [2, 97] pretraining tokens (documents split at eos, positions reset);
                                  padded: [3, 40] rows, real tokens given by <batch>_mask (1 = token, right / left padded)
  <batch>_loss                    mean CE of the batch (packed: every position; padded: targets of real positions)
  <batch>_logits                  fp32 logits of every LOGIT_ROW_STRIDE-th real position, in token order
  <batch>_grad:<name>             every parameter's gradient, flattened: whole up to FULL_GRAD elements, else every
                                  GRAD_STRIDE-th element
The oracle (oracle/dolomite_oracle.py) is checked against the reference before anything is written.
"""

from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")
GRAD_STRIDE = 16
FULL_GRAD = 4096  # small tensors (biases, norm weights) are kept whole: a few samples of them say little
LOGIT_ROW_STRIDE = 8
EOS = 7
MODELS = {
    # the StarCoder / bigcode shape of the reference's pretraining examples, untied head
    "bigcode_2053": dict(vocab_size=2053, n_positions=256, n_embd=128, n_layer=2, n_head=8, n_inner=512,
                         attention_head_type="mqa", activation_function="gelu_pytorch_tanh", add_bias=True,
                         normalization_function="layernorm", position_embedding_type="learned_absolute",
                         tie_word_embeddings=False),
    "gqa_rope_2051": dict(vocab_size=2051, n_positions=256, n_embd=128, n_layer=2, n_head=8, num_key_value_heads=2,
                          n_inner=256, attention_head_type="gqa", activation_function="swiglu", add_bias=False),
    "moe_2055": dict(vocab_size=2055, n_positions=256, n_embd=128, n_layer=2, n_head=8, n_inner=128,
                     attention_head_type="mha", activation_function="swiglu", add_bias=False, num_experts=8,
                     num_experts_per_tok=2),
}


def subsample(g: torch.Tensor) -> torch.Tensor:
    g = g.flatten()
    return g if g.numel() <= FULL_GRAD else g[::GRAD_STRIDE]


def packed_batch(O, V: int):
    """[2, 97] tokens with documents split at eos (reset attention mask and positions)"""
    rng = np.random.default_rng(V)
    tokens = rng.integers(0, V, size=(2, 97), dtype=np.int64)
    tokens[0, 30] = EOS
    tokens[1, 60] = EOS
    tokens[:, -1] = V - 1  # the last vocabulary entry, whose 16-byte vector is the partial one, is a target
    inp, labels = O.split_tokens(tokens)
    b = O.prepare_model_inputs(inp.copy(), EOS, True, True)
    return tokens, b["input_ids"], b["position_ids"], b["cu_seqlens"], np.ascontiguousarray(labels).reshape(-1)


def padded_mask(B: int = 3, S: int = 40) -> np.ndarray:
    m = np.zeros((B, S), dtype=np.int64)
    m[0, :] = 1
    m[1, : S - 7] = 1  # right padded
    m[2, S - 17 :] = 1  # left padded
    return m


def padded_batch(V: int):
    """[3, 40] rows; each row's real tokens are one document, targets are the successors that are real tokens"""
    rng = np.random.default_rng(V + 1)
    tokens = rng.integers(0, V, size=(3, 40), dtype=np.int64)
    tokens[1, 5] = V - 1
    mask = padded_mask()
    m = mask.astype(bool)
    ids = tokens[m]
    lens = m.sum(1)
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    pos = np.concatenate([np.arange(n) for n in lens])
    labels = np.full(ids.shape, -100, dtype=np.int64)
    for d in range(len(lens)):
        s, e = cu[d], cu[d + 1]
        labels[s : e - 1] = ids[s + 1 : e]
    return tokens, mask, ids, pos, cu, labels


def _moe_block_class():
    from dolomite_engine.hf_models.models.moe_dolomite.layer import SparseMoEBlock

    class MoEBlock(SparseMoEBlock):
        """SparseMoEBlock with the dense block's constructor and return value (eager experts)"""

        def __init__(self, rc, normalization_implementation, attention_implementation, padding_free, layer_idx):
            super().__init__(rc, normalization_implementation, attention_implementation, padding_free, "eager", layer_idx)

        def forward(self, h, attention_mask=None, rope_cos_sin=None):
            out = super().forward(h, attention_mask=attention_mask, rope_cos_sin=rope_cos_sin)
            return out[0] if isinstance(out, tuple) else out

    return MoEBlock


def reference_run(R, cfg, params, ids, pos, cu, labels):
    from oracle.validate_against_reference import reference_forward

    if cfg.num_experts > 0:
        R = types.SimpleNamespace(**{**vars(R), "GPTDolomiteBlock": _moe_block_class()})
    p = {k: v.clone() for k, v in params.items()}
    head = None
    if not cfg.tie_word_embeddings:
        head = p["lm_head.weight"] = p["lm_head.weight"].requires_grad_(True)
    logits, blocks, wte, wpe, ln_f_grads = reference_forward(R, cfg, p, ids, pos, cu)
    loss = torch.nn.functional.cross_entropy(logits, torch.as_tensor(labels), ignore_index=-100)
    loss.backward()
    grads = {f"transformer.h.{i}.{k}": v.grad for i, blk in enumerate(blocks) for k, v in blk.named_parameters()}
    grads["transformer.wte.weight"] = wte.grad
    grads.update(ln_f_grads())
    if wpe is not None:
        grads["transformer.wpe.weight"] = wpe.grad
    if head is not None:
        grads["lm_head.weight"] = head.grad
    return loss.detach(), logits.detach(), grads


def oracle_run(O, cfg, params, ids, pos, cu, labels):
    p = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    logits = O.forward_logits(p, cfg, ids, pos, cu)
    loss = torch.nn.functional.cross_entropy(logits, torch.as_tensor(labels), ignore_index=-100)
    loss.backward()
    return loss.detach(), logits.detach(), {k: v.grad for k, v in p.items()}


def main():
    from oracle.validate_against_reference import import_reference

    import oracle.dolomite_oracle as O

    R = import_reference()
    for name, kw in MODELS.items():
        cfg = O.OracleConfig(**kw)
        params = O.init_params(cfg, seed=42)
        if cfg.add_bias:  # non-zero biases, so that the bias path is checked (as validate_against_reference does)
            g = torch.Generator().manual_seed(7)
            for k in params:
                if k.endswith(".bias"):
                    params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        tokens, ids, pos, cu, labels = packed_batch(O, cfg.vocab_size)
        ptok, mask, pids, ppos, pcu, plabels = padded_batch(cfg.vocab_size)
        fx = {"packed_tokens": tokens, "padded_tokens": ptok, "padded_mask": mask}
        if cfg.add_bias:
            fx.update({f"bias:{k}": v.numpy() for k, v in params.items() if k.endswith(".bias")})
        for batch, args in (("packed", (ids, pos, cu, labels)), ("padded", (pids, ppos, pcu, plabels))):
            loss, logits, grads = reference_run(R, cfg, params, *args)
            loss_o, logits_o, grads_o = oracle_run(O, cfg, params, *args)
            assert set(grads) == set(grads_o), sorted(set(grads) ^ set(grads_o))
            dl = (logits - logits_o).abs().max().item()
            dg = max(((grads_o[k] - v).abs().max() / (v.abs().max() + 1e-30)).item() for k, v in grads.items())
            print(f"{name} {batch}: loss {loss.item():.6f} vs oracle {loss_o.item():.6f}, logits {dl:.2e}, "
                  f"grads (relative to each absmax) {dg:.2e}")
            assert abs(loss.item() - loss_o.item()) <= 1e-5 and dl <= 2e-5 and dg <= 1e-4, name
            fx[f"{batch}_loss"] = loss.numpy()
            fx[f"{batch}_logits"] = logits[::LOGIT_ROW_STRIDE].numpy()
            for k, v in grads.items():
                fx[f"{batch}_grad:{k}"] = subsample(v).numpy()
        np.savez_compressed(os.path.join(GOLDEN, f"model_vocab_{name}.npz"), **fx)
    print("vocabulary fixtures written to", GOLDEN)


if __name__ == "__main__":
    main()
