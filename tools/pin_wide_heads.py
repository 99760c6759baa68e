"""Pin models with wide attention heads (head_dim 160, 192, 256) against the reference (needs the reference checkout;
writes tests/golden fixtures).

    python tools/pin_wide_heads.py

tests/golden/model_wide_<name>.npz, for MODELS (fp32 reference leaf modules, glued as oracle/validate_against_reference.py
does):
- mqa_hd256, gqa_hd192, mha_hd160_bigcode: a packed batch (documents split at eos) and a right / left padded batch, run as
  tools/pin_vocab.py runs its models; loss, the logits of every 8th real position and subsampled gradients of every
  parameter (tensors of up to 4096 elements whole, larger ones every 61st element: a prime stride samples every row and
  column);
- mqa_hd256_alibi_sdpa: a padded, masked batch through the reference's GPTDolomiteBlocks with SDPA and the ALiBi mask
  of `_get_maybe_causal_mask`, run as tools/pin_alibi.py runs its models; loss, the logits of the real positions and
  the same gradient samples.

mqa_hd256 is the 3B research baseline's shape (MQA, RoPE, RMSNorm, SwiGLU, biases; n_embd / n_head = 256) at a width of 512.
The oracle (oracle/dolomite_oracle.py) is checked against the reference before anything is written.
"""

from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

GOLDEN = os.path.join(ROOT, "tests", "golden")
FULL_GRAD = 4096
GRAD_STRIDE = 61


def subsample(g: torch.Tensor) -> torch.Tensor:
    g = g.flatten()
    return g if g.numel() <= FULL_GRAD else g[::GRAD_STRIDE]


# the same table as tests/test_gpu_wide_heads_model.py MODELS
MODELS = {
    "mqa_hd256": dict(vocab_size=256, n_positions=256, n_embd=512, n_layer=2, n_head=2, n_inner=512,
                      attention_head_type="mqa", position_embedding_type="rope", normalization_function="rmsnorm",
                      activation_function="swiglu", add_bias=True),
    "gqa_hd192": dict(vocab_size=256, n_positions=256, n_embd=768, n_layer=2, n_head=4, num_key_value_heads=2,
                      n_inner=512, attention_head_type="gqa", position_embedding_type="rope",
                      normalization_function="rmsnorm", activation_function="swiglu", add_bias=False),
    "mha_hd160_bigcode": dict(vocab_size=256, n_positions=256, n_embd=320, n_layer=2, n_head=2, n_inner=640,
                              attention_head_type="mha", position_embedding_type="learned_absolute",
                              normalization_function="layernorm", activation_function="gelu_pytorch_tanh", add_bias=True),
}
ALIBI_MODEL = ("mqa_hd256_alibi_sdpa", dict(vocab_size=512, n_positions=256, n_embd=512, n_layer=2, n_head=2,
                                            n_inner=512, attention_head_type="mqa", position_embedding_type="alibi",
                                            activation_function="swiglu", add_bias=False), "sdpa", "right")


def main():
    import pin_alibi as PA
    import pin_vocab as PV
    from oracle.validate_against_reference import import_reference

    import oracle.dolomite_oracle as O

    R = import_reference()
    for name, kw in MODELS.items():
        cfg = O.OracleConfig(**kw)
        params = O.init_params(cfg, seed=42)
        if cfg.add_bias:  # non-zero biases, so that the bias path is checked
            g = torch.Generator().manual_seed(7)
            for k in params:
                if k.endswith(".bias"):
                    params[k] = torch.randn(params[k].shape, generator=g) * 0.02
        tokens, ids, pos, cu, labels = PV.packed_batch(O, cfg.vocab_size)
        ptok, mask, pids, ppos, pcu, plabels = PV.padded_batch(cfg.vocab_size)
        fx = {"packed_tokens": tokens, "padded_tokens": ptok, "padded_mask": mask}
        if cfg.add_bias:
            fx.update({f"bias:{k}": v.numpy() for k, v in params.items() if k.endswith(".bias")})
        for batch, args in (("packed", (ids, pos, cu, labels)), ("padded", (pids, ppos, pcu, plabels))):
            loss, logits, grads = PV.reference_run(R, cfg, params, *args)
            loss_o, logits_o, grads_o = PV.oracle_run(O, cfg, params, *args)
            assert set(grads) == set(grads_o), sorted(set(grads) ^ set(grads_o))
            dl = (logits - logits_o).abs().max().item()
            dg = max(((grads_o[k] - v).abs().max() / (v.abs().max() + 1e-30)).item() for k, v in grads.items())
            print(f"{name} {batch}: loss {loss.item():.6f} vs oracle {loss_o.item():.6f}, logits {dl:.2e}, "
                  f"grads (relative to each absmax) {dg:.2e}")
            assert abs(loss.item() - loss_o.item()) <= 1e-5 and dl <= 2e-5 and dg <= 1e-4, name
            fx[f"{batch}_loss"] = loss.numpy()
            fx[f"{batch}_logits"] = logits[:: PV.LOGIT_ROW_STRIDE].numpy()
            for k, v in grads.items():
                fx[f"{batch}_grad:{k}"] = subsample(v).numpy()
        np.savez_compressed(os.path.join(GOLDEN, f"model_wide_{name}.npz"), **fx)

    from dolomite_engine.hf_models.enums import PositionEmbeddingType as PET
    from dolomite_engine.hf_models.modeling_utils.position_embedding.alibi import Alibi
    from dolomite_engine.hf_models.models.gpt_dolomite.base import GPTDolomiteModel

    R.Alibi, R.GPTDolomiteModel, R.PositionEmbeddingType = Alibi, GPTDolomiteModel, PET
    name, kw, impl, kind = ALIBI_MODEL
    cfg = O.OracleConfig(**kw)
    params = O.init_params(cfg, seed=42)
    tokens = np.random.default_rng(99).integers(0, cfg.vocab_size, size=(3, 48), dtype=np.int64)
    mask = PA._mask(kind, 3, 48)
    loss, logits, grads = PA.reference_padded(R, cfg, impl, params, tokens, mask)
    loss_o, logits_o, grads_o, m = PA.oracle_padded(cfg, impl, params, tokens, mask)
    real = torch.as_tensor(m)
    dl = (logits[real] - logits_o).abs().max().item()
    dg = max(((grads_o[k] - v).abs().max() / (v.abs().max() + 1e-30)).item() for k, v in grads.items())
    print(f"{name}: loss {loss.item():.6f} vs oracle {loss_o.item():.6f}, logits {dl:.2e}, grads (relative) {dg:.2e}")
    assert abs(loss.item() - loss_o.item()) <= 1e-5 and dl <= 2e-5 and dg <= 1e-4, name
    fx = {"tokens": tokens, "mask": mask, "loss": loss.numpy(), "logits": logits[real].numpy()}
    for k, v in grads.items():
        fx[f"grad:{k}"] = subsample(v).numpy()
    np.savez_compressed(os.path.join(GOLDEN, f"model_wide_{name}.npz"), **fx)
    print("wide-head fixtures written to", GOLDEN)


if __name__ == "__main__":
    main()
