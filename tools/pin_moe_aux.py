"""Pin the MoE load-balancing loss and write tests/golden/moe_aux.npz.

    python tools/pin_moe_aux.py [--reference DIR]

Runs the installed transformers' Mixtral `load_balancing_loss_func` on seeded router logits, unmasked and with an
attention mask (left and right padding), and the reference's `get_moe_loss` glue (moe_dolomite/base.py:24-43) imported
read-only from a checkout of the reference, as oracle/validate_against_reference.py imports it.  When that module does
not import, the glue is restated (loss = CE + router_aux_loss_coef * aux; aux alone without labels) and the fixture
records that it was.

The logits have no near-ties: each row is a shuffled grid of values 0.5 apart, exact in bf16.  bf16 probabilities can
tie where logits do not, and then a top-k of the probabilities (transformers) and a top-k of the logits (this engine's
routing plan) may select different experts.
"""

from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "moe_aux.npz")

CASES = [  # (name, layers, batch, seq, experts, top-k, padding)
    ("e8_k2_right", 2, 3, 11, 8, 2, "right"),
    ("e8_k2_left", 2, 3, 11, 8, 2, "left"),
    ("e16_k4_none", 3, 2, 9, 16, 4, "none"),
    ("e40_k1_right", 1, 4, 7, 40, 1, "right"),
    ("e64_k8_left", 2, 2, 13, 64, 8, "left"),
]
COEF = 0.02


def case_inputs(layers: int, batch: int, seq: int, experts: int, padding: str, seed: int):
    g = np.random.default_rng(seed)
    grid = (np.arange(experts) - experts // 2) * 0.5  # exact in bf16 for |x| <= 64
    logits = np.stack([np.stack([g.permutation(grid) for _ in range(batch * seq)]) for _ in range(layers)]).astype(np.float32)
    mask = np.ones((batch, seq), dtype=np.int64)
    if padding != "none":
        lens = g.integers(1, seq + 1, size=batch)
        lens[0] = seq
        for b, n in enumerate(lens):
            mask[b] = 0
            if padding == "right":
                mask[b, :n] = 1
            else:
                mask[b, seq - n :] = 1
    return logits, mask


def reference_glue(ref_dir: str | None):
    import oracle.validate_against_reference as V

    V.REF = ref_dir or V.REF
    if not os.path.isdir(V.REF):
        return None
    try:
        V.import_reference()
        from dolomite_engine.hf_models.models.moe_dolomite.base import MoEDolomitePreTrainedModel

        return MoEDolomitePreTrainedModel.get_moe_loss
    except Exception as e:  # the fixture then records the restated glue
        print(f"reference get_moe_loss did not import ({type(e).__name__}: {e}); restating it", file=sys.stderr)
        return None


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=None, help="reference checkout (default: validate_against_reference's)")
    a = ap.parse_args()
    from transformers.models.mixtral.modeling_mixtral import load_balancing_loss_func

    get_moe_loss = reference_glue(a.reference)
    out = {"coef": np.float64(COEF), "glue_from_reference": np.int64(get_moe_loss is not None)}
    for i, (name, L, B, S, E, k, padding) in enumerate(CASES):
        logits, mask = case_inputs(L, B, S, E, padding, seed=100 + i)
        gate = tuple(torch.from_numpy(logits[l]).double() for l in range(L))
        aux_plain = load_balancing_loss_func(gate, E, k)
        aux_masked = load_balancing_loss_func(gate, E, k, attention_mask=torch.from_numpy(mask))
        ce = torch.tensor(1.2345, dtype=torch.float64)
        if get_moe_loss is not None:
            owner = type("Owner", (), {"get_autoregressive_language_modeling_loss": lambda self, *args: None if args[1] is None else ce.clone()})()
            glue_loss, glue_aux = get_moe_loss(owner, None, torch.zeros(1), None, gate, E, k, COEF, True)
            none_loss, none_aux = get_moe_loss(owner, None, None, None, gate, E, k, COEF, True)
            assert none_loss is None
            off_loss, off_aux = get_moe_loss(owner, None, torch.zeros(1), None, gate, E, k, COEF, None)
            assert off_aux is None and float(off_loss) == float(ce)  # the flag unresolved (None): no term
        else:
            glue_loss, glue_aux = ce + COEF * aux_plain, aux_plain
            none_aux = aux_plain
        out.update({
            f"{name}/logits": logits, f"{name}/mask": mask, f"{name}/shape": np.array([L, B, S, E, k], dtype=np.int64),
            f"{name}/aux": np.float64(aux_plain), f"{name}/aux_masked": np.float64(aux_masked),
            f"{name}/ce": np.float64(ce), f"{name}/glue_loss": np.float64(glue_loss), f"{name}/glue_aux": np.float64(glue_aux),
            f"{name}/glue_aux_no_labels": np.float64(none_aux),
        })
        print(f"{name}: aux {float(aux_plain):.9f}  masked {float(aux_masked):.9f}  loss {float(glue_loss):.9f}")
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
