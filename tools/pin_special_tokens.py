"""Pin the reference's vocabulary resize for `tokenizer_args.additional_special_tokens` (needs the reference checkout;
writes tests/golden/special_tokens.npz).

    python tools/pin_special_tokens.py

The reference adds the tokens to its tokenizer and, when len(tokenizer) changed, calls
`model.resize_token_embeddings(len(tokenizer))` (model_wrapper/base.py:102-108): transformers' resize on the reference's
GPTDolomiteForCausalLM (get/set_input_embeddings, get/set_output_embeddings), with mean_resizing=True, on CPU, drawing
from torch's global generator.  The tokenizer is a word-level one built locally with `tokenizers` (tests/special_tokens_util.py
builds the same one), so no download is needed.

For each case <c> in CASES (grow and shrink, tied and untied head):
  <c>_meta            [V_config, V_tokenizer, V_new, tied, H, seed]
  <c>_wte, <c>_lm_head                     the rows before the resize (fp32; lm_head only when untied)
  <c>_new_wte, <c>_new_lm_head             the rows after it
  <c>_after           torch.rand(8) drawn right after the resize: the generator consumed what the reference consumed
"""

from __future__ import annotations

import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from special_tokens_util import ADDED_TOKENS, build_tokenizer  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "special_tokens.npz")
H = 32
BASE_VOCAB = 300  # the tokenizer's length before the tokens are added
# name -> (config vocab_size, tied head, seed of the global generator before the resize)
CASES = {
    "grow_tied": (BASE_VOCAB, True, 11),
    "grow_untied": (BASE_VOCAB, False, 12),
    # vocab_size padded above the tokenizer: len(tokenizer) + 3 < vocab_size, so the resize shrinks the model
    "shrink_tied": (BASE_VOCAB + 8, True, 13),
    "shrink_untied": (BASE_VOCAB + 8, False, 14),
}


def reference_model(R, V: int, tied: bool, g: torch.Generator):
    """the reference's GPTDolomiteForCausalLM with only what resize_token_embeddings touches (its full constructor needs
    config attributes this transformers version no longer sets)"""
    import torch.nn as nn

    m = R.GPTDolomiteForCausalLM.__new__(R.GPTDolomiteForCausalLM)
    nn.Module.__init__(m)
    m.config = R.GPTDolomiteConfig(vocab_size=V, n_embd=H, n_layer=1, n_head=4, tie_word_embeddings=tied)
    m._tied_word_embeddings = tied
    # resize_token_embeddings ends with tie_weights(), which in this transformers version cannot read the reference's list
    # form of `_tied_weights_keys`; the reference's tied model has no lm_head module, so tying changes nothing here
    m.tie_weights = lambda *args, **kwargs: None
    m.transformer = nn.Module()
    m.transformer.wte = R.ParameterizedEmbedding(V, H, std=0.02)
    with torch.no_grad():
        m.transformer.wte.weight.copy_(torch.randn(V, H, generator=g) * 0.02)
    if not tied:
        m.lm_head = R.ParameterizedLinear(H, V, bias=False, std=0.02)
        with torch.no_grad():
            m.lm_head.weight.copy_(torch.randn(V, H, generator=g) * 0.02)
    return m


def main() -> None:
    import types

    from oracle.validate_against_reference import import_reference

    import_reference()
    from dolomite_engine.hf_models import GPTDolomiteConfig
    from dolomite_engine.hf_models.models.gpt_dolomite.main import GPTDolomiteForCausalLM
    from dolomite_engine.hf_models.modeling_utils import ParameterizedEmbedding, ParameterizedLinear

    R = types.SimpleNamespace(GPTDolomiteConfig=GPTDolomiteConfig, GPTDolomiteForCausalLM=GPTDolomiteForCausalLM,
                              ParameterizedEmbedding=ParameterizedEmbedding, ParameterizedLinear=ParameterizedLinear)
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for name, (V, tied, seed) in CASES.items():
            tok = build_tokenizer(d, BASE_VOCAB)
            before = len(tok)
            tok.add_special_tokens({"additional_special_tokens": list(ADDED_TOKENS)})
            assert len(tok) != before
            V_new = len(tok)
            m = reference_model(R, V, tied, torch.Generator().manual_seed(1000 + seed))
            out[f"{name}_wte"] = m.transformer.wte.weight.detach().numpy().copy()
            if not tied:
                out[f"{name}_lm_head"] = m.lm_head.weight.detach().numpy().copy()
            torch.manual_seed(seed)
            m.resize_token_embeddings(V_new)
            out[f"{name}_after"] = torch.rand(8).numpy()
            assert m.config.vocab_size == V_new and m.transformer.wte.weight.shape == (V_new, H)
            out[f"{name}_new_wte"] = m.transformer.wte.weight.detach().numpy().copy()
            if not tied:
                out[f"{name}_new_lm_head"] = m.lm_head.weight.detach().numpy().copy()
            out[f"{name}_meta"] = np.array([V, before, V_new, int(tied), H, seed], dtype=np.int64)
            print(f"{name}: vocab_size {V} -> {V_new} (tokenizer {before} -> {V_new}), tied={tied}")
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
