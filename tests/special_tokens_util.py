"""A word-level tokenizer built locally with `tokenizers` (no download), shared by tools/pin_special_tokens.py and the
tests of `tokenizer_args.additional_special_tokens`: tokens "t0" .. "t<n-3>", then <unk> and <|endoftext|> (eos)."""

from __future__ import annotations

import os

ADDED_TOKENS = ("<|system|>", "<|user|>", "<|assistant|>")


def build_tokenizer(directory: str, length: int):
    """save a tokenizer of `length` entries under `directory`/tok_<length> and return it loaded by AutoTokenizer"""
    from tokenizers import Tokenizer, models, pre_tokenizers
    from transformers import AutoTokenizer, PreTrainedTokenizerFast

    path = os.path.join(directory, f"tok_{length}")
    vocab = {f"t{i}": i for i in range(length - 2)}
    vocab.update({"<unk>": length - 2, "<|endoftext|>": length - 1})
    tk = Tokenizer(models.WordLevel(vocab, unk_token="<unk>"))
    tk.pre_tokenizer = pre_tokenizers.Whitespace()
    fast = PreTrainedTokenizerFast(tokenizer_object=tk, unk_token="<unk>", eos_token="<|endoftext|>")
    fast.save_pretrained(path)
    return AutoTokenizer.from_pretrained(path)
