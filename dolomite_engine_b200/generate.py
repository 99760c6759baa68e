"""`python -m dolomite_engine_b200.generate --config <yaml>` -- the reference's generate.py (:14-143): for every
dataset, prompts are batched (`generation_parameters.batch_size`), left padded, decoded with `model.generate` and written
as one JSON line per example to `<output_dir>/output-<data_name>.jsonl`:

    {"generated_text": <str | token ids without a tokenizer>, "num_generated_tokens": <int, eos included>}

The model comes either from `model_args` (pretrained directory or config) or from a training checkpoint (`load_args`,
rebuilt from the `training_config.yml` stored with it).  Single GPU, like the reference.  Decoding re-runs the packed
forward per token (hf_models/generation.py): exact, no KV cache.
"""

from __future__ import annotations

import json
import os

import torch
import yaml

from .arguments import InferenceArgs, get_args
from .data.finetuning import JSONLinesSFTDataset, collate


def generate(args: InferenceArgs, model, datasets_list: list) -> None:
    """generate.py:14-68.  `datasets_list`: objects with `.data_name`, `__len__`, `__getitem__ -> {"input": [ids]}`"""
    gp = args.generation_parameters
    os.makedirs(args.output_dir, exist_ok=True)
    cfg = args.model_dump(mode="json") if hasattr(args, "model_dump") else dict(args)
    yaml.safe_dump(cfg, open(os.path.join(args.output_dir, "inference_config.yml"), "w"), indent=2)
    generate_kwargs = {k: v for k, v in gp.to_dict().items() if k != "batch_size"}
    for dataset in datasets_list:
        with open(os.path.join(args.output_dir, f"output-{dataset.data_name}.jsonl"), "w") as out:
            batch = []
            for index in range(len(dataset)):
                batch.append(dataset[index])
                if len(batch) == gp.batch_size or index == len(dataset) - 1:
                    collated = collate(batch, model.eos_token_id, use_padding_free_transformer=False, training=False)
                    texts, counts = model.generate(collated, dict(generate_kwargs))
                    for text, count in zip(texts, counts):
                        out.write(json.dumps({"generated_text": text, "num_generated_tokens": count}) + "\n")
                    batch = []


def build_datasets(args: InferenceArgs, tokenize, eos_token_id: int) -> list:
    out = []
    for ds in args.datasets:
        if "data_path" not in ds.class_args:
            raise NotImplementedError(f"dataset class {ds.class_name}: the B200 inference feed reads JSON-lines files "
                                      "(class_args.data_path)")
        d = JSONLinesSFTDataset(ds.class_args["data_path"], tokenize, eos_token_id, ds.input_format, ds.output_format,
                                ds.max_input_tokens, ds.max_output_tokens, training=False)
        d.data_name = ds.data_name
        out.append(d)
    return out


def main() -> None:
    args: InferenceArgs = get_args("inference")
    torch.cuda.set_device(0)  # generate.py:87: single GPU
    device = torch.device("cuda", 0)
    torch.manual_seed(args.random_args.seed)
    if args.load_args is None:
        from .model_wrapper import ModelWrapperForFinetuning

        m = args.model_args
        assert not m.efficient_initialization and not m.use_padding_free_transformer  # generate.py:90-91
        model = ModelWrapperForFinetuning(mode="inference", model_name=m.model_name, pretrained_config=m.pretrained_config,
                                          model_class=m.model_class, dtype=torch.bfloat16,
                                          attention_implementation=m.attention_implementation or "flash_attention_2",
                                          use_padding_free_transformer=False, random_seed=args.random_args.seed,
                                          tokenizer_name=args.tokenizer_args.tokenizer_name,
                                          additional_special_tokens=args.tokenizer_args.additional_special_tokens, device=device)
    else:
        from .checkpointing import load_checkpoint_for_inference

        model, _, _ = load_checkpoint_for_inference(args, "inference", device=device)
    if model.tokenizer is None:
        raise ValueError("generation from text needs a tokenizer: set tokenizer_args.tokenizer_name (or model_args.model_name) "
                         "to a local directory")
    tokenize = lambda text: model.tokenizer(text, add_special_tokens=False)["input_ids"]  # noqa: E731
    model.eval()
    generate(args, model, build_datasets(args, tokenize, model.eos_token_id))


if __name__ == "__main__":
    main()
