"""`python -m dolomite_engine_b200.unshard --config unshard.yml` -- the reference's unshard.py: a training checkpoint
(`<load_path>/global_step<N>/model.pt`, or the DCP directory `model/` of `fsdp_algorithm: 2`, written by
`checkpointing.save_checkpoint` or by the reference)
-> a `save_pretrained` directory (safetensors with the reference's parameter names + config.json) that
`from_pretrained`, `export_to_huggingface` and the reference itself can read.  Pure CPU: no model is instantiated.

YAML (reference UnshardingArgs, arguments.py:506-517):
    load_args: {load_path: ..., iteration: null}
    unsharded_path: ...
"""

from __future__ import annotations

import argparse
import json
import os

import torch
import yaml

from .hf_models.config import config_class_for
from .utils.safetensors import SafeTensorsWeightsManager

_PREFIX = "model."
_CKPT_WRAPPER = "._checkpoint_wrapped_module"  # checkpointing.py:41 (activation-checkpoint wrapper in reference-written files)


def _read_model_state(base: str) -> dict[str, torch.Tensor]:
    """model.pt (fsdp_algorithm 1) or the torch.distributed.checkpoint directory model/ (fsdp_algorithm 2): the
    directory's metadata names every tensor and its global shape, whatever sharding wrote it"""
    if os.path.isfile(os.path.join(base, "model.pt")):
        return torch.load(os.path.join(base, "model.pt"), map_location="cpu")
    import torch.distributed.checkpoint as dcp
    from torch.distributed.checkpoint import FileSystemReader
    from torch.distributed.checkpoint.metadata import TensorStorageMetadata

    path = os.path.join(base, "model")
    md = FileSystemReader(path).read_metadata().state_dict_metadata
    state = {k: torch.empty(tuple(m.size), dtype=m.properties.dtype) for k, m in md.items() if isinstance(m, TensorStorageMetadata)}
    dcp.load(state, checkpoint_id=path, no_dist=True)
    return state


def unshard(load_path: str, unsharded_path: str, iteration: int | None = None, dtype: str | None = None) -> str:
    if iteration is None:
        iteration = json.load(open(os.path.join(load_path, "latest_checkpointed_iteration.json")))["latest_checkpointed_iteration"]
    base = os.path.join(load_path, f"global_step{iteration}")
    state = _read_model_state(base)
    training_config = yaml.safe_load(open(os.path.join(base, "training_config.yml")))
    pretrained_config = (training_config.get("model_args") or {}).get("pretrained_config")
    if pretrained_config is None:
        raise ValueError(f"{base}/training_config.yml carries no model_args.pretrained_config; cannot write config.json")
    config = config_class_for(pretrained_config.get("model_type", "gpt_dolomite")).from_dict(dict(pretrained_config))
    out = {}
    for k, v in state.items():
        k = k.replace(_CKPT_WRAPPER, "")
        if not k.startswith(_PREFIX):
            raise KeyError(f"unexpected key {k!r} in model.pt (expected the ModelWrapper prefix '{_PREFIX}')")
        t = v.detach()
        if dtype is not None:
            t = t.to(getattr(torch, dtype))
        out[k[len(_PREFIX):]] = t.contiguous()
    # a run with tokenizer_args.additional_special_tokens resized the vocabulary after building from pretrained_config
    config.vocab_size = int(out["transformer.wte.weight"].shape[0])
    os.makedirs(unsharded_path, exist_ok=True)
    SafeTensorsWeightsManager.save_state_dict(out, unsharded_path)
    config.save_pretrained(unsharded_path)
    return unsharded_path


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", required=True)
    a = ap.parse_args()
    cfg = yaml.safe_load(open(a.config))
    la = cfg.get("load_args") or {}
    if not la.get("load_path") or not cfg.get("unsharded_path"):
        raise ValueError("unshard config needs load_args.load_path and unsharded_path")
    mp = (cfg.get("mixed_precision_args") or {}).get("dtype")
    dtype = {"fp32": "float32", "bf16": "bfloat16", "fp16": "float16"}.get(mp) if mp else None
    print(unshard(la["load_path"], cfg["unsharded_path"], la.get("iteration"), dtype))


if __name__ == "__main__":
    main()
