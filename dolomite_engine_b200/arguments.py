"""`--config <yaml>` argument tree of the reference's entry points (arguments.py:30-547, utils/pydantic.py:7-8,
utils/yaml.py:6-23) restricted to the knobs of the data-parallel path.  Same section / key names, same
`extra="forbid"` strictness; keys that select out-of-scope subsystems are accepted only at their default values and
raise NotImplementedError otherwise, so an existing reference YAML either runs or fails loudly.

The schema is ONE table (`_SCHEMA`: section -> {key: (type, default)}); the pydantic classes are generated from it and
the per-section rules live in `_RULES`.  Two additions (SURVEY.md section 5 quirk): `model_args.moe_implementation` and
`model_args.normalization_implementation` are accepted because the reference's own configs/testing/scattermoe.yml sets
them although its ModelArgs rejects them; `distributed_args.reshard_after_forward` is a B200 extension."""

from __future__ import annotations

import re
from argparse import ArgumentParser
from typing import Any, Callable, Optional

import yaml
from pydantic import BaseModel, ConfigDict, create_model

_RULES: dict[str, Callable[[Any], None]] = {}


class BaseArgs(BaseModel):
    model_config = ConfigDict(extra="forbid", protected_namespaces=())

    def model_post_init(self, __context: Any) -> None:
        rule = _RULES.get(type(self).__name__)
        if rule is not None:
            rule(self)


def load_yaml(file_path: str) -> dict:
    """utils/yaml.py:6-23: PyYAML follows YAML 1.1, where `1e-5` is a string; teach the loader the 1.2 float grammar"""
    floats = re.compile(r"""^(?:
        [-+]?(?:[0-9][0-9_]*)\.[0-9_]*(?:[eE][-+]?[0-9]+)?     # 1.5, 1.5e3
       |[-+]?(?:[0-9][0-9_]*)(?:[eE][-+]?[0-9]+)               # 1e-5
       |\.[0-9_]+(?:[eE][-+][0-9]+)?                           # .5
       |[-+]?[0-9][0-9_]*(?::[0-5]?[0-9])+\.[0-9_]*            # sexagesimal
       |[-+]?\.(?:inf|Inf|INF)
       |\.(?:nan|NaN|NAN))$""", re.X)

    class Loader(yaml.SafeLoader):
        pass

    Loader.add_implicit_resolver("tag:yaml.org,2002:float", floats, list("-+0123456789."))
    with open(file_path) as f:
        return yaml.load(f, Loader)


def _need(obj, *names: str) -> None:
    for n in names:
        assert getattr(obj, n) is not None, f"{n} cannot be None"


def _check_not_None(pairs) -> None:
    for obj, name in pairs:
        assert obj is not None, f"{name} cannot be None"


# ------------------------------------------------------------------------------------------------
# schema: section -> {key: (annotation, default)}.  `None` defaults of non-Optional keys mark required keys
# (checked by the section's rule, like the reference's `_check_not_None`).
# ------------------------------------------------------------------------------------------------
O = Optional
_SCHEMA: dict[str, dict[str, tuple]] = {
    "RandomArgs": {"seed": (int, 42)},
    "TokenizerArgs": {"tokenizer_name": (O[str], None), "additional_special_tokens": (O[list[str]], None)},
    "ModelArgs": {
        "model_name": (O[str], None), "pretrained_config": (O[dict], None), "model_class": (str, None),
        "trust_remote_code": (bool, False), "attention_implementation": (O[str], None),
        "use_padding_free_transformer": (bool, False), "efficient_initialization": (bool, False),
        "reset_attention_mask": (bool, False), "reset_position_ids": (bool, False),
        "moe_implementation": (O[str], None), "normalization_implementation": (O[str], None)},
    "TuningArgs": {"tuning_method": (str, None), "prompt_tuning_args": (O[dict], None), "lora_args": (O[dict], None)},
    "TrainingParameters": {
        "ignore_sampling_proportion_for_validation": (bool, False), "num_training_steps": (O[int], None),
        "gradient_accumulation_steps": (int, 1), "eval_interval": (O[int], None), "micro_batch_size": (int, None),
        "eval_during_training": (bool, True), "loss_mask": (str, "output_only"), "gradient_clipping": (O[float], 1)},
    "SaveArgs": {"save_path": (str, None), "save_interval": (int, None), "save_optimizer": (bool, True)},
    "LoadArgs": {
        "load_path": (str, None), "iteration": (O[int], None), "load_optimizer": (bool, True), "load_lr_scheduler": (bool, True),
        "load_rng_state": (bool, True), "load_dataloader_state": (bool, True), "load_experiments_tracker_state": (bool, True),
        "load_starting_iteration": (bool, True), "resume_learning_rate": (bool, True)},
    "DatasetArgs": {
        "class_name": (str, None), "class_args": (dict, {}), "data_name": (str, None), "input_format": (str, "__input__"),
        "output_format": (str, "__output__"), "data_sampling_ratio": (O[int], None), "max_input_tokens": (O[int], None),
        "max_output_tokens": (O[int], None)},
    "OptimizerArgs": {
        "class_name": (str, "TorchAdamW"), "params_group_method": (O[str], None),
        "class_args": (dict, {"lr": 1e-5, "weight_decay": 0.1, "betas": [0.9, 0.95], "eps": 1e-10})},
    "LRSchedulerArgs": {
        "num_warmup_steps": (int, 200), "num_constant_steps": (int, 0), "num_decay_steps": (O[int], None),
        "lr_decay_style": (str, "cosine"), "lr_decay_factor": (float, 0.1), "extra_lr_scheduler_args": (dict, {})},
    "MixedPrecisionArgs": {"dtype": (str, "fp32"), "fp8_backend": (O[str], None)},
    "ZeroTopologyArgs": {"data_parallel_replication_world_size": (O[int], None), "data_parallel_sharding_world_size": (O[int], None)},
    "DistributedArgs": {
        "stage": (int, 3), "distributed_backend": (str, "torch"), "overlap_comm": (bool, False),
        "contiguous_gradients": (bool, False), "cpu_offload": (bool, False), "gradient_checkpointing_method": (O[str], None),
        "gradient_checkpointing_args": (dict, {}), "zero_topology": ("ZeroTopologyArgs", "new"),
        "zero_quantized_weights": (bool, False), "zero_quantized_gradients": (bool, False), "communication_dtype": (O[str], None),
        "torch_compile": (bool, False), "dispatching_dataloader": (bool, False), "tensor_parallel_size": (int, 1),
        "tensor_parallel_word_embeddings": (bool, False), "sequence_parallel": (bool, False),
        "data_parallel_size": (O[int], None), "timeout_minutes": (O[int], None), "fsdp_algorithm": (int, 1),
        "reshard_after_forward": (O[bool], None)},
    "LoggingArgs": {
        "logging_level": (str, "INFO"), "log_interval": (int, 1), "aim_args": (O[dict], None), "wandb_args": (O[dict], None),
        "experiments_tracker_name": (O[str], None), "use_colored_logs": (bool, False), "torch_profiler_trace_path": (O[str], None)},
    "ResearchArgs": {"neft_alpha": (O[float], None)},
    "GenerationParameters": {
        "batch_size": (int, None), "do_sample": (O[bool], None), "max_new_tokens": (int, None), "temperature": (O[float], None),
        "top_k": (O[int], None), "top_p": (O[float], None)},
    # ---- roots (arguments.py:405-517): section members are written ("<Section>", "new" | None | "list") ----
    "TrainingArgs": {
        "random_args": ("RandomArgs", "new"), "tokenizer_args": ("TokenizerArgs", "new"), "model_args": ("ModelArgs", None),
        "tuning_args": ("TuningArgs", None), "optimizer_args": ("OptimizerArgs", "new"),
        "lr_scheduler_args": ("LRSchedulerArgs", "new"), "datasets": ("DatasetArgs", "list"), "save_args": ("SaveArgs", None),
        "load_args": ("LoadArgs", None), "training_parameters": ("TrainingParameters", None),
        "logging_args": ("LoggingArgs", "new"), "mixed_precision_args": ("MixedPrecisionArgs", "new"),
        "distributed_args": ("DistributedArgs", "new"), "research_args": ("ResearchArgs", "new")},
    "InferenceArgs": {
        "random_args": ("RandomArgs", "new"), "tokenizer_args": ("TokenizerArgs", "new"), "model_args": ("ModelArgs", None),
        "datasets": ("DatasetArgs", "list"), "load_args": ("LoadArgs", None),
        "generation_parameters": ("GenerationParameters", None), "mixed_precision_args": ("MixedPrecisionArgs", "new"),
        "logging_args": ("LoggingArgs", "new"), "output_dir": (str, None)},
    "UnshardingArgs": {
        "load_args": ("LoadArgs", None), "unsharded_path": (str, None), "mixed_precision_args": ("MixedPrecisionArgs", "new"),
        "logging_args": ("LoggingArgs", "new")},
}


def _generate() -> dict[str, type[BaseArgs]]:
    made: dict[str, type[BaseArgs]] = {}
    for section, keys in _SCHEMA.items():  # sections are listed before the roots that embed them
        fields = {}
        for key, (kind, default) in keys.items():
            if isinstance(kind, str):  # an embedded section
                sub = made[kind]
                if default == "new":
                    fields[key] = (sub, sub())
                elif default == "list":
                    fields[key] = (list[sub], [])
                else:
                    fields[key] = (Optional[sub], None)
            else:
                fields[key] = (kind, default)
        made[section] = create_model(section, __base__=BaseArgs, __module__=__name__, **fields)
    return made


globals().update(_generate())


# ------------------------------------------------------------------------------------------------
# per-section rules (the reference's model_post_init bodies, plus the out-of-scope guards of this path)
# ------------------------------------------------------------------------------------------------
def _rule(section: str):
    def register(fn):
        _RULES[section] = fn
        return fn

    return register


@_rule("ModelArgs")
def _(a) -> None:
    _need(a, "model_class")
    if a.model_name is None:
        _need(a, "pretrained_config")
    else:
        assert a.pretrained_config is None, "pretrained_config shouldn't be specified with model_name"
    assert a.model_class in ["AutoModelForCausalLM", "AutoModelForSeq2SeqLM"], f"unexpected model_class ({a.model_class})"
    if a.model_class != "AutoModelForCausalLM":
        raise NotImplementedError("only AutoModelForCausalLM is on the B200 hot path")


@_rule("TuningArgs")
def _(a) -> None:
    _need(a, "tuning_method")
    if a.tuning_method not in ("pretraining", "full_finetuning"):
        raise NotImplementedError(f"tuning_method={a.tuning_method}: PEFT is out of scope of the B200 hot path")


@_rule("TrainingParameters")
def _(a) -> None:
    _need(a, "num_training_steps", "micro_batch_size")
    if a.eval_during_training:
        _need(a, "eval_interval")


@_rule("SaveArgs")
def _(a) -> None:
    _need(a, "save_path", "save_interval")


@_rule("DatasetArgs")
def _(a) -> None:
    assert a.class_name is not None, "dataset class_name cannot be None"
    _need(a, "data_name")


@_rule("MixedPrecisionArgs")
def _(a) -> None:
    a.dtype = {"bfloat16": "bf16", "float32": "fp32", "float16": "fp16", "float8": "fp8"}.get(a.dtype, a.dtype)
    if a.fp8_backend is not None:
        # arguments.py:278-280 of the reference
        assert a.dtype == "fp8", "fp8_backend can only be used with fp8 dtype"
        a.fp8_backend = str(getattr(a.fp8_backend, "value", a.fp8_backend))
        if a.fp8_backend == "msamp":
            raise NotImplementedError("fp8_backend msamp is not implemented; use nvte (TransformerEngine delayed scaling)")
        if a.fp8_backend != "nvte":
            raise ValueError(f"unexpected fp8_backend ({a.fp8_backend})")
    elif a.dtype == "fp8":
        raise ValueError("dtype fp8 needs an fp8_backend (nvte)")


_OUT_OF_SCOPE_FLAGS = ("cpu_offload", "zero_quantized_weights", "zero_quantized_gradients", "torch_compile",
                       "dispatching_dataloader", "tensor_parallel_word_embeddings", "sequence_parallel")


@_rule("DistributedArgs")
def _(a) -> None:
    if a.distributed_backend != "torch":
        raise NotImplementedError("no DeepSpeed / multi-backend dispatch on the B200 path (north_star)")
    for flag in _OUT_OF_SCOPE_FLAGS:
        if getattr(a, flag):
            raise NotImplementedError(f"distributed_args.{flag} is out of scope of the data-parallel B200 path")
    if a.tensor_parallel_size != 1:
        raise NotImplementedError("tensor parallelism is out of scope of the data-parallel B200 path")
    if a.gradient_checkpointing_method is not None:
        # the reference's GradientCheckpointingMethod enum has the single member `block`
        if str(a.gradient_checkpointing_method).split(".")[-1] != "block":
            raise ValueError(f"unexpected gradient_checkpointing_method ({a.gradient_checkpointing_method})")
        extra = set(a.gradient_checkpointing_args) - {"checkpoint_every", "use_reentrant", "block_name"}
        if extra:
            raise ValueError(f"unexpected gradient_checkpointing_args {sorted(extra)}")
    zt = a.zero_topology
    if (zt.data_parallel_replication_world_size is None) != (zt.data_parallel_sharding_world_size is None):
        raise AssertionError("data_parallel_replication_world_size and data_parallel_sharding_world_size go together")
    if a.communication_dtype is not None:
        a.communication_dtype = {"bfloat16": "bf16", "float32": "fp32"}.get(a.communication_dtype, a.communication_dtype)
        assert a.communication_dtype in ("bf16", "fp32")


@_rule("GenerationParameters")
def _(a) -> None:
    _need(a, "batch_size", "max_new_tokens")


@_rule("TrainingArgs")
def _(a) -> None:
    _need(a, "model_args", "tuning_args", "save_args")
    assert a.datasets, "datasets cannot be None"
    if a.mixed_precision_args.dtype not in ("bf16", "fp8"):
        raise NotImplementedError("the B200 path trains in bf16 mixed precision, optionally with FP8 linears "
                                  "(mixed_precision_args.dtype: bf16 | fp8)")


@_rule("InferenceArgs")
def _(a) -> None:
    assert a.datasets, "datasets cannot be None"
    _need(a, "generation_parameters", "output_dir")
    if a.load_args is None:
        assert a.model_args is not None, "model_args need to be specified if load_args are not specified"
    else:
        assert a.model_args is None, "model_args can't be specified with load_args"


@_rule("UnshardingArgs")
def _(a) -> None:
    _need(a, "load_args", "unsharded_path")


GenerationParameters.to_dict = lambda self: self.model_dump()  # noqa: E731,F821  (reference: BaseArgs.to_dict)

_MODE_ARGS = {"training": TrainingArgs, "inference": InferenceArgs, "unsharding": UnshardingArgs}  # noqa: F821


def get_args_from_dict(config: dict, mode=None):
    return _MODE_ARGS[str(getattr(mode, "value", mode) or "training")](**config)


def get_args(mode=None):
    """arguments.py:527-547; `mode` is "training" (default), "inference" or "unsharding" (enums.Mode values)"""
    parser = ArgumentParser()
    parser.add_argument("--config", type=str, required=True, help="path for the config")
    a = parser.parse_args()
    return get_args_from_dict(load_yaml(a.config), mode)
