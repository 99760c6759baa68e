"""CPU: host-side logic of the drop-in boundary -- config surface, YAML argument tree, integer bookkeeping (bit-exact
against the oracle), flat-unit layout, LR schedules, safetensors manager."""

import os

import numpy as np
import pytest
import torch

import oracle.dolomite_oracle as O
from dolomite_engine_b200.arguments import get_args_from_dict, load_yaml
from dolomite_engine_b200.engine import FlatUnit, _block_specs, _root_specs, check_supported
from dolomite_engine_b200.hf_models import GPTDolomiteConfig, MoEDolomiteConfig
from dolomite_engine_b200.hf_models.config import CommonConfig
from dolomite_engine_b200.hf_models.utils import prepare_pretraining_inputs_host
from dolomite_engine_b200.optimization import get_scheduler

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_config_defaults_aliases_and_validation(tmp_path):
    c = GPTDolomiteConfig()
    assert c.n_inner == 4 * c.n_embd and c.attention_head_type == "mqa" and c.num_key_value_heads == 1
    assert c.hidden_size == c.n_embd and c.num_hidden_layers == c.n_layer and c.max_position_embeddings == c.n_positions
    c2 = GPTDolomiteConfig(hidden_size=128, num_attention_heads=8, attention_head_type="gqa", num_key_value_heads=2)
    assert c2.n_embd == 128 and c2.n_head == 8
    with pytest.raises(AssertionError):
        GPTDolomiteConfig(attention_head_type="gqa")
    with pytest.raises(AssertionError):
        GPTDolomiteConfig(attention_head_type="mha", n_head=8, num_key_value_heads=2)
    with pytest.raises(ValueError):
        GPTDolomiteConfig(position_embedding_type="bogus")
    c2.save_pretrained(str(tmp_path))
    c3 = CommonConfig.from_pretrained(str(tmp_path))
    assert isinstance(c3, GPTDolomiteConfig) and c3.to_dict() == c2.to_dict()
    m = MoEDolomiteConfig(num_experts=4, num_experts_per_tok=1, n_embd=64, n_head=4, attention_head_type="mha")
    assert m.model_type == "moe_dolomite" and m.to_dict()["num_experts"] == 4


def test_unsupported_configs_fail_loudly():
    ok = GPTDolomiteConfig(n_embd=256, n_head=4, attention_head_type="mha", position_embedding_type="rope",
                           activation_function="swiglu", normalization_function="rmsnorm", resid_pdrop=0, embd_pdrop=0,
                           attn_pdrop=0, vocab_size=2048)
    check_supported(ok)
    for kw in (dict(position_embedding_type="alibi"), dict(normalization_function="apex_layernorm"),
               dict(activation_function="geglu"), dict(n_head=32, num_key_value_heads=32),
               dict(rope_scaling={"type": "linear", "factor": 2, "original_max_position_embeddings": 64})):
        d = ok.to_dict()
        d.update(kw)
        with pytest.raises(NotImplementedError):
            check_supported(GPTDolomiteConfig.from_dict(d))
    # the StarCoder / bigcode shape of the reference's example YAMLs (configs/pretraining-examples/*.yml, dropout 0)
    d = ok.to_dict()
    d.update(position_embedding_type="learned_absolute", normalization_function="layernorm",
             activation_function="gelu_pytorch_tanh", attention_head_type="mqa", num_key_value_heads=1, add_bias=True)
    check_supported(GPTDolomiteConfig.from_dict(d))
    d.update(m_emb=12.0)  # (wte + wpe) * m_emb: the scale is a separate pass after the sum (tests/test_gpu_dropout.py "bigcode")
    check_supported(GPTDolomiteConfig.from_dict(d))


@pytest.mark.parametrize("ram,rpi", [(False, False), (True, False), (True, True)])
def test_pretraining_bookkeeping_bit_exact(ram, rpi):
    rng = np.random.default_rng(3)
    for _ in range(5):
        tokens = rng.integers(0, 50, size=(3, 65), dtype=np.int64)
        eos = 7
        inp, lab = O.split_tokens(tokens)
        ref = O.prepare_model_inputs(inp.copy(), eos, ram, rpi)
        got = prepare_pretraining_inputs_host(tokens, eos, ram, rpi)
        assert np.array_equal(got["input_ids"], ref["input_ids"])
        assert np.array_equal(got["labels"], np.ascontiguousarray(lab).reshape(-1))
        assert np.array_equal(got["cu_seqlens"], ref["cu_seqlens"]) and got["cu_seqlens"].dtype == np.int32
        assert np.array_equal(got["position_ids"], ref["position_ids"])
        assert got["position_ids"].dtype == ref["position_ids"].dtype
        assert got["max_seqlen"] == ref["max_seqlen"]


def test_bookkeeping_edge_cases():
    # every token is EOS -> documents of length 1; and EOS at the row boundary
    tokens = np.full((2, 9), 7, dtype=np.int64)
    got = prepare_pretraining_inputs_host(tokens, 7, True, True)
    assert np.array_equal(got["cu_seqlens"], np.arange(0, 17, dtype=np.int32))
    assert got["max_seqlen"] == 1 and np.all(got["position_ids"] == 0)
    tokens = np.arange(18, dtype=np.int64).reshape(2, 9) + 100
    got = prepare_pretraining_inputs_host(tokens, 7, True, True)
    assert np.array_equal(got["cu_seqlens"], np.array([0, 8, 16], dtype=np.int32)) and got["max_seqlen"] == 8


def test_flat_unit_layout_and_sharding():
    cfg = GPTDolomiteConfig(n_embd=64, n_head=4, n_layer=2, n_inner=128, vocab_size=256, attention_head_type="gqa",
                            num_key_value_heads=2, add_bias=True, activation_function="swiglu",
                            normalization_function="rmsnorm", position_embedding_type="rope")
    specs = _block_specs(cfg, 0)
    names = [s[0] for s in specs]
    assert names[0] == "transformer.h.0.ln_1.weight" and "transformer.h.0.mlp.c_fc.bias" in names
    shapes = dict((s[0], s[1]) for s in specs)
    assert shapes["transformer.h.0.attn.c_attn.weight"] == (64 + 2 * 2 * 16, 64)  # H + 2*nkv*hd
    assert shapes["transformer.h.0.mlp.c_fc.weight"] == (256, 64)  # 2F for GLU
    for ws in (1, 2, 8):
        u = FlatUnit("h.0", specs, world_size=ws, rank=0)
        assert u.padded % (ws * 64) == 0 and u.shard_numel * ws == u.padded
        offs = [(s.offset, s.numel) for s in u.specs]
        for (o1, n1), (o2, _) in zip(offs, offs[1:]):
            assert o1 + n1 <= o2 and o2 % 64 == 0  # no overlap, 128-byte aligned
    assert [s[0] for s in _root_specs(cfg)] == ["transformer.wte.weight", "transformer.ln_f.weight"]
    cfg.tie_word_embeddings = False
    assert _root_specs(cfg)[-1][0] == "lm_head.weight"
    # config defaults = the GPT-2 / bigcode shape: LayerNorm biases and the learned position table join the units (appended,
    # so the layout of the rope / rmsnorm configurations above is a prefix of it)
    big = GPTDolomiteConfig(n_embd=64, n_head=4, n_layer=2, vocab_size=256, n_positions=128, add_bias=True)
    assert [s[0] for s in _root_specs(big)] == ["transformer.wte.weight", "transformer.ln_f.weight", "transformer.ln_f.bias",
                                                "transformer.wpe.weight"]
    bnames = [s[0] for s in _block_specs(big, 1)]
    assert bnames[-2:] == ["transformer.h.1.ln_1.bias", "transformer.h.1.ln_2.bias"]
    assert dict((s[0], s[1]) for s in _block_specs(big, 1))["transformer.h.1.mlp.c_fc.weight"] == (256, 64)  # F, not 2F


def test_yaml_argument_tree():
    a = get_args_from_dict(load_yaml(os.path.join(ROOT, "configs", "c2_granite3b_shape.yml")))
    assert a.model_args.pretrained_config["n_embd"] == 2560 and a.optimizer_args.class_args["lr"] == 1e-5
    assert a.datasets[0].class_args["sequence_length"] == 4096
    bad = load_yaml(os.path.join(ROOT, "configs", "c1_tiny.yml"))
    bad["model_args"]["bogus_key"] = 1
    with pytest.raises(Exception):  # extra="forbid"
        get_args_from_dict(bad)
    ds = load_yaml(os.path.join(ROOT, "configs", "c1_tiny.yml"))
    ds["distributed_args"]["distributed_backend"] = "deepspeed"
    with pytest.raises(NotImplementedError):
        get_args_from_dict(ds)


def test_cosine_schedule_matches_reference_formula():
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([p], lr=1.0)
    s = get_scheduler(opt, 4, 2, None, 20, "cosine", 0.1)
    lrs = []
    for _ in range(22):
        lrs.append(s.get_last_lr()[0])
        opt.step()
        s.step()
    assert lrs[0] == 0 and abs(lrs[4] - 1.0) < 1e-12 and abs(lrs[6] - 1.0) < 1e-12
    import math

    x, t = 10 - 6, 20 - 6
    assert abs(lrs[10] - (0.9 * (1 + math.cos(math.pi * x / t)) / 2 + 0.1)) < 1e-12
    assert abs(lrs[21] - 0.1) < 1e-12


def test_safetensors_manager_roundtrip(tmp_path):
    from dolomite_engine_b200.utils.safetensors import SafeTensorsWeightsManager

    sd = {"a.weight": torch.randn(4, 8), "b.bias": torch.arange(5, dtype=torch.float32)}
    SafeTensorsWeightsManager.save_state_dict(sd, str(tmp_path))
    m = SafeTensorsWeightsManager(str(tmp_path))
    assert len(m) == 2 and m.has_tensor("a.weight") and list(m.get_shape("a.weight")) == [4, 8]
    assert torch.equal(m.get_tensor("b.bias"), sd["b.bias"]) and m == SafeTensorsWeightsManager(str(tmp_path))


def test_product_path_never_imports_the_oracle():
    import subprocess
    import sys

    code = ("import sys; import dolomite_engine_b200.engine, dolomite_engine_b200.kernels, dolomite_engine_b200.distributed, "
            "dolomite_engine_b200.model_wrapper, dolomite_engine_b200.pretrain, dolomite_engine_b200.hf_models; "
            "assert not any(m.startswith('oracle') for m in sys.modules), 'oracle imported by the product path'")
    subprocess.run([sys.executable, "-c", code], check=True, cwd=ROOT)


def test_no_gpu_means_loud_failure():
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from dolomite_engine_b200.hf_models import GPTDolomiteForCausalLM

    cfg = GPTDolomiteConfig(n_embd=256, n_head=4, attention_head_type="mha", position_embedding_type="rope",
                            activation_function="swiglu", normalization_function="rmsnorm", resid_pdrop=0, embd_pdrop=0,
                            attn_pdrop=0, vocab_size=2048, n_layer=1)
    with pytest.raises(RuntimeError, match="no CPU path"):
        GPTDolomiteForCausalLM(cfg)


def test_gradient_checkpointing_args_follow_the_reference_surface():
    """distributed_args.gradient_checkpointing_method: block + gradient_checkpointing_args.checkpoint_every
    (arguments.py:312-314, gradient_checkpointing/__init__.py)"""
    d = load_yaml(os.path.join(ROOT, "configs", "c1_tiny.yml"))
    d["distributed_args"]["gradient_checkpointing_method"] = "block"
    d["distributed_args"]["gradient_checkpointing_args"] = {"checkpoint_every": 2}
    a = get_args_from_dict(d)
    assert a.distributed_args.gradient_checkpointing_args["checkpoint_every"] == 2
    d["distributed_args"]["gradient_checkpointing_method"] = "selective"
    with pytest.raises(Exception):
        get_args_from_dict(d)


def test_rope_tables_plain_and_yarn_equal_the_pinned_oracle_tables():
    """engine._setup_rope restates RoPE / YaRNScaledRoPE (position_embedding/rope.py:9-101); the oracle's tables are pinned
    bit-exactly against the reference classes (oracle/validate_against_reference.py), the engine's must equal them in bf16"""
    import torch

    import oracle.dolomite_oracle as O
    from dolomite_engine_b200.engine import DolomiteEngine

    for rs, theta in [(None, 10000), ({"type": "yarn", "factor": 4.0, "original_max_position_embeddings": 64}, 10000),
                      ({"factor": 8.0, "original_max_position_embeddings": 128}, 500000)]:
        cfg = GPTDolomiteConfig(n_embd=320, n_head=4, n_layer=1, n_inner=640, vocab_size=256, n_positions=512,
                                attention_head_type="mha", position_embedding_type="rope", activation_function="swiglu",
                                normalization_function="rmsnorm", resid_pdrop=0, embd_pdrop=0, attn_pdrop=0, rope_theta=theta,
                                rope_scaling=rs)
        eng = DolomiteEngine(cfg, "cpu", seed=None)
        cos, sin = O.rope_tables(80, 512, theta, bf16=True, rope_scaling=rs)
        assert torch.equal(eng.rope_cos.float(), cos) and torch.equal(eng.rope_sin.float(), sin)
    with pytest.raises(ValueError):
        check_supported(GPTDolomiteConfig.from_dict({**cfg.to_dict(), "rope_scaling": {"factor": 2.0}}))


def test_every_shipped_config_parses():
    """configs/*.yml follow the reference's TrainingArgs tree (extra=forbid): C1, C2/C3, C4 (MoE), C5 (Llama-3-8B finetune)"""
    names = sorted(f for f in os.listdir(os.path.join(ROOT, "configs")) if f.endswith(".yml"))
    assert {"c1_tiny.yml", "c2_granite3b_shape.yml", "c4_moe_8x_top2.yml", "c5_llama3_8b_finetune.yml"} <= set(names)
    for f in names:
        a = get_args_from_dict(load_yaml(os.path.join(ROOT, "configs", f)))
        assert a.training_parameters.micro_batch_size >= 1
    a = get_args_from_dict(load_yaml(os.path.join(ROOT, "configs", "c5_llama3_8b_finetune.yml")))
    assert a.distributed_args.gradient_checkpointing_args == {"checkpoint_every": 2} and a.model_args.model_name


def test_dropout_mask_generator_host_side():
    """dropout masks are counter-based: (pass seed, call site) -> two 32-bit keys (kernels.dropout_keys, restated by the
    oracle's DropoutOracle), element index -> keep bit.  Host-side properties: the keys of the product and of the oracle agree,
    sites / passes give different masks, the keep rate is 1 - p, the kept scale is 1 / (1 - p); eval mode draws no seed."""
    import numpy as np
    import torch

    import oracle.dolomite_oracle as O
    from dolomite_engine_b200.engine import DolomiteEngine
    from dolomite_engine_b200.hf_models import GPTDolomiteConfig
    from dolomite_engine_b200.kernels import dropout_keys

    for seed in (0, 1, 12345678901234567):
        for site in (0, 1, 7, 130):
            assert O.DropoutOracle(seed).keys(site) == dropout_keys(seed, site)
    d = O.DropoutOracle(99)
    m1, m2 = d.flat_scale(1, (4096, 64), 0.1), d.flat_scale(2, (4096, 64), 0.1)
    assert abs(float((m1 > 0).float().mean()) - 0.9) < 5e-3 and abs(float(m1.max()) - 1 / 0.9) < 1e-6
    assert 0.75 < float(((m1 > 0) == (m2 > 0)).float().mean()) < 0.89  # independent masks agree on 0.9^2 + 0.1^2 = 0.82
    assert not torch.equal(O.DropoutOracle(100).flat_scale(1, (4096, 64), 0.1), m1)
    a = d.attn_scale(3, 5, np.arange(1000, 1400), np.arange(1000, 1400), 0.25)
    assert abs(float((a > 0).float().mean()) - 0.75) < 1e-2
    assert not torch.equal(a, d.attn_scale(3, 6, np.arange(1000, 1400), np.arange(1000, 1400), 0.25))  # per head
    assert torch.equal(a[10:20, 30:50], d.attn_scale(3, 5, np.arange(1010, 1020), np.arange(1030, 1050), 0.25))  # position based
    assert d.threshold(0.0) == 0 and float((d.flat_scale(0, (1000,), 0.0) == 1.0).float().mean()) == 1.0

    cfg = GPTDolomiteConfig(n_embd=64, n_head=4, n_layer=1, vocab_size=264, n_positions=64)  # the reference's defaults: pdrop 0.1
    engine = DolomiteEngine(cfg, "cpu", seed=1)
    assert engine.has_dropout and engine.training
    engine.dropout_seed = 7
    engine._begin_dropout_pass()
    first = engine._dropout_now
    engine._begin_dropout_pass()
    assert first == 7 and engine._dropout_now == 8 and engine._drop_p("attn_pdrop") == pytest.approx(0.1)
    engine.training = False
    engine._begin_dropout_pass()
    assert engine._dropout_now is None and engine._drop_p("resid_pdrop") == 0.0
    assert not DolomiteEngine(GPTDolomiteConfig(n_embd=64, n_head=4, n_layer=1, vocab_size=264, resid_pdrop=0, embd_pdrop=0,
                                                attn_pdrop=0), "cpu", seed=1).has_dropout


def test_profiler_hook_and_throughput_helper(tmp_path):
    """logging_args.torch_profiler_trace_path (train_utils.py:182-194) and the B tokens/day figure of the step log"""
    from dolomite_engine_b200.train_utils import billion_tokens_per_day, get_torch_profiler

    assert get_torch_profiler(None) is None
    prof = get_torch_profiler(str(tmp_path / "trace"), rank=0, wait=1, warmup=1)
    with prof:
        for _ in range(4):
            sum(range(1000))
            prof.step()
    assert any(f.endswith(".json") or f.endswith(".json.gz") for f in os.listdir(tmp_path / "trace"))  # one traced step
    # 6 x 4096 tokens every 0.5625 s on 8 GPUs
    assert billion_tokens_per_day(8 * 6 * 4096, 0.5625) == pytest.approx(8 * 6 * 4096 * 86400 / 0.5625 / 1e9)


def test_lr_schedules_match_the_reference_sequences():
    """optimization/scheduler.py:50-219 incl. the Granite `power` schedule: learning-rate sequences produced BY THE REFERENCE's
    module (oracle/pin_lr_schedules.py -> tests/golden/lr_schedules.json), reproduced bit for bit"""
    import json

    import torch

    from dolomite_engine_b200.optimization import get_scheduler

    cases = json.load(open(os.path.join(ROOT, "tests", "golden", "lr_schedules.json")))
    assert {c["style"] for c in cases} == {"constant", "cosine", "exponential", "linear", "power"}
    for c in cases:
        opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=c["lr"])
        sched = get_scheduler(opt, c["warmup"], c["constant"], c["decay"], 40, c["style"], 0.1, c["extra"])
        got = []
        for _ in range(len(c["values"])):
            got.append(sched.get_last_lr()[0])
            opt.step()
            sched.step()
        assert got == c["values"], c["style"]
    with pytest.raises(ValueError):
        get_scheduler(torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=1.0), 1, 0, None, 10, "step", 0.1)
    with pytest.raises(AssertionError):
        get_scheduler(torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=1.0), 1, 2, None, 10, "power", 0.1,
                      {"a": 1.0, "b": -0.5, "c": 1.0})


def test_config_surface_matches_the_reference_classes():
    """defaults and constructor checks of CommonConfig / MoEDolomiteConfig as produced by the REFERENCE's classes
    (oracle/pin_config_surface.py -> tests/golden/config_surface.json)"""
    import json

    from dolomite_engine_b200.hf_models.config import CommonConfig, MoEDolomiteConfig

    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "config_surface.json")))
    for cls, key in ((CommonConfig, "common_defaults"), (MoEDolomiteConfig, "moe_defaults")):
        c = cls()
        for k, v in gold[key].items():
            assert getattr(c, k) == v, (key, k)
    probe = ("num_key_value_heads", "n_inner", "n_embd", "n_head", "n_layer", "n_positions", "multi_query")
    for case in gold["grid"]:
        for cls, key in ((CommonConfig, "common"), (MoEDolomiteConfig, "moe")):
            try:
                c = cls(**case["kwargs"])
                got = {k: getattr(c, k, None) for k in probe}
            except Exception as e:  # noqa
                got = {"error": type(e).__name__}
            want = case[key]
            if case["alias"]:  # aliases are resolved BEFORE the derived defaults here, after them in the reference (see the pin script)
                got, want = ({k: d.get(k) for k in ("n_embd", "n_head", "n_layer", "n_positions")} for d in (got, want))
            assert got == want, (case["kwargs"], key, got)


def test_yaml_schema_matches_the_reference_sections():
    """every section / key / default of the reference's arguments.py (oracle/pin_arguments_schema.py ->
    tests/golden/arguments_schema.json) exists here with the same default; the only additions are the documented ones"""
    import json

    from dolomite_engine_b200 import arguments as A

    def plain(v):
        if hasattr(type(v), "model_fields"):
            return {k: plain(getattr(v, k)) for k in type(v).model_fields}
        return [plain(x) for x in v] if isinstance(v, (list, tuple)) else v

    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "arguments_schema.json")))
    additions = {"ModelArgs": {"moe_implementation", "normalization_implementation"}, "DistributedArgs": {"reshard_after_forward"}}
    nested_elsewhere = {"AimArgs", "LoRAArgs", "PromptTuningArgs", "WandBArgs"}  # accepted as plain dicts (out-of-scope subsystems)
    assert set(gold) - nested_elsewhere == set(A._SCHEMA)
    for section, keys in gold.items():
        if section in nested_elsewhere:
            continue
        fields = getattr(A, section).model_fields
        assert set(fields) - additions.get(section, set()) == set(keys), section
        for k, default in keys.items():
            mine = plain(fields[k].default)
            if isinstance(mine, dict) and isinstance(default, dict):  # embedded section: ignore the documented additions
                mine = {kk: vv for kk, vv in mine.items() if kk in default}
            assert mine == default, (section, k)


def test_model_tflops_formula_with_checkpointed_blocks():
    """train_utils.py:197-236 (checked against the reference function on a grid while pinning): recomputed blocks add
    `fraction` forward passes to the 2x backward"""
    from dolomite_engine_b200.hf_models import GPTDolomiteConfig
    from dolomite_engine_b200.train_utils import get_model_tflops

    c = GPTDolomiteConfig(n_embd=2560, n_head=32, n_layer=32, n_inner=10240, vocab_size=49152, attention_head_type="mha",
                          activation_function="swiglu")
    b, s, h, f, v, l = 6, 4096, 2560, 10240, 49152, 32
    fwd = 4 * b * s * h * (h * 2 + s) + 6 * b * s * h * f
    assert get_model_tflops(c, b, s) == pytest.approx((l * 3 * fwd + 6 * b * s * h * v) / 1e12)
    assert get_model_tflops(c, b, s, checkpointed_fraction=0.5) == pytest.approx((l * 3.5 * fwd + 6 * b * s * h * v) / 1e12)


def test_init_rules_match_the_reference_block_modules():
    """std of every weight and the shape of every block parameter as constructed by the REFERENCE's GPTDolomiteBlock
    (oracle/pin_init_rules.py -> tests/golden/init_rules.json) == engine._block_specs"""
    import json

    from dolomite_engine_b200.engine import _block_specs
    from dolomite_engine_b200.hf_models import GPTDolomiteConfig

    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "init_rules.json")))
    for name, case in gold.items():
        kw = {"normalization_function": "rmsnorm", **case["config"]}
        cfg = GPTDolomiteConfig(vocab_size=264, n_positions=64, position_embedding_type="rope", resid_pdrop=0, embd_pdrop=0,
                                attn_pdrop=0, **kw)
        specs = {n[len("transformer.h.1."):]: (shape, init) for n, shape, init in _block_specs(cfg, 1)}
        assert {k: list(v[0]) for k, v in specs.items()} == case["shapes"], name
        for pname, std in case["std"].items():
            kind, _, value = specs[pname][1].partition(":")
            assert kind == "normal" and float(value) == pytest.approx(std, rel=1e-12), (name, pname)
        for pname, (shape, init) in specs.items():
            if pname.endswith(".bias"):
                assert init == "zeros", (name, pname)
            elif pname.startswith("ln_"):
                assert init == "ones", (name, pname)


def test_root_parameter_init_rules():
    """gpt_dolomite/base.py:136, :528 and main.py:19-21: wte, wpe and an untied lm_head are all drawn with
    std = initializer_range -- the muP width scaling applies to the block projections only"""
    from dolomite_engine_b200.engine import _root_specs
    from dolomite_engine_b200.hf_models import GPTDolomiteConfig

    cfg = GPTDolomiteConfig(n_embd=64, n_head=4, n_layer=2, vocab_size=264, n_positions=32, init_method="mup", m_width=4.0,
                            initializer_range=0.1, tie_word_embeddings=False, position_embedding_type="learned_absolute",
                            normalization_function="layernorm")
    specs = {n: (tuple(s), i) for n, s, i in _root_specs(cfg)}
    assert specs["transformer.wte.weight"] == ((264, 64), "normal:0.1")
    assert specs["lm_head.weight"] == ((264, 64), "normal:0.1")
    assert specs["transformer.wpe.weight"] == ((32, 64), "normal:0.1")
    assert specs["transformer.ln_f.weight"][1] == "ones" and specs["transformer.ln_f.bias"][1] == "zeros"


def test_stage3_slot_table_never_hands_a_live_buffer_away():
    """distributed._SlotTable: the ownership bookkeeping of the shared parameter buffers of the stage-3 (reshard) mode.
    Replays the engine's hook order (forward: prefetch depth 1; backward: re-gather i and i-1) for several depths / slot
    counts and checks that the buffer a block computes from holds that block's parameters, and that the slot given to a
    prefetch never belongs to the block being computed."""
    from dolomite_engine_b200.distributed import _SlotTable

    for n_layer in (1, 2, 3, 4, 7):
        for n_slots in (2, 3):
            n = n_layer + 1
            t = _SlotTable([False] + [True] * n_layer, n_slots)
            gathers = []

            def issue(i, busy=()):
                if t.is_fresh(i):
                    return
                prev = t.claim(i)
                assert prev not in busy, (n_layer, n_slots, i, prev, busy)
                t.fresh[i] = True  # (the wait happens before use)
                gathers.append(i)

            for step in range(2):
                t.invalidate()  # optimizer step: every gathered copy is stale
                gathers.clear()
                for i in range(n):  # forward
                    issue(i)
                    if i + 1 < n:
                        issue(i + 1, busy=(i,))
                    assert t.is_fresh(i)
                fwd = len(gathers)
                assert fwd == n  # one all-gather per unit
                for i in reversed(range(1, n)):  # backward (root is not pooled and stays gathered)
                    issue(i)
                    if i - 1 >= 1:
                        issue(i - 1, busy=(i,))
                    assert t.is_fresh(i)
                # blocks still resident at the end of forward are not gathered again
                resident_at_end = min(n_slots, n_layer)
                assert len(gathers) - fwd == n_layer - resident_at_end
            assert t.is_fresh(0)


def test_lazy_gradient_clearing_bookkeeping(monkeypatch):
    """engine.zero_grad() leaves the buffers of weights whose FIRST gradient of a window comes from an overwriting weight-gradient GEMM
    untouched (`_lazy_zero`): dense linears, the tied head / embedding, 3-D expert weights.  Everything that is accumulated by
    reduction kernels or atomics is cleared: norm weights, biases, the MoE router, scatter-only embedding tables."""
    from dolomite_engine_b200.engine import DolomiteEngine

    common = dict(n_embd=256, n_head=4, n_layer=2, vocab_size=512, n_positions=64, attention_head_type="mha",
                  normalization_function="rmsnorm", activation_function="swiglu", resid_pdrop=0, embd_pdrop=0, attn_pdrop=0)
    moe = DolomiteEngine(MoEDolomiteConfig(num_experts=64, num_experts_per_tok=2, n_inner=64, add_bias=False,
                                           position_embedding_type="rope", **{**common, "n_embd": 1024, "n_head": 8}), "cpu", seed=None)
    for u in moe.units:
        u.grad_full.fill_(7.0)
    moe.zero_grad()
    fresh = set(moe._fresh_grads)
    assert "transformer.h.0.mlp.c_fc.weight" in fresh and "transformer.h.1.mlp.c_proj.weight" in fresh
    assert "transformer.h.0.attn.c_attn.weight" in fresh and "transformer.wte.weight" in fresh  # tied: the head's wgrad writes first
    gate = "transformer.h.0.mlp.gate.weight"  # 64 x 1024 elements = as large as a lazily cleared weight, but split-K ADDS into it
    assert moe.units[1].gviews[gate].numel() >= moe._LAZY_ZERO_MIN_NUMEL and gate not in fresh
    for name, unit, _ in moe.named_views():
        v = unit.gviews[name]
        assert bool((v == 7.0).all()) if name in fresh else bool((v == 0).all()), name
    assert moe.take_fresh("transformer.h.0.mlp.c_fc.weight") and not moe.take_fresh("transformer.h.0.mlp.c_fc.weight")

    dense = DolomiteEngine(GPTDolomiteConfig(n_inner=512, add_bias=True, position_embedding_type="learned_absolute",
                                             tie_word_embeddings=False, **{**common, "n_positions": 1024}), "cpu", seed=None)
    for u in dense.units:
        u.grad_full.fill_(7.0)
    dense.zero_grad()
    fresh = set(dense._fresh_grads)
    assert "lm_head.weight" in fresh and "transformer.h.1.mlp.c_fc.weight" in fresh
    # embedding tables that only ever receive scattered atomics start from zero; so do biases and norm weights
    for name in ("transformer.wte.weight", "transformer.wpe.weight", "transformer.h.0.mlp.c_fc.bias", "transformer.ln_f.weight"):
        assert name not in fresh and bool((dict((n, u.gviews[n]) for n, u, _ in dense.named_views())[name] == 0).all()), name

    monkeypatch.setenv("DOLO_EAGER_GRAD_ZERO", "1")  # A/B switch: every buffer is cleared, nothing is overwritten
    eager = DolomiteEngine(MoEDolomiteConfig(num_experts=8, num_experts_per_tok=2, n_inner=128, add_bias=False,
                                             position_embedding_type="rope", **common), "cpu", seed=None)
    eager.units[1].grad_full.fill_(7.0)
    eager.zero_grad()
    assert not eager._fresh_grads and bool((eager.units[1].grad_full[: eager.units[1].numel] == 0).all())


def test_lm_head_chunking_covers_the_token_rows_within_the_budget():
    """engine._head_chunk_rows: the LM head + cross entropy run chunk by chunk so that [T, V] logits never exist (DESIGN 8.1).
    Properties: chunks of `rows` rows cover T with no remainder beyond the last chunk, every chunk but the last has a multiple of 8
    rows (it is the contraction length of the head's weight-gradient GEMM), a chunk's bf16 logits stay within the budget
    (except the 8-row minimum), and the split is as even as the 8-row granularity allows."""
    from hypothesis import given, settings
    from hypothesis import strategies as st

    from dolomite_engine_b200.engine import DolomiteEngine

    @settings(max_examples=300, deadline=None)
    @given(T=st.integers(1, 200_000), V=st.sampled_from([8, 264, 2048, 49152, 50304, 128256, 262144]),
           budget=st.sampled_from([1 << 12, 1 << 20, 1 << 28, 1 << 30, 1 << 33]))
    def check(T, V, budget):
        rows = DolomiteEngine._head_chunk_rows(T, V, budget)
        assert 1 <= rows <= T
        n_chunks = -(-T // rows)
        assert rows == T or rows % 8 == 0
        assert rows * V * 2 <= budget or rows <= 8 or rows == T and T < 8  # 8 rows is the floor
        cap = max(8, budget // (2 * V) // 8 * 8)
        assert n_chunks >= -(-T // cap)  # never fewer chunks than the budget demands ...
        assert n_chunks == -(-T // cap) or rows % 8 == 0 and n_chunks - -(-T // cap) <= 1  # ... and at most one more (rounding rows up to 8)
        assert (n_chunks - 1) * rows < T  # the last chunk is not empty

    check()
    # the workloads of bench.py: C2 mbs 6 x 4096 tokens -> 3 chunks of 8192 rows (0.8 GB each); C5 8192 tokens -> 2 x 4096
    assert DolomiteEngine._head_chunk_rows(24576, 49152) == 8192
    assert DolomiteEngine._head_chunk_rows(8192, 128256) == 4096
