"""CPU: MoE blocks of any expert count (1 to 256) and any width that is a multiple of 8.

The oracle reproduces the reference-derived fixtures of tools/pin_moe_shapes.py (eager SparseMoE layers with E 3, 20 and
1; two-layer MoEDolomite models with E 6 / top-2 and E 12 / top-8), check_supported accepts those shapes and still
refuses the routing limits, the engine lays the parameters out under the reference's names and shapes, the router buffers
follow one layout rule, and a world-size-2 gloo run round-trips the flat layout of the E 6 model."""

import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import oracle.dolomite_oracle as O
from dolomite_engine_b200 import kernels as K
from dolomite_engine_b200.engine import DolomiteEngine, check_supported
from dolomite_engine_b200.hf_models import MoEDolomiteConfig
from moe_aux_oracle import forward_logits_with_router, load_balancing_loss
from moe_shapes_inputs import layer_inputs, subsample
from test_moe_bias import model_batches

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
LOGIT_ROW_STRIDE = 8
LAYERS = ["e3_k2", "e20_k4", "e1_k1"]
MODELS = {  # tools/pin_moe_shapes.py MODELS
    "e6_swiglu": dict(vocab_size=512, n_positions=256, n_embd=160, n_layer=2, n_head=5, n_inner=424,
                      attention_head_type="mha", activation_function="swiglu", add_bias=False, num_experts=6,
                      num_experts_per_tok=2, normalization_function="rmsnorm", position_embedding_type="rope"),
    "e12_gelu": dict(vocab_size=512, n_positions=256, n_embd=96, n_layer=2, n_head=3, n_inner=200,
                     attention_head_type="mha", activation_function="gelu_pytorch_tanh", add_bias=True, num_experts=12,
                     num_experts_per_tok=8, normalization_function="rmsnorm", position_embedding_type="learned_absolute"),
}


def layer_case(fx, name):
    """-> (oracle config, x, dy, params under prefix "m.") of one case of moe_shapes_layer.npz"""
    T, H, F, E, k = (int(v) for v in fx[f"{name}/shape"])
    act, bias = str(fx[f"{name}/activation"]), bool(fx[f"{name}/add_bias"])
    cfg = O.OracleConfig(vocab_size=256, n_embd=H, n_layer=1, n_head=H // 16, n_inner=F, num_experts=E,
                         num_experts_per_tok=k, add_bias=bias, activation_function=act)
    x, params = layer_inputs(T, H, F, E, act, bias, int(fx[f"{name}/seed"]))
    return cfg, x, torch.from_numpy(fx[f"{name}/dy"]), {"m." + n: v for n, v in params.items()}


def model_params(fx, name):
    cfg = O.OracleConfig(**MODELS[name])
    params = O.init_params(cfg, seed=int(fx["seed"]))
    for k in params:
        if k.endswith(".bias"):
            params[k] = torch.from_numpy(fx[f"bias:{k}"])
    return cfg, params


def hf_config(name, **kw):
    return MoEDolomiteConfig(**{**MODELS[name], "resid_pdrop": 0, "embd_pdrop": 0, "attn_pdrop": 0, "eos_token_id": 7, **kw})


@pytest.mark.parametrize("name", LAYERS)
def test_oracle_reproduces_the_layer_fixture(name):
    fx = np.load(os.path.join(GOLDEN, "moe_shapes_layer.npz"))
    cfg, x, dy, params = layer_case(fx, name)
    assert cfg.n_embd % 64 and cfg.n_inner % 64  # widths with K tails in the grouped GEMMs
    p = {n: v.clone().requires_grad_(True) for n, v in params.items()}
    x = x.requires_grad_(True)
    y, logits = O.sparse_moe(x, p, "m.", cfg)
    y.backward(dy)
    ref_y = torch.from_numpy(fx[f"{name}/y"])
    assert (y - ref_y).abs().max() <= 1e-5 * ref_y.abs().max()
    assert (logits - torch.from_numpy(fx[f"{name}/router_logits"])).abs().max() <= 1e-5
    ref = torch.from_numpy(fx[f"{name}/grad:x"])
    assert (x.grad - ref).abs().max() <= 1e-5 * ref.abs().max()
    names = {k.split("/grad:", 1)[1] for k in fx.files if k.startswith(f"{name}/grad:") and not k.endswith(":x")}
    assert names == {n[2:] for n in p}, sorted(names ^ {n[2:] for n in p})
    for n, v in p.items():
        got = subsample(v.grad) if v.dim() == 3 else v.grad
        ref = torch.from_numpy(fx[f"{name}/grad:{n[2:]}"])
        assert (got - ref).abs().max() <= 1e-5 * (ref.abs().max() + 1e-30), n


@pytest.mark.parametrize("name", list(MODELS))
def test_oracle_reproduces_the_model_fixture(name):
    fx = np.load(os.path.join(GOLDEN, f"moe_shapes_model_{name}.npz"))
    cfg, params = model_params(fx, name)
    for batch, (ids, pos, cu, labels) in model_batches(fx).items():
        p = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        logits = O.forward_logits(p, cfg, ids, pos, cu)
        loss = torch.nn.functional.cross_entropy(logits, torch.as_tensor(labels), ignore_index=-100)
        loss.backward()
        assert abs(loss.item() - float(fx[f"{batch}_loss"])) <= 1e-5, batch
        assert (logits[::LOGIT_ROW_STRIDE].detach() - torch.from_numpy(fx[f"{batch}_logits"])).abs().max() <= 2e-5, batch
        names = {k.split(":", 1)[1] for k in fx.files if k.startswith(f"{batch}_grad:")}
        assert names == set(p), sorted(names ^ set(p))
        for k, v in p.items():
            ref = torch.from_numpy(fx[f"{batch}_grad:{k}"])
            assert (subsample(v.grad) - ref).abs().max() <= 1e-4 * (ref.abs().max() + 1e-30), (batch, k)


@pytest.mark.parametrize("name", list(MODELS))
def test_oracle_reproduces_the_router_logits_and_aux_loss(name):
    fx = np.load(os.path.join(GOLDEN, f"moe_shapes_model_{name}.npz"))
    cfg, params = model_params(fx, name)
    ids, pos, cu, _ = model_batches(fx)["padded"]
    with torch.no_grad():
        _, router = forward_logits_with_router(params, cfg, ids, pos, cu)
    assert len(router) == cfg.n_layer
    for layer, r in enumerate(router):
        assert (r - torch.from_numpy(fx[f"padded_router_logits:{layer}"])).abs().max() <= 2e-5, layer
    aux = load_balancing_loss([r.double() for r in router], cfg.num_experts, cfg.num_experts_per_tok)
    assert abs(aux.item() - float(fx["padded_aux"])) <= 1e-6 * float(fx["padded_aux"])


def _moe(E=6, k=2, H=160, F=424, **kw):
    base = dict(vocab_size=512, n_positions=64, n_embd=H, n_layer=2, n_head=H // 32 if H % 32 == 0 else H // 16, n_inner=F,
                attention_head_type="mha", num_experts=E, num_experts_per_tok=k, position_embedding_type="rope",
                normalization_function="rmsnorm", activation_function="swiglu", resid_pdrop=0, embd_pdrop=0, attn_pdrop=0)
    return MoEDolomiteConfig(**{**base, **kw})


@pytest.mark.parametrize("E", [1, 3, 4, 6, 12, 20, 60, 256])
def test_check_supported_accepts_any_expert_count(E):
    check_supported(_moe(E=E, k=1))
    check_supported(_moe(E=E, k=min(8, E)))


@pytest.mark.parametrize("H,F", [(80, 72), (96, 80), (144, 96), (160, 424), (48, 1376), (208, 200)])
def test_check_supported_accepts_widths_that_are_multiples_of_8(H, F):
    assert H % 64 in (16, 32, 48) and F % 64 in (8, 16, 32, 40)
    for bias in (False, True):
        check_supported(_moe(H=H, F=F, add_bias=bias))


def test_check_supported_keeps_the_routing_and_width_limits():
    for kw in (dict(E=257, k=2), dict(E=6, k=9), dict(E=3, k=4), dict(E=16, k=0), dict(F=100), dict(F=430), dict(H=84, F=96)):
        with pytest.raises(NotImplementedError):
            check_supported(_moe(**kw))
    with pytest.raises(NotImplementedError, match="MoE blocks are implemented with rmsnorm"):
        check_supported(_moe(normalization_function="layernorm"))


@pytest.mark.parametrize("name", list(MODELS))
def test_engine_parameters_match_the_reference_names_and_shapes(name):
    fx = np.load(os.path.join(GOLDEN, f"moe_shapes_model_{name}.npz"))
    eng = DolomiteEngine(hf_config(name), "cpu", seed=1)
    shapes = {n: tuple(unit.views[n].shape) for n, unit, _ in eng.named_views()}
    ref_names = {k.split(":", 1)[1] for k in fx.files if k.startswith("packed_grad:")}  # the reference's named_parameters
    assert set(shapes) == ref_names, sorted(set(shapes) ^ ref_names)
    _, params = model_params(fx, name)
    assert shapes == {k: tuple(v.shape) for k, v in params.items()}
    E = MODELS[name]["num_experts"]
    assert shapes["transformer.h.0.mlp.gate.weight"] == (E, MODELS[name]["n_embd"])


@pytest.mark.parametrize("E", [1, 3, 6, 8, 12, 20, 60, 64, 256])
def test_router_buffer_layout_rule(E):
    """gate output (16-byte rows) -> contiguous [T, E] for the router kernels; router dlogits (contiguous) -> 16-byte
    rows for the gate GEMMs.  For E % 8 == 0 both are the tensor they were given (no copy)."""
    T = 37
    gate_out = K.rows_empty(T, E)
    gate_out.copy_(torch.randn(T, E))
    logits = K.router_logits(gate_out)
    assert logits.is_contiguous() and logits.stride() == (E, 1) and torch.equal(logits, gate_out)
    dl = torch.randn(T, E).bfloat16()
    staged = K.router_grad(dl)
    assert torch.equal(staged, dl) and staged.stride(1) == 1 and staged.stride(0) % 8 == 0 and staged.data_ptr() % 16 == 0
    if E % 8 == 0:
        assert logits is gate_out and staged is dl
    else:
        assert gate_out.stride(0) == -(-E // 8) * 8 and logits.data_ptr() != gate_out.data_ptr()
        assert staged.data_ptr() != dl.data_ptr()


def _gloo_worker(rank: int, world: int, port: int, q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dolomite_engine_b200.checkpointing import _named, _scatter_named
        from dolomite_engine_b200.engine import FlatUnit, _block_specs

        for E, add_bias in ((6, False), (3, True)):
            cfg = MoEDolomiteConfig(**{**MODELS["e6_swiglu"], "num_experts": E, "add_bias": add_bias})
            for i in range(cfg.n_layer):
                u = FlatUnit(f"h.{i}", _block_specs(cfg, i), world, rank)
                u.allocate("cpu")
                full = u.init_full(torch.Generator().manual_seed(42 + i))  # same seed on every rank
                u.full_master_from(full)
                assert u.shard_numel * world == u.padded and u.padded >= sum(s.numel for s in u.specs)
                for s in u.specs:  # every view starts on a 16-byte boundary of the bf16 buffer
                    assert s.offset % 8 == 0, s.name
                parts = [torch.empty(u.shard_numel) for _ in range(world)]
                dist.all_gather(parts, u.master.data)
                gathered = torch.cat(parts)
                assert torch.equal(gathered, full)
                named = _named(u, gathered)
                w = named[f"model.transformer.h.{i}.mlp.c_fc.weight"]  # checkpoint names
                assert tuple(w.shape) == (E, 2 * cfg.n_inner, cfg.n_embd)
                shard = torch.empty(u.shard_numel)
                _scatter_named(u, named, shard, "round trip")
                assert torch.equal(shard, u.master.data)
        q.put((rank, "ok"))
    except Exception:  # noqa
        import traceback

        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_world_size_2_flat_layout_round_trip_of_odd_expert_shapes():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = [q.get(timeout=240) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    for rank, status in results:
        assert status == "ok", f"rank {rank}: {status}"


def test_router_of_an_odd_expert_count_stays_bf16_under_fp8():
    """the gate runs as an FP8 linear only when E % 16 == 0 and n_embd % 16 == 0: the E 6 model keeps it in bf16"""
    from dolomite_engine_b200.fp8 import fp8_weight_names

    names = fp8_weight_names(hf_config("e6_swiglu"))
    assert "transformer.h.0.attn.c_attn.weight" in names
    assert not any(n.endswith("mlp.gate.weight") for n in names)
    assert "transformer.h.0.mlp.gate.weight" in fp8_weight_names(hf_config("e6_swiglu", num_experts=16))
