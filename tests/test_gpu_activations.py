"""GPU: the MLP activation kernels (every function x form) against the activation oracle, and models with the new
activations against the CPU oracle with the bars of test_gpu_model.py (dense) and test_gpu_moe.py (MoE)."""

import numpy as np
import pytest
import torch

import act_oracle
import oracle.dolomite_oracle as O
from dolomite_engine_b200 import activations as A

pytestmark = pytest.mark.gpu

CASES = [(i, f) for i in range(23) for f in (A.PLAIN, A.GLU)] + [(A.SIGMOID, A.SIGMOID_GLU)]
# the non-differentiable points of each function, where dx must carry torch autograd's value exactly
KINKS = {A.RELU: [0.0], A.RELU2: [0.0], A.RELU6: [0.0, 6.0], A.HARDTANH: [-1.0, 1.0], A.HARDSWISH: [-3.0, 3.0],
         A.HARDSIGMOID: [-3.0, 3.0], A.HARDSHRINK: [-0.5, 0.5], A.SOFTSHRINK: [-0.5, 0.5], A.LEAKY_RELU: [0.0],
         A.SOFTPLUS: [20.0, 20.125], A.ELU: [0.0], A.CELU: [0.0], A.SELU: [0.0]}


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _k():
    from dolomite_engine_b200 import kernels

    return kernels


def _inputs(T, F, form, seed):
    g = torch.Generator().manual_seed(seed)
    W = F if form == A.PLAIN else 2 * F
    x = (torch.randn(T, W, generator=g) * 3).bfloat16()
    kinks = torch.tensor([0.0, 0.5, -0.5, 1.0, -1.0, 3.0, -3.0, 6.0, 20.0, 20.125]).bfloat16()
    n = min(kinks.numel(), F)
    x[0, W - n :] = kinks[:n]  # kink points in the (gate) columns of the first row
    dy = torch.randn(T, F, generator=g).bfloat16()
    return x, dy


@pytest.mark.parametrize("T,F", [(77, 256), (1000, 328), (8, 8)])
@pytest.mark.parametrize("act_id,form", CASES)
def test_kernel_forward_backward_and_bias_gradient(act_id, form, T, F):
    K = _k()
    x, dy = _inputs(T, F, form, seed=act_id * 7 + form)
    y = K.act_fwd(x.cuda(), act_id, form).cpu().float()
    ref16 = act_oracle.apply(x.float(), act_id, form, bf16=True)
    assert y.shape == (T, F)
    # within 2 bf16 ulp, relative to max(|ref|, 1)
    err = (y - ref16).abs() / ref16.abs().clamp(min=1.0)
    assert err.max().item() <= 2 * 2.0**-7, (err.max().item(), torch.nonzero(err == err.max())[0].tolist())

    xf = x.float().requires_grad_(True)
    (act_oracle.apply(xf, act_id, form) * dy.float()).sum().backward()
    dx = K.act_bwd(dy.cuda(), x.cuda(), act_id, form)
    assert rel_l2(dx, xf.grad) <= 5e-3, rel_l2(dx, xf.grad)

    # kink points: dy = 1 (and u = 1) there, so dx is bf16(f'(x)) and must equal the oracle's (autograd's) value
    kinks = KINKS.get(act_id, [])
    if kinks:
        x2, dy2 = x.clone(), torch.ones_like(dy)
        if form != A.PLAIN:
            x2[:, :F] = 1.0
        x2f = x2.float().requires_grad_(True)
        act_oracle.apply(x2f, act_id, form).sum().backward()
        dx2 = K.act_bwd(dy2.cuda(), x2.cuda(), act_id, form).cpu()
        gate = x2[:, -F:].float()
        at = torch.zeros_like(gate, dtype=torch.bool)
        for k in kinks:
            at |= gate == torch.tensor(k).bfloat16().float()
        if at.any():
            got, want = dx2[:, -F:].float()[at], x2f.grad[:, -F:].bfloat16().float()[at]
            assert torch.equal(got, want), (got.tolist(), want.tolist())

    # the fused bias gradient: identical dx, and += the column sums of the bf16 dx on top of the buffer's contents
    W = x.shape[1]
    db0 = torch.randn(W, generator=torch.Generator().manual_seed(3)).cuda()
    db = db0.clone()
    dxf = K.act_bwd(dy.cuda(), x.cuda(), act_id, form, bias_grad_accum=db)
    assert torch.equal(dxf, dx)
    want = db0.double() + dx.double().sum(0)
    bound = 1e-5 * (dx.double().abs().sum(0) + db0.double().abs()) + 1e-6  # fp32 sums of T terms
    assert ((db.double() - want).abs() <= bound).all()


def test_existing_entry_points_are_the_same_kernels():
    K = _k()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(300, 2 * 264, generator=g).bfloat16().cuda()
    dy = torch.randn(300, 264, generator=g).bfloat16().cuda()
    assert torch.equal(K.swiglu_fwd(x), K.act_fwd(x, A.SILU, A.GLU))
    assert torch.equal(K.swiglu_bwd(dy, x), K.act_bwd(dy, x, A.SILU, A.GLU))
    a, b = torch.zeros(528, device="cuda"), torch.zeros(528, device="cuda")
    assert torch.equal(K.swiglu_bwd(dy, x, bias_grad_accum=a), K.act_bwd(dy, x, A.SILU, A.GLU, bias_grad_accum=b))
    assert torch.equal(a, b)
    xg = x[:, :264].contiguous()
    assert torch.equal(K.gelu_fwd(xg), K.act_fwd(xg, A.GELU_TANH, A.PLAIN))
    assert torch.equal(K.gelu_bwd(dy, xg), K.act_bwd(dy, xg, A.GELU_TANH, A.PLAIN))


# ---------------------------------------------------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------------------------------------------------
DENSE = {
    "bigcode_gelu": dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_head=8, n_inner=512,
                         attention_head_type="mqa", activation_function="gelu", add_bias=True,
                         normalization_function="layernorm", position_embedding_type="learned_absolute"),
    "gelu_tanh_glu_gqa_bias": dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_head=8,
                                   num_key_value_heads=2, n_inner=256, attention_head_type="gqa",
                                   activation_function="gelu_pytorch_tanh_glu", add_bias=True),
    "relu2": dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=1, n_head=4, n_inner=512, attention_head_type="mha",
                  activation_function="relu2", add_bias=False),
    "glu": dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=1, n_head=4, n_inner=256, attention_head_type="mha",
                activation_function="glu", add_bias=True),
}


@pytest.fixture(autouse=True)
def _oracle_activations():
    act_oracle.install()


def _dense_model(monkeypatch, name):
    """test_gpu_model's checks, run on one more configuration"""
    import test_gpu_model as M

    monkeypatch.setitem(M.GPU_CONFIGS, name, DENSE[name])
    return M


@pytest.mark.parametrize("name", list(DENSE))
@pytest.mark.parametrize("ragged", [False, True])
def test_dense_logits_and_loss_match_oracle(monkeypatch, name, ragged):
    _dense_model(monkeypatch, name).test_logits_and_loss_match_oracle(name, ragged)


@pytest.mark.parametrize("name", list(DENSE))
def test_dense_all_gradients_match_oracle(monkeypatch, name):
    _dense_model(monkeypatch, name).test_all_gradients_match_oracle(name)


def _moe_model(act, E=16, n_inner=192):
    from dolomite_engine_b200.hf_models import MoEDolomiteConfig, MoEDolomiteForCausalLM

    kw = dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_head=8, n_inner=n_inner, attention_head_type="mha",
              add_bias=False, num_experts=E, num_experts_per_tok=2, activation_function=act)
    ocfg = O.OracleConfig(**kw)
    cfg = MoEDolomiteConfig(position_embedding_type="rope", normalization_function="rmsnorm", resid_pdrop=0, embd_pdrop=0,
                            attn_pdrop=0, eos_token_id=7, **kw)
    params = O.init_params(ocfg, seed=42)
    model = MoEDolomiteForCausalLM(cfg, seed=None)
    model.load_state_dict(params)
    return model, ocfg, params


def _poison_allocator():
    """fill the free blocks of torch's caching allocator with NaN, so that buffers the MoE path allocates (grouped
    activations, padding rows) start as NaN"""
    big = torch.full((64 << 20,), float("nan"), dtype=torch.float32, device="cuda")
    del big
    small = [torch.full((1 << 16,), float("nan"), dtype=torch.float32, device="cuda") for _ in range(256)]
    del small


@pytest.mark.parametrize("act,ragged", [("reglu", False), ("reglu", True), ("softplus", True)])
def test_moe_logits_loss_and_grads_match_oracle(act, ragged):
    """MoE (16 experts, top-2) with reglu, and with softplus (f(0) = ln 2: padding rows of the grouped activation are not
    zero) on ragged routing with the grouped buffers starting as NaN"""
    model, ocfg, params = _moe_model(act)
    model.assume_unit_loss_grad = True
    rng = np.random.default_rng(3)
    tokens = rng.integers(0, ocfg.vocab_size, size=(2, 97), dtype=np.int64)
    tokens[0, 30] = 7
    tokens[1, 60] = 7
    inp, labels = O.split_tokens(tokens)
    b = O.prepare_model_inputs(inp.copy(), 7, ragged, ragged)
    args = (torch.from_numpy(b["input_ids"]).cuda(), torch.from_numpy(b["position_ids"]).cuda(),
            torch.from_numpy(b["cu_seqlens"]).cuda(), b["max_seqlen"])
    model.engine.zero_grad()
    lab = torch.from_numpy(np.ascontiguousarray(labels).reshape(-1)).cuda()
    if act == "softplus":
        _poison_allocator()
    loss = model.forward_pretraining_loss(*args, lab)
    saved = model.engine._saved["layers"]
    routing = {f"transformer.h.{i}.mlp.": layer[-1][0].sel_idx.long().cpu() for i, layer in enumerate(saved)}
    if act == "softplus":
        counts = saved[0][-1][0].counts.cpu()
        assert bool(((counts % 128) != 0).any()), "routing gives no padded segment"
    loss.backward()
    out = model(input_ids=args[0], position_ids=args[1], cu_seqlens=args[2], max_seqlen=args[3])
    logits = out.logits.float().cpu().detach()
    assert torch.isfinite(logits).all()
    O.FORCED_ROUTING.clear()
    O.FORCED_ROUTING.update(routing)
    try:
        p_req = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        loss_ref, logits_ref = O.pretraining_loss(p_req, ocfg, tokens, 7, ragged, ragged, bf16=True)
        loss_ref.backward()
    finally:
        O.FORCED_ROUTING.clear()
    assert rel_l2(logits, logits_ref.detach()) < 1e-2
    assert abs(loss.item() - loss_ref.item()) / loss_ref.item() < 1e-3
    # test_gpu_moe's bar is 3e-2.  ReLU's derivative is a step: an expert pre-activation whose bf16 value lands on the
    # other side of 0 than the oracle's flips a whole entry of dx (measured on an H100: 3.3e-2 for reglu's
    # ln_2 / c_fc gradients of layer 1), so the ReLU-gated MoE gets 5e-2.
    bar = 5e-2 if act == "reglu" else 3e-2
    bad = []
    for pname, unit, spec in model.engine.named_views():
        g = unit.gviews[pname]
        assert torch.isfinite(g).all(), pname
        e = rel_l2(g, p_req[pname].grad)
        if e > bar:
            bad.append((pname, round(e, 4)))
    assert not bad, bad


def test_bigcode_gelu_checkpoint_imports_and_matches_transformers(tmp_path):
    """a gpt_bigcode checkpoint with exact-erf GELU (transformers, random weights on CPU) imports and runs"""
    from transformers import GPTBigCodeConfig, GPTBigCodeForCausalLM

    from dolomite_engine_b200.hf_models import AutoModelForCausalLM, import_from_huggingface

    torch.manual_seed(0)
    hf_cfg = GPTBigCodeConfig(vocab_size=512, n_positions=128, n_embd=128, n_layer=2, n_head=4, n_inner=512,
                              activation_function="gelu", multi_query=True, resid_pdrop=0.0, embd_pdrop=0.0,
                              attn_pdrop=0.0)
    hf = GPTBigCodeForCausalLM(hf_cfg).eval()
    src, dst = tmp_path / "hf", tmp_path / "dolomite"
    hf.save_pretrained(src, safe_serialization=True)
    import_from_huggingface(str(src), str(dst))
    model = AutoModelForCausalLM.from_pretrained(str(dst))
    assert model.config.activation_function == "gelu"
    ids = torch.randint(0, 512, (2, 40), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        want = hf(input_ids=ids).logits.float()
    got = model(input_ids=ids.tolist()).logits.detach().float().cpu().view(want.shape)  # padding-free: rows are packed
    # the bf16 engine against transformers in fp32.  rtol / atol 5e-3 do not hold for every element (largest difference
    # measured on an H100: 6.5e-3, at a logit of 0.27), so the bars are those test_gpu_model.py puts on the bf16 engine
    # against the fp32 oracle, and rtol / atol 5e-3 for 99 % of the logits
    close = torch.isclose(got, want, rtol=5e-3, atol=5e-3).float().mean().item()
    err, rel = (got - want).abs().max().item(), rel_l2(got, want)
    print(f"gelu bigcode vs transformers: {close:.4f} within 5e-3, max |diff| {err:.2e}, rel-L2 {rel:.2e}")
    assert close > 0.99 and err < 4e-2 and rel < 1e-2


def _engine(act="gelu_pytorch_tanh_glu", **kw):
    from test_fp8 import _cfg

    from dolomite_engine_b200.engine import DolomiteEngine

    cfg = _cfg(num_key_value_heads=2, vocab_size=1024, n_layer=2, activation_function=act, add_bias=True, **kw)
    return DolomiteEngine(cfg, "cuda", seed=42)


def test_training_steps_bit_identical_and_checkpointing_exact():
    from test_gpu_fp8 import _batch, _grads, _step

    runs = []
    for ck in (None, None, 1):
        eng = _engine()
        eng.checkpoint_every = ck
        losses = [_step(eng, _batch(1024, seed=s), False, lr=0.05) for s in range(2)]
        runs.append((losses, _grads(eng)))
    (l1, g1), (l2, g2), (l3, g3) = runs
    assert l1 == l2 == l3
    assert all(torch.equal(g1[n], g2[n]) for n in g1)
    assert all(torch.equal(g1[n], g3[n]) for n in g1)


def test_fp8_gelu_tanh_glu_tracks_bf16():
    from test_gpu_fp8 import _batch, _step

    eng = _engine()
    eng.enable_fp8()
    losses = [_step(eng, _batch(1024, seed=s % 4), True, lr=0.05) for s in range(30)]
    ref = _engine()
    ref_losses = [_step(ref, _batch(1024, seed=s % 4), False, lr=0.05) for s in range(30)]
    assert ref_losses[-1] < ref_losses[0] - 0.2 and losses[-1] < losses[0] - 0.2
    assert abs(losses[-1] - ref_losses[-1]) / ref_losses[-1] <= 2e-2


def test_greedy_decoding_gelu_tanh_glu_equals_stepwise_argmax(monkeypatch):
    import test_zzz_generation as G

    monkeypatch.setattr(G, "CFG", dict(G.CFG, activation_function="gelu_pytorch_tanh_glu", add_bias=True))
    G.test_greedy_generation_equals_stepwise_argmax(True)
