"""GPU: MoE experts with biases (ParameterizedExperts with add_bias, moe_dolomite/moe/base.py:12-50).

Kernels: the M-grouped expert GEMM with a per-expert bias (plain and gather-on-load) per element against fp64, and the
per-segment bias-gradient reductions against fp64 column sums.  Layer: the reference-derived fixture of
tools/pin_moe_bias.py.  Model: logits, loss and every gradient against the oracle with the GPU's routing pinned, packed
and padded batches; bit-identical repeats and block checkpointing; dropout; the load-balancing loss; FP8 mode; greedy
KV-cache decoding."""

import os

import numpy as np
import pytest
import torch

import oracle.dolomite_oracle as O
from test_moe_bias import layer_case, subsample

pytestmark = pytest.mark.gpu

F32_EPS = 2.0**-24
BF16_EPS = 2.0**-8  # one bf16 rounding: relative error <= 2^-9; the bar allows two


def K():
    from dolomite_engine_b200 import kernels

    return kernels


def bf(x):
    return x.to(torch.bfloat16)


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _plan(T, E, k, g, empty=()):
    logits = torch.randn(T, E, device="cuda", generator=g)
    for i, e in enumerate(empty):
        logits[:, e] = -1e4 * (i + 1)  # never among the top-k
    return K().moe_route(bf(logits), k)


# ---------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,E,k,H,N", [(5, 8, 1, 128, 192), (300, 8, 2, 256, 384), (1000, 64, 8, 128, 264),
                                       (8192, 8, 2, 512, 512), (2048, 64, 1, 256, 128), (777, 64, 2, 192, 136)])
def test_grouped_gemm_with_bias_vs_fp64(T, E, k, H, N):
    """D[row] = x[token] W[e]^T + b[e] on every real row, plain and gather-on-load, per element within two bf16 roundings of
    the result plus K fp32 roundoffs of sum |x w| + |b|; experts without tokens (E - 2, E - 1 when k < E - 2) are skipped;
    with a zero bias tensor the results equal the bias-free entry points bit for bit"""
    g = torch.Generator(device="cuda").manual_seed(T + E + k)
    empty = (E - 2, E - 1) if k < E - 2 else ()
    plan = _plan(T, E, k, g, empty)
    x = bf(torch.randn(T, H, device="cuda", generator=g))
    w = bf(torch.randn(E, N, H, device="cuda", generator=g) * 0.05)
    b = bf(torch.randn(E, N, device="cuda", generator=g) * 0.3)
    cnt = plan.counts.cpu()
    assert all(int(cnt[e]) == 0 for e in empty)
    real = plan.slot_of_row >= 0
    rows = torch.nonzero(real).flatten()
    tok = plan.token_of_row[rows].long()
    grp = plan.tile_group[rows // 128].long()
    exact = torch.einsum("rh,rnh->rn", x[tok].double(), w[grp].double()) + b[grp].double()
    mag = torch.einsum("rh,rnh->rn", x[tok].double().abs(), w[grp].double().abs()) + b[grp].double().abs()
    bar = BF16_EPS * exact.abs() + (H + 2) * F32_EPS * mag + 1e-30
    xg = K().moe_gather(x, plan)
    plain = K().gemm_grouped_m(xg, w, plan, b_mn=False, bias=b)
    gather = K().gemm_grouped_m_gather(x, w, plan, bias=b)
    for got in (plain, gather):
        err = (got[rows].double() - exact).abs()
        assert bool((err <= bar).all()), (err / bar).max().item()
    assert torch.equal(plain[real], gather[real])
    zero = torch.zeros_like(b)
    assert torch.equal(K().gemm_grouped_m(xg, w, plan, b_mn=False, bias=zero)[real], K().gemm_grouped_m(xg, w, plan, b_mn=False)[real])
    assert torch.equal(K().gemm_grouped_m_gather(x, w, plan, bias=zero)[real], K().gemm_grouped_m_gather(x, w, plan)[real])


def test_grouped_gemm_bias_rejects_bad_layouts():
    from dolomite_engine_b200 import _lib

    g = torch.Generator(device="cuda").manual_seed(0)
    plan = _plan(64, 8, 2, g)
    xg = K().moe_gather(bf(torch.randn(64, 64, device="cuda", generator=g)), plan)
    w = bf(torch.randn(8, 64, 64, device="cuda", generator=g))
    with pytest.raises(AssertionError):
        K().gemm_grouped_m(xg, w, plan, b_mn=False, bias=bf(torch.zeros(8, 32, device="cuda")))  # [E, N] only
    odd = bf(torch.zeros(8, 65, device="cuda"))[:, :64]  # row stride 65: a bias row would not be 4-byte aligned
    with pytest.raises(_lib.DolomiteB200Error, match="ld_bias"):
        K().gemm_grouped_m(xg, w, plan, b_mn=False, bias=odd)


def _segments(plan):
    off = plan.offsets.cpu().long()
    return [(int(off[e]), int(off[e + 1])) for e in range(plan.E)]


@pytest.mark.parametrize("T,E,k,N", [(5, 8, 1, 128), (600, 8, 2, 384), (3000, 64, 8, 264), (8192, 64, 2, 2048)])
def test_segmented_colsum_vs_fp64(T, E, k, N):
    """out[e] += scale * column sums of expert e's (padded) segment rows: within (rows + 24) fp32 roundoffs of fp64; an
    expert without rows keeps its out row bit for bit; repeats are byte-identical; accumulating adds to the buffer"""
    g = torch.Generator(device="cuda").manual_seed(T * 3 + N)
    plan = _plan(T, E, k, g, empty=(1, E - 1) if k < E - 2 else ())
    buf = bf(torch.randn(plan.max_rows, N + 8, device="cuda", generator=g))
    x = buf[:, :N]  # a row stride wider than N
    out0 = torch.randn(E, N, device="cuda", generator=g)
    scale = 0.71
    runs = []
    for _ in range(2):
        out = out0.clone()
        K().colsum_accum_segmented(x, plan.offsets, out, scale)
        runs.append(out)
    assert torch.equal(runs[0], runs[1])
    xd = x.double()
    for e, (s0, s1) in enumerate(_segments(plan)):
        if s1 == s0:
            assert torch.equal(runs[0][e], out0[e]), e  # exact zero contribution
            continue
        ref = out0[e].double() + scale * xd[s0:s1].sum(0)
        bar = (s1 - s0 + 24) * F32_EPS * (out0[e].double().abs() + scale * xd[s0:s1].abs().sum(0))
        assert bool(((runs[0][e].double() - ref).abs() <= bar).all()), e
    # accumulate (scale 1: out += s rounds once, like the addition of torch): into a zero buffer, then into out0
    s = torch.zeros(E, N, device="cuda")
    K().colsum_accum_segmented(x, plan.offsets, s)
    acc = out0.clone()
    K().colsum_accum_segmented(x, plan.offsets, acc)
    assert torch.equal(acc, out0 + s)


@pytest.mark.parametrize("act", ["swiglu", "gelu_pytorch_tanh", "softplus"])
@pytest.mark.parametrize("T,E,k,F", [(7, 8, 2, 64), (1500, 8, 2, 192), (4000, 64, 8, 256)])
def test_segmented_act_bwd_vs_fp64(act, T, E, k, F):
    """act_bwd_segmented writes the same dx as act_bwd on every segment row, and adds each segment's column sums of that
    bf16 dx to its bias-gradient row (fp32 bound as colsum); an empty expert's row is left bit for bit"""
    from dolomite_engine_b200.activations import resolve

    act_id, form = resolve(act)
    W = 2 * F if form != 0 else F
    g = torch.Generator(device="cuda").manual_seed(T + F)
    plan = _plan(T, E, k, g, empty=(0,) if k < E - 2 else ())
    dy = bf(torch.randn(plan.max_rows, F, device="cuda", generator=g))
    x = bf(torch.randn(plan.max_rows, W, device="cuda", generator=g))
    dx_ref = K().act_bwd(dy, x, act_id, form)
    out0 = torch.randn(E, W, device="cuda", generator=g)
    runs = []
    for _ in range(2):
        acc = out0.clone()
        dx = K().act_bwd_segmented(dy, x, act_id, form, plan.offsets, acc)
        runs.append((dx, acc))
    assert torch.equal(runs[0][1], runs[1][1])
    end = int(plan.offsets[-1])
    assert torch.equal(runs[0][0][:end], dx_ref[:end]) and torch.equal(runs[1][0][:end], dx_ref[:end])
    d = dx_ref.double()
    for e, (s0, s1) in enumerate(_segments(plan)):
        if s1 == s0:
            assert torch.equal(runs[0][1][e], out0[e]), e
            continue
        ref = out0[e].double() + d[s0:s1].sum(0)
        bar = (s1 - s0 + 24) * F32_EPS * (out0[e].double().abs() + d[s0:s1].abs().sum(0))
        assert bool(((runs[0][1][e].double() - ref).abs() <= bar).all()), e


# ---------------------------------------------------------------------------------------------------------------------
# layer
# ---------------------------------------------------------------------------------------------------------------------
def _layer_model(cfg):
    from dolomite_engine_b200.hf_models import MoEDolomiteConfig, MoEDolomiteForCausalLM

    hf = MoEDolomiteConfig(vocab_size=256, n_embd=cfg.n_embd, n_layer=1, n_head=4, n_inner=cfg.n_inner,
                           num_experts=cfg.num_experts, num_experts_per_tok=cfg.num_experts_per_tok, attention_head_type="mha",
                           add_bias=True, position_embedding_type="rope", normalization_function="rmsnorm",
                           activation_function=cfg.activation_function, resid_pdrop=0, embd_pdrop=0, attn_pdrop=0)
    return MoEDolomiteForCausalLM(hf, seed=0)


@pytest.mark.parametrize("name", ["e8_k2", "e16_k4"])
def test_moe_bias_layer_matches_golden(golden_dir, name):
    """the reference's eager SparseMoE with biases: output, dx and every parameter gradient within rel-L2 2e-2; the routing
    is the reference's (its router logits have no near-ties at bf16 resolution)"""
    from dolomite_engine_b200 import moe

    fx = np.load(os.path.join(golden_dir, "moe_bias_layer.npz"))
    cfg, x, dy, params = layer_case(fx, name)
    model = _layer_model(cfg)
    sd = model.state_dict()
    for n, v in params.items():
        sd["transformer.h.0.mlp." + n[2:]] = v
    model.load_state_dict(sd)
    eng = model.engine
    p = "transformer.h.0."
    eng.zero_grad()
    xc = bf(x).cuda()
    y, saved = moe.forward(eng, eng.units[1], p, xc, torch.zeros_like(xc), 1.0)
    ref_sel = torch.from_numpy(fx[f"{name}/router_logits"]).topk(cfg.num_experts_per_tok, dim=-1).indices
    assert torch.equal(saved[0].sel_idx.long().cpu().sort(-1).values, ref_sel.sort(-1).values)
    assert rel_l2(y, torch.from_numpy(fx[f"{name}/y"])) < 2e-2
    dx = moe.backward(eng, eng.units[1], p, xc, bf(dy).cuda(), 1.0, saved)
    torch.cuda.synchronize()
    assert rel_l2(dx, torch.from_numpy(fx[f"{name}/grad:x"])) < 2e-2
    for n in params:
        got = eng.units[1].gviews[p + "mlp." + n[2:]]
        got = subsample(got.cpu()) if got.dim() == 3 else got
        assert rel_l2(got, torch.from_numpy(fx[f"{name}/grad:{n[2:]}"])) < 2e-2, n


# ---------------------------------------------------------------------------------------------------------------------
# model
# ---------------------------------------------------------------------------------------------------------------------
def _cfgs(act="swiglu", E=8, **kw):
    from dolomite_engine_b200.hf_models import MoEDolomiteConfig

    shape = dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_head=8, n_inner=192, attention_head_type="mha",
                 add_bias=True, num_experts=E, num_experts_per_tok=2)
    drop = dict(resid_pdrop=0, embd_pdrop=0, attn_pdrop=0)
    drop.update({k: kw.pop(k) for k in list(kw) if k.endswith("pdrop")})
    cfg = MoEDolomiteConfig(position_embedding_type="rope", normalization_function="rmsnorm", activation_function=act,
                            eos_token_id=7, **drop, **shape, **kw)
    return cfg, O.OracleConfig(activation_function=act, **shape)


def _params(ocfg, seed=42):
    params = O.init_params(ocfg, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in params:
        if k.endswith(".bias"):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.25  # a zero bias would hide a missing one
    return params


def _model(cfg, params, padding_free=True, **kw):
    from dolomite_engine_b200.hf_models import MoEDolomiteForCausalLM

    m = MoEDolomiteForCausalLM(cfg, seed=None, use_padding_free_transformer=padding_free, **kw)
    m.load_state_dict(params)
    return m


def _grad_errors(model, ref):
    return [(n, round(rel_l2(u.gviews[n], ref[n]), 4)) for n, u, _ in model.engine.named_views() if rel_l2(u.gviews[n], ref[n]) > 3e-2]


@pytest.mark.parametrize("act", ["swiglu", "gelu_pytorch_tanh"])
@pytest.mark.parametrize("ragged", [False, True])
def test_biased_moe_model_packed_logits_loss_and_grads_match_oracle(act, ragged):
    """packed batches (documents split at eos when ragged): logits, loss and every gradient, the expert biases' included,
    against the oracle in bf16 with the GPU's expert choices pinned"""
    cfg, ocfg = _cfgs(act)
    params = _params(ocfg)
    model = _model(cfg, params)
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
    loss = model.forward_pretraining_loss(*args, torch.from_numpy(np.ascontiguousarray(labels).reshape(-1)).cuda())
    routing = {f"transformer.h.{i}.mlp.": layer[-1][0].sel_idx.long().cpu() for i, layer in enumerate(model.engine._saved["layers"])}
    loss.backward()
    logits = model(input_ids=args[0], position_ids=args[1], cu_seqlens=args[2], max_seqlen=args[3]).logits.float().cpu().detach()
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
    grads_ref = {k: v.grad for k, v in p_req.items()}
    assert not _grad_errors(model, grads_ref), _grad_errors(model, grads_ref)
    for i in range(cfg.n_layer):  # the expert bias gradients are real signals, not zeros that match zeros
        for n in ("c_fc.bias", "c_proj.bias"):
            assert grads_ref[f"transformer.h.{i}.mlp.{n}"].abs().max() > 0


def _padded_batch(padding="right", B=3, S=40, seed=5):
    rng = np.random.default_rng(seed)
    lens = [S, 23, 31]
    ids = np.zeros((B, S), dtype=np.int64)
    mask = np.zeros((B, S), dtype=np.int64)
    docs = []
    for r, n in enumerate(lens):
        d = rng.integers(8, 512, size=n)
        sl = slice(S - n, S) if padding == "left" else slice(0, n)
        ids[r, sl], mask[r, sl] = d, 1
        docs.append(d.tolist())
    return ids, mask, np.where(mask == 1, ids, -100), docs


def _run_padded(model, ids, mask, labels, flag=False, aux_weight=0.3):
    eng = model.engine
    eng.zero_grad()
    t = torch.from_numpy
    out = model(input_ids=t(ids), attention_mask=t(mask), labels=t(labels), output_router_logits=flag)
    routing = [layer[-1][0].sel_idx.long().cpu() for layer in eng._saved["layers"] if len(layer) > 1]
    (out.loss + aux_weight * out.aux_loss).backward() if flag else out.loss.backward()
    torch.cuda.synchronize()
    return out, routing, {n: u.gviews[n].clone() for n, u, _ in eng.named_views()}


def _oracle_padded(params, ocfg, docs, routing, coef=0.0, aux_weight=0.3, with_aux=False):
    from moe_aux_oracle import forward_logits_with_router, load_balancing_loss

    b = O.convert_padding_free_lists_to_tensors(docs, labels=docs)
    O.FORCED_ROUTING.clear()
    O.FORCED_ROUTING.update({f"transformer.h.{i}.mlp.": r for i, r in enumerate(routing)})
    try:
        p_req = {n: v.clone().requires_grad_(True) for n, v in params.items()}
        logits, router = forward_logits_with_router(p_req, ocfg, b["input_ids"], b["position_ids"], b["cu_seqlens"], bf16=True)
        shift = torch.as_tensor(O.finetune_shift_labels(b["labels"], b["cu_seqlens"]), dtype=torch.long)
        ce = torch.nn.functional.cross_entropy(logits[:-1].float(), shift, ignore_index=-100)
        aux = load_balancing_loss(router, ocfg.num_experts, ocfg.num_experts_per_tok, selected=routing) if with_aux else None
        loss = ce + coef * aux if with_aux else ce
        (loss + aux_weight * aux).backward() if with_aux else loss.backward()
    finally:
        O.FORCED_ROUTING.clear()
    return loss.detach(), (aux.detach() if with_aux else None), {n: v.grad for n, v in p_req.items()}


@pytest.mark.parametrize("padding", ["right", "left"])
def test_biased_moe_model_padded_loss_and_grads_match_oracle(padding):
    cfg, ocfg = _cfgs()
    params = _params(ocfg)
    model = _model(cfg, params, padding_free=False)
    ids, mask, labels, docs = _padded_batch(padding)
    out, routing, grads = _run_padded(model, ids, mask, labels)
    T_real = int(mask.sum())
    loss_ref, _, grads_ref = _oracle_padded(params, ocfg, docs, [r[:T_real] for r in routing])
    assert abs(out.loss.item() - loss_ref.item()) / loss_ref.item() < 1e-3
    bad = [(n, round(rel_l2(grads[n], grads_ref[n]), 4)) for n in grads if rel_l2(grads[n], grads_ref[n]) > 3e-2]
    assert not bad, bad


def test_biased_moe_load_balancing_loss_matches_oracle():
    cfg, ocfg = _cfgs(router_aux_loss_coef=1.0)
    params = _params(ocfg)
    model = _model(cfg, params, padding_free=False)
    ids, mask, labels, docs = _padded_batch("right")
    out, routing, grads = _run_padded(model, ids, mask, labels, flag=True)
    T_real = int(mask.sum())
    loss_ref, aux_ref, grads_ref = _oracle_padded(params, ocfg, docs, [r[:T_real] for r in routing], coef=1.0, with_aux=True)
    assert abs(out.loss.item() - loss_ref.item()) / loss_ref.item() < 1e-3
    assert abs(out.aux_loss.item() - aux_ref.item()) / aux_ref.item() < 1e-3
    bad = [(n, round(rel_l2(grads[n], grads_ref[n]), 4)) for n in grads if rel_l2(grads[n], grads_ref[n]) > 3e-2]
    assert not bad, bad


def _packed_step(model, seed=0, T=300):
    eng = model.engine
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, 512, (T + 1,), generator=g)
    cu = torch.tensor([0, 120, T], dtype=torch.int32).cuda()
    pos = torch.cat([torch.arange(120), torch.arange(T - 120)]).cuda()
    eng.zero_grad()
    _, loss = eng.forward(ids[:-1].cuda(), pos, cu, 180, ids[1:].cuda(), fuse_head_loss=True)
    eng.backward()
    torch.cuda.synchronize()
    return loss.clone(), {n: u.gviews[n].clone() for n, u, _ in eng.named_views()}


def test_biased_moe_steps_are_bit_identical_across_runs_and_checkpointing():
    cfg, ocfg = _cfgs()
    model = _model(cfg, _params(ocfg))
    la, ga = _packed_step(model)
    lb, gb = _packed_step(model)
    model.engine.checkpoint_every = 1
    lc, gc = _packed_step(model)
    model.engine.checkpoint_every = None
    for loss, g in ((lb, gb), (lc, gc)):
        assert torch.equal(loss, la)
        assert all(torch.equal(g[n], ga[n]) for n in ga), [n for n in ga if not torch.equal(g[n], ga[n])]
    assert all(ga[f"transformer.h.{i}.mlp.{n}"].abs().max() > 0 for i in range(2) for n in ("c_fc.bias", "c_proj.bias"))


def test_biased_moe_with_dropout_trains():
    cfg, ocfg = _cfgs(resid_pdrop=0.1, embd_pdrop=0.1, attn_pdrop=0.1)
    model = _model(cfg, _params(ocfg))
    assert model.engine.has_dropout
    model.engine.training = True
    loss, grads = _packed_step(model)
    assert torch.isfinite(loss).all()
    for n, v in grads.items():
        assert bool(torch.isfinite(v).all()), n
    assert grads["transformer.h.0.mlp.c_proj.bias"].abs().max() > 0


def test_biased_moe_fp8_mode_trains():
    """FP8 linears, the router included (E % 16 == 0); the experts and their biases stay bf16"""
    from dolomite_engine_b200.fp8 import fp8_autocast

    cfg, ocfg = _cfgs(E=16)
    model = _model(cfg, _params(ocfg))
    eng = model.engine
    eng.enable_fp8()
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 512, (257,), generator=g)
    cu = torch.tensor([0, 256], dtype=torch.int32).cuda()
    pos = torch.arange(256).cuda()
    losses = []
    for _ in range(8):
        eng.zero_grad()
        with fp8_autocast(eng):
            _, loss = eng.forward(ids[:-1].cuda(), pos, cu, 256, ids[1:].cuda(), fuse_head_loss=True)
        eng.backward()
        for u in eng.units:  # plain SGD on the fp32 masters
            u.master.data.add_(u.master.grad, alpha=-0.05)
        eng.refresh_compute_from_master()
        losses.append(loss.item())
    assert all(np.isfinite(losses)), losses
    assert losses[-1] < losses[0], losses


def test_biased_moe_greedy_decoding_equals_stepwise_argmax():
    cfg, ocfg = _cfgs()
    params = _params(ocfg)
    params["transformer.wte.weight"] = params["transformer.wte.weight"] * 20  # logits with clear argmaxes (tied head)
    model = _model(cfg, params, padding_free=False)
    rng = np.random.default_rng(9)
    ids = torch.from_numpy(rng.integers(8, 512, size=(3, 12)))
    mask = torch.ones_like(ids)
    mask[1, :4] = 0  # left padded prompts
    mask[2, :7] = 0
    ids = ids * mask
    out = model.generate(input_ids=ids, attention_mask=mask, max_new_tokens=6, eos_token_id=-1).cpu()
    assert out.shape == (3, 18) and torch.equal(out[:, :12], ids)
    checked = 0
    for r in range(3):
        n0 = int(mask[r].sum())
        row = out[r, 12 - n0 :]
        for t in range(6):
            prefix = row[: n0 + t][None]
            with torch.no_grad():
                logits = model(input_ids=prefix, attention_mask=torch.ones_like(prefix)).logits[0, -1].float()
            top2 = logits.topk(2).values
            if float(top2[0] - top2[1]) < 0.05:  # near tie: the batch composition may legitimately flip a bf16 argmax
                break
            assert int(logits.argmax()) == int(row[n0 + t]), (r, t)
            checked += 1
    assert checked >= 6
