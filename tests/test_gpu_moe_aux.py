"""GPU: the MoE load-balancing loss (output_router_logits=True on padded MoEDolomite batches).

Kernels: the statistics C_e (exact) and P_e (within the fp32 summation bound of an fp64 oracle), aux and its backward
coefficients, the router backward with the dense term (per element against fp64 autograd, within one bf16 ulp), and
byte-identical repeats.  Model: loss, aux_loss, router logits and every parameter gradient against the oracle's autograd
(tests/moe_aux_oracle.py) with left, right and no padding, block checkpointing, the FP8 router and repeated runs."""

import math

import numpy as np
import pytest
import torch

import oracle.dolomite_oracle as O
from moe_aux_oracle import forward_logits_with_router, load_balancing_loss

pytestmark = pytest.mark.gpu

U32 = 2.0**-24  # fp32 unit roundoff


def K():
    from dolomite_engine_b200 import kernels

    return kernels


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


# (T, T_real, E, k): every E the engine supports a shape of (8, 16, 64, 256) plus a width that is not a multiple of 8
KERNEL_CASES = [(16384, 16384, 8, 2), (16384, 16001, 64, 8), (8192, 8190, 256, 1), (4096, 4001, 256, 8),
                (1000, 997, 40, 1), (513, 500, 16, 2), (64, 1, 8, 1), (2048, 2048, 40, 8), (777, 700, 64, 1)]
LAYERS = 3


def _layers(T, E, k, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    logits = [(torch.randn(T, E, device="cuda", generator=g) * 2).to(torch.bfloat16) for _ in range(LAYERS)]
    return logits, [K().moe_route(lg, k) for lg in logits]


def _stats(logits, plans, T_real, coef, loss0):
    acc = K().moe_aux_acc(logits[0].shape[1], "cuda")
    for lg, plan in zip(logits, plans):
        K().moe_aux_stats(lg, plan, T_real, acc)
    loss = torch.tensor([loss0], dtype=torch.float32, device="cuda")
    aux, c = K().moe_aux_finalize(acc, LAYERS * T_real, coef, loss)
    return acc, aux, c, loss


@pytest.mark.parametrize("T,T_real,E,k", KERNEL_CASES)
def test_statistics_aux_and_coefficients_against_fp64(T, T_real, E, k):
    logits, plans = _layers(T, E, k, seed=T + E + k)
    acc, aux, c, loss = _stats(logits, plans, T_real, 0.37, 1.5)
    torch.cuda.synchronize()
    sel = torch.cat([p.sel_idx[:T_real].reshape(-1) for p in plans]).long().cpu()
    C = torch.bincount(sel, minlength=E).double()
    assert torch.equal(acc[1].double().cpu(), C)  # counts are exact
    P = sum(torch.softmax(lg[:T_real].double(), -1).sum(0) for lg in logits).cpu()
    # all terms are positive: the sequential depth of the fixed-order sums (8 tokens per lane, 8 warps, the CTA partials,
    # the layers) plus the softmax's own few roundings bound the relative error of each P_e
    depth = 8 + 8 + math.ceil(T_real / 64) + LAYERS + 8
    err = (acc[0].double().cpu() - P).abs()
    assert torch.all(err <= depth * U32 * P + 1e-30), (err / P).max().item()
    N = LAYERS * T_real
    aux_ref = E * float((C * P).sum()) / N**2
    assert abs(aux.item() - aux_ref) <= depth * U32 * aux_ref + 2 * U32 * aux_ref
    assert torch.allclose(c.double().cpu(), E * C / N**2, rtol=2 * U32, atol=0)
    assert abs(loss.item() - (1.5 + 0.37 * aux.item())) <= 4 * U32 * loss.item()
    # and again: byte-identical
    acc2, aux2, c2, loss2 = _stats(logits, plans, T_real, 0.37, 1.5)
    assert torch.equal(acc, acc2) and torch.equal(aux, aux2) and torch.equal(c, c2) and torch.equal(loss, loss2)


def _bf16_ulp(x):
    """spacing of bf16 numbers at |x| (that of the smallest normal for |x| below it)"""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0**-126)))
    return torch.pow(2.0, e - 7)


@pytest.mark.parametrize("T,T_real,E,k", KERNEL_CASES)
def test_router_backward_with_the_term_against_fp64_autograd(T, T_real, E, k):
    logits, plans = _layers(T, E, k, seed=7 * T + E + k)
    _, _, c, _ = _stats(logits, plans, T_real, 1.0, 0.0)
    lg, plan = logits[0], plans[0]
    g = torch.Generator(device="cuda").manual_seed(T + 1)
    dw = torch.randn(T, k, device="cuda", generator=g) * 1e-2
    s = torch.tensor([0.8], device="cuda")
    got = K().moe_router_bwd_aux(lg, plan, dw, c, s, T_real)
    again = K().moe_router_bwd_aux(lg, plan, dw, c, s, T_real)
    plain = K().moe_router_bwd(plan, dw)
    zero_s = K().moe_router_bwd_aux(lg, plan, dw, c, torch.zeros(1, device="cuda"), T_real)
    torch.cuda.synchronize()
    assert torch.equal(got, again)
    assert torch.equal(zero_s.float(), plain.float())  # s = 0: exactly moe_router_bwd (values; -0 == +0)
    assert torch.equal(got[T_real:].float(), plain[T_real:].float())  # alignment rows: top-k term only
    # fp64 autograd of  s * sum_e c_e P_e  (P over the real rows)  +  sum_j dw_j softmax(selected logits)_j
    x = lg.double().cpu().requires_grad_(True)
    sel = plan.sel_idx.long().cpu()
    p = torch.softmax(x, -1)
    term = 0.8 * (p[:T_real] * c.double().cpu()).sum()
    top = (torch.softmax(x.gather(1, sel), -1) * dw.double().cpu()).sum()
    (term + top).backward()
    ref = x.grad
    # one bf16 rounding of an fp32 value whose own error is a few fp32 roundings of the terms' magnitudes
    scale = 0.8 * p.detach().abs() * c.double().cpu().abs().max() + (dw.double().cpu().abs().sum(1, keepdim=True))
    bar = _bf16_ulp(ref) + 64 * U32 * scale
    err = (got.double().cpu() - ref).abs()
    assert torch.all(err <= bar), (err / bar).max().item()


# ---------------------------------------------------------------------------------------------------------------------
# model
# ---------------------------------------------------------------------------------------------------------------------
def _cfgs(E=8, k=2, coef=1.0):
    from dolomite_engine_b200.hf_models import MoEDolomiteConfig

    kw = dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_head=8, n_inner=192, attention_head_type="mha",
              add_bias=False, num_experts=E, num_experts_per_tok=k)
    cfg = MoEDolomiteConfig(position_embedding_type="rope", normalization_function="rmsnorm", activation_function="swiglu",
                            resid_pdrop=0, embd_pdrop=0, attn_pdrop=0, eos_token_id=7, router_aux_loss_coef=coef, **kw)
    return cfg, O.OracleConfig(**kw)


def _batch(padding: str, B=3, S=40, seed=5):
    rng = np.random.default_rng(seed)
    lens = [S, 23, 31] if padding != "none" else [S] * B
    ids = np.zeros((B, S), dtype=np.int64)
    mask = np.zeros((B, S), dtype=np.int64)
    docs = []
    for r, n in enumerate(lens):
        d = rng.integers(8, 512, size=n)
        sl = slice(S - n, S) if padding == "left" else slice(0, n)
        ids[r, sl], mask[r, sl] = d, 1
        docs.append(d.tolist())
    labels = np.where(mask == 1, ids, -100)
    return ids, mask, labels, docs


def _model(cfg, params):
    from dolomite_engine_b200.hf_models import MoEDolomiteForCausalLM

    m = MoEDolomiteForCausalLM(cfg, seed=None, use_padding_free_transformer=False)
    m.load_state_dict(params)
    return m


def _run(model, ids, mask, labels, aux_weight=0.3, flag=True):
    eng = model.engine
    eng.zero_grad()
    t = lambda a: torch.from_numpy(a)  # noqa: E731
    out = model(input_ids=t(ids), attention_mask=t(mask), labels=t(labels), output_router_logits=flag)
    routing = [layer[-1][0].sel_idx.long().cpu() for layer in eng._saved["layers"] if len(layer) > 1]
    (out.loss + aux_weight * out.aux_loss).backward() if flag else out.loss.backward()
    torch.cuda.synchronize()
    grads = {n: u.gviews[n].clone() for n, u, _ in eng.named_views()}
    return out, routing, grads


def _padded(routing, keep):
    """per-layer [T_real, k] expert ids -> [B*S, k] rows of the batch (padding rows: expert 0, masked out)"""
    out = []
    for r in routing:
        full = torch.zeros(keep.numel(), r.shape[1], dtype=torch.long, device=keep.device)
        full[keep] = r.to(keep.device)
        out.append(full)
    return out


def _oracle(params, ocfg, docs, routing, coef, aux_weight=0.3, with_term=True):
    b = O.convert_padding_free_lists_to_tensors(docs, labels=docs)
    O.FORCED_ROUTING.clear()
    O.FORCED_ROUTING.update({f"transformer.h.{i}.mlp.": r for i, r in enumerate(routing)})
    try:
        p_req = {n: v.clone().requires_grad_(True) for n, v in params.items()}
        logits, router = forward_logits_with_router(p_req, ocfg, b["input_ids"], b["position_ids"], b["cu_seqlens"], bf16=True)
        shift = torch.as_tensor(O.finetune_shift_labels(b["labels"], b["cu_seqlens"]), dtype=torch.long)
        ce = torch.nn.functional.cross_entropy(logits[:-1].float(), shift, ignore_index=-100)
        aux = load_balancing_loss(router, ocfg.num_experts, ocfg.num_experts_per_tok, selected=routing)
        loss = ce + coef * aux
        (loss + aux_weight * aux).backward() if with_term else ce.backward()
    finally:
        O.FORCED_ROUTING.clear()
    return loss.detach(), aux.detach(), [r.detach() for r in router], {n: v.grad for n, v in p_req.items()}


@pytest.mark.parametrize("padding", ["right", "left", "none"])
def test_padded_moe_loss_aux_router_logits_and_grads_match_oracle(padding):
    cfg, ocfg = _cfgs(coef=1.0)
    params = O.init_params(ocfg, seed=42)
    model = _model(cfg, params)
    ids, mask, labels, docs = _batch(padding)
    out, routing, grads = _run(model, ids, mask, labels)
    T_real = int(mask.sum())
    routing = [r[:T_real] for r in routing]
    loss_ref, aux_ref, router_ref, grads_ref = _oracle(params, ocfg, docs, routing, 1.0)
    assert abs(out.loss.item() - loss_ref.item()) / loss_ref.item() < 1e-3
    assert abs(out.aux_loss.item() - aux_ref.item()) / aux_ref.item() < 1e-3
    assert out.aux_loss.dim() == 0 and len(out.router_logits) == cfg.n_layer
    keep = torch.from_numpy(mask.reshape(-1)).bool().cuda()
    for lg, lr in zip(out.router_logits, router_ref):
        assert lg.shape == (ids.size, cfg.num_experts) and lg.dtype == torch.bfloat16
        assert torch.all(lg[~keep] == 0)  # padding rows are zeros
        assert rel_l2(lg[keep], lr) < 1e-2
    # the masked form on the returned (padded) router logits gives the same value (experts of the routing plan: bf16
    # logits can tie, and a top-k of the probabilities may then pick another of the tied experts)
    masked = load_balancing_loss(out.router_logits, cfg.num_experts, cfg.num_experts_per_tok,
                                 attention_mask=torch.from_numpy(mask).cuda(), selected=_padded(routing, keep))
    assert abs(masked.item() - out.aux_loss.item()) <= 1e-5 * out.aux_loss.item()
    bad = [(n, round(rel_l2(grads[n], grads_ref[n]), 4)) for n in grads if rel_l2(grads[n], grads_ref[n]) > 3e-2]
    assert not bad, bad
    # coef = 1: the router's gradient visibly depends on the term (the bar above would catch a missing term)
    _, _, _, grads_ce = _oracle(params, ocfg, docs, routing, 1.0, with_term=False)
    for i in range(cfg.n_layer):
        n = f"transformer.h.{i}.mlp.gate.weight"
        assert rel_l2(grads_ref[n], grads_ce[n]) > 0.06, n
    # return_dict=False keeps the reference's order
    tup = model(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), labels=torch.from_numpy(labels),
                output_router_logits=True, return_dict=False)
    assert len(tup) == 3 and torch.equal(tup[0], out.loss) and torch.equal(tup[1], out.aux_loss)
    assert all(torch.equal(a, b) for a, b in zip(tup[2], out.router_logits))


def test_repeat_and_block_checkpointing_are_bit_identical():
    cfg, ocfg = _cfgs(coef=1.0)
    params = O.init_params(ocfg, seed=42)
    model = _model(cfg, params)
    ids, mask, labels, _ = _batch("right")
    a, _, ga = _run(model, ids, mask, labels)
    b, _, gb = _run(model, ids, mask, labels)
    model.engine.checkpoint_every = 1
    c, _, gc = _run(model, ids, mask, labels)
    model.engine.checkpoint_every = None
    for o in (b, c):
        assert torch.equal(o.loss, a.loss) and torch.equal(o.aux_loss, a.aux_loss)
        assert all(torch.equal(x, y) for x, y in zip(o.router_logits, a.router_logits))
    for g in (gb, gc):
        assert all(torch.equal(g[n], ga[n]) for n in ga), [n for n in ga if not torch.equal(g[n], ga[n])]


def test_without_labels_aux_is_returned_and_differentiable():
    cfg, ocfg = _cfgs(coef=1.0)
    model = _model(cfg, O.init_params(ocfg, seed=42))
    ids, mask, _, _ = _batch("left")
    model.engine.zero_grad()
    out = model(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask), output_router_logits=True)
    assert out.loss is None and out.logits.shape == (*ids.shape, 512) and out.aux_loss.dim() == 0
    out.aux_loss.backward()  # only the load-balancing term
    torch.cuda.synchronize()
    grads = {n: u.gviews[n].clone() for n, u, _ in model.engine.named_views()}
    assert float(grads["transformer.h.1.mlp.gate.weight"].abs().max()) > 0
    assert float(grads["transformer.h.0.attn.c_attn.weight"].abs().max()) > 0  # through the routers' inputs
    assert float(grads["transformer.h.1.mlp.c_fc.weight"].abs().max()) == 0.0  # the experts get nothing


def test_flag_off_and_config_flag_alone_are_unchanged():
    """output_router_logits not passed (the config's True is not read, as in the reference's main.py): the outputs and
    gradients are byte-identical to a run without the flag anywhere"""
    cfg, ocfg = _cfgs(coef=1.0)
    params = O.init_params(ocfg, seed=42)
    ids, mask, labels, _ = _batch("right")
    plain, _, g_plain = _run(_model(cfg, params), ids, mask, labels, flag=False)
    cfg_on, _ = _cfgs(coef=1.0)
    cfg_on.output_router_logits = True
    on, _, g_on = _run(_model(cfg_on, params), ids, mask, labels, flag=None)
    assert type(on).__name__ == type(plain).__name__ == "CausalLMOutputWithPast"
    assert torch.equal(on.loss, plain.loss)
    assert all(torch.equal(g_on[n], g_plain[n]) for n in g_plain)


def test_fp8_router_carries_the_term_into_its_cast():
    """num_experts % 16 == 0: the router is an FP8 linear; its output gradient -- what is cast to e5m2 and enters the
    amax history -- holds the load-balancing term"""
    from dolomite_engine_b200.fp8 import fp8_autocast

    cfg, ocfg = _cfgs(E=16, k=2, coef=1.0)
    params = O.init_params(ocfg, seed=42)
    ids, mask, labels, _ = _batch("right")

    def run(aux_weight, coef):
        model = _model(_cfgs(E=16, k=2, coef=coef)[0], params)
        eng = model.engine
        eng.enable_fp8()
        assert any(n.endswith("mlp.gate.weight") for n in eng.fp8.names)
        seen = {}
        orig = eng._linear_bwd_fp8

        def spy(unit, wname, bname, x, dy, *a, **kw):
            if wname.endswith("mlp.gate.weight"):
                seen[wname] = dy.clone()
            return orig(unit, wname, bname, x, dy, *a, **kw)

        eng._linear_bwd_fp8 = spy
        eng.zero_grad()
        with fp8_autocast(eng):
            out = model(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask),
                        labels=torch.from_numpy(labels), output_router_logits=True)
        routing = [layer[-1][0].sel_idx.long() for layer in eng._saved["layers"]]
        (out.loss + aux_weight * out.aux_loss).backward()
        torch.cuda.synchronize()
        return out, seen, routing

    a, da, routing = run(0.3, 1.0)
    b, db, _ = run(0.3, 1.0)
    z, dz, _ = run(0.0, 0.0)  # s = 0: the plain top-k router gradient
    assert len(da) == cfg.n_layer and torch.isfinite(a.loss)
    assert torch.equal(a.loss, b.loss) and torch.equal(a.aux_loss, b.aux_loss)
    assert all(torch.equal(da[n], db[n]) for n in da)
    keep = torch.from_numpy(mask.reshape(-1)).bool().cuda()
    T_real = int(mask.sum())
    masked = load_balancing_loss(a.router_logits, 16, 2, attention_mask=torch.from_numpy(mask).cuda(),
                                 selected=_padded([r[:T_real] for r in routing], keep))
    assert abs(masked.item() - a.aux_loss.item()) <= 1e-5 * a.aux_loss.item()
    assert all(rel_l2(da[n], dz[n]) > 1e-2 for n in da)
