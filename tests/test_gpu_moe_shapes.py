"""GPU: MoE blocks of any expert count and width.

Kernels, per element against fp64 with the bars of test_gpu_moe_bias.py: the M-grouped expert GEMM over K tails
(K = 8, 16, 56 mod 64) and N tails, K-major and MN-major B, plain / gather-on-load / bias, with experts without tokens;
an expert whose weights are all NaN next to one with tokens; the K-grouped weight gradient over M and N tails, overwrite
and accumulate, with canaries after the buffer and between the rows of the groups; the router kernels for E that are not
multiples of 8; bit-identical results against the dense GEMM per expert.  Layers and models: the reference-derived
fixtures of tools/pin_moe_shapes.py, the load-balancing loss and router logits, bit-identical repeats and checkpointing,
dropout, FP8 mode with a bf16 router, greedy KV-cache decoding."""

import os

import numpy as np
import pytest
import torch

import oracle.dolomite_oracle as O
from moe_shapes_inputs import subsample
from test_moe_shapes import MODELS, hf_config, layer_case, model_params

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


def _rows(plan):
    """real grouped rows, their tokens and experts"""
    rows = torch.nonzero(plan.slot_of_row >= 0).flatten()
    return rows, plan.token_of_row[rows].long(), plan.tile_group[rows // 128].long()


def _per_expert(a, grp, w, E, transpose):
    """fp64 (a[r] W[grp[r]]^T if transpose else a[r] W[grp[r]], and the same over absolute values), one expert at a time"""
    ex = torch.zeros(a.shape[0], w.shape[1] if transpose else w.shape[2], dtype=torch.float64, device=a.device)
    mg = torch.zeros_like(ex)
    for e in range(E):
        sel = grp == e
        if bool(sel.any()):
            we = w[e].double().t() if transpose else w[e].double()
            ex[sel] = a[sel].double() @ we
            mg[sel] = a[sel].double().abs() @ we.abs()
    return ex, mg


def _check(got, exact, mag, K_):
    bar = BF16_EPS * exact.abs() + (K_ + 2) * F32_EPS * mag + 1e-30
    err = (got.double() - exact).abs()
    assert bool(torch.isfinite(got).all())
    assert bool((err <= bar).all()), (err / bar).max().item()


# ---------------------------------------------------------------------------------------------------------------------
# M-grouped expert GEMM
# ---------------------------------------------------------------------------------------------------------------------
SWEEP = [  # (T, E, k, K, N): K = 8, 16, 56 (mod 64), N tails of the 128-wide tile
    (300, 3, 2, 72, 136), (1000, 6, 2, 144, 200), (777, 20, 4, 120, 80), (64, 1, 1, 200, 424),
    (2048, 12, 8, 1352, 96), (5, 60, 1, 88, 48), (4096, 6, 2, 1376, 160),
]


@pytest.mark.parametrize("T,E,k,Kd,N", SWEEP)
@pytest.mark.parametrize("bias", [False, True])
def test_grouped_m_k_major_b_vs_fp64(T, E, k, Kd, N, bias):
    """forward of the expert linears, w3 [E, N, K]: plain and gather-on-load give the same bits and are within the bar;
    experts without tokens (the last two when k < E - 2) are skipped"""
    g = torch.Generator(device="cuda").manual_seed(T + E + Kd + N)
    empty = (E - 2, E - 1) if k < E - 2 else ()
    plan = _plan(T, E, k, g, empty)
    assert all(int(plan.counts[e]) == 0 for e in empty)
    x = bf(torch.randn(T, Kd, device="cuda", generator=g))
    w = bf(torch.randn(E, N, Kd, device="cuda", generator=g) * 0.05)
    b = bf(torch.randn(E, N, device="cuda", generator=g) * 0.3) if bias else None
    rows, tok, grp = _rows(plan)
    exact, mag = _per_expert(x[tok], grp, w, E, transpose=True)
    if bias:
        exact, mag = exact + b[grp].double(), mag + b[grp].double().abs()
    plain = K().gemm_grouped_m(K().moe_gather(x, plan), w, plan, b_mn=False, bias=b)
    gather = K().gemm_grouped_m_gather(x, w, plan, bias=b)
    _check(plain[rows], exact, mag, Kd)
    assert torch.equal(plain[rows], gather[rows])


@pytest.mark.parametrize("T,E,k,Kd,N", SWEEP)
@pytest.mark.parametrize("bias", [False, True])
def test_grouped_m_mn_major_b_vs_fp64(T, E, k, Kd, N, bias):
    """dgrad of the expert linears, w3 [E, K, N] (D = A W[e]): the K tail of each expert is its own, zero-filled"""
    g = torch.Generator(device="cuda").manual_seed(3 * T + E + Kd + N)
    empty = (0, E - 1) if k < E - 2 else ()
    plan = _plan(T, E, k, g, empty)
    a = bf(torch.randn(plan.max_rows, Kd, device="cuda", generator=g))
    w = bf(torch.randn(E, Kd, N, device="cuda", generator=g) * 0.05)
    b = bf(torch.randn(E, N, device="cuda", generator=g) * 0.3) if bias else None
    rows, _, grp = _rows(plan)
    exact, mag = _per_expert(a[rows], grp, w, E, transpose=False)
    if bias:
        exact, mag = exact + b[grp].double(), mag + b[grp].double().abs()
    _check(K().gemm_grouped_m(a, w, plan, b_mn=True, bias=b)[rows], exact, mag, Kd)


@pytest.mark.parametrize("Kd,N", [(64, 128), (128, 192), (72, 136), (1376, 160), (120, 80)])
def test_grouped_m_equals_the_dense_gemm_per_expert(Kd, N):
    """every expert's rows equal a dense GEMM of those rows bit for bit (same 128-wide kernel, same k-blocks): K-major and
    MN-major B, on and off multiples of 64.  Grouped launches always run 128-wide tiles, whatever gemm_tile_n forces."""
    g = torch.Generator(device="cuda").manual_seed(Kd + N)
    E, T = 6, 1500
    plan = _plan(T, E, 2, g)
    a = bf(torch.randn(plan.max_rows, Kd, device="cuda", generator=g))
    w_k = bf(torch.randn(E, N, Kd, device="cuda", generator=g) * 0.05)
    w_mn = bf(torch.randn(E, Kd, N, device="cuda", generator=g) * 0.05)
    off = plan.offsets.cpu().tolist()
    old = K().get_option("gemm_tile_n")
    try:
        outs = []
        for tile in (128, 256):
            K().set_option("gemm_tile_n", tile)
            outs.append((K().gemm_grouped_m(a, w_k, plan, b_mn=False), K().gemm_grouped_m(a, w_mn, plan, b_mn=True)))
        K().set_option("gemm_tile_n", 128)
        for e in range(E):
            n = int(plan.counts[e])
            if n == 0:
                continue
            seg = a[off[e] : off[e] + n]
            dense_k = K().gemm(seg, w_k[e])
            dense_mn = K().gemm(seg, w_mn[e], b_mn=True)
            for fwd, dgrad in outs:
                assert torch.equal(fwd[off[e] : off[e] + n], dense_k), e
                assert torch.equal(dgrad[off[e] : off[e] + n], dense_mn), e
    finally:
        K().set_option("gemm_tile_n", old)


@pytest.mark.parametrize("H,F", [(80, 40), (144, 200), (160, 424), (96, 1376)])
def test_nan_weights_of_an_expert_without_tokens_do_not_reach_its_neighbour(H, F):
    """experts 1 and 3 get no tokens and hold NaN weights and biases; experts 0 and 2 (directly before them) must stay
    finite and correct in the forward GEMM and in both dgrads (d_act = dy W_proj[e], dxg = d_fc W_fc[e]), whose K tails
    end inside their own expert"""
    g = torch.Generator(device="cuda").manual_seed(H + F)
    E, T = 4, 700
    plan = _plan(T, E, 1, g, empty=(1, 3))
    assert int(plan.counts[1]) == 0 and int(plan.counts[3]) == 0
    rows, tok, grp = _rows(plan)
    assert set(grp.unique().tolist()) == {0, 2}
    x = bf(torch.randn(T, H, device="cuda", generator=g))
    w_fc = bf(torch.randn(E, F, H, device="cuda", generator=g) * 0.05)     # [E, fc_out, H]
    w_proj = bf(torch.randn(E, H, F, device="cuda", generator=g) * 0.05)   # [E, H, F]
    b_fc = bf(torch.randn(E, F, device="cuda", generator=g) * 0.3)
    for t in (w_fc, w_proj, b_fc):
        t[1] = float("nan")
        t[3] = float("nan")
    # forward, K = H: fc = x W_fc[e]^T + b
    exact, mag = _per_expert(x[tok], grp, w_fc, E, transpose=True)
    exact, mag = exact + b_fc[grp].double(), mag + b_fc[grp].double().abs()
    for fc in (K().gemm_grouped_m(K().moe_gather(x, plan), w_fc, plan, b_mn=False, bias=b_fc),
               K().gemm_grouped_m_gather(x, w_fc, plan, bias=b_fc)):
        _check(fc[rows], exact, mag, H)
    # dgrad of c_proj, K = H: d_act = dyg W_proj[e]
    dyg = bf(torch.randn(plan.max_rows, H, device="cuda", generator=g))
    exact, mag = _per_expert(dyg[rows], grp, w_proj, E, transpose=False)
    _check(K().gemm_grouped_m(dyg, w_proj, plan, b_mn=True)[rows], exact, mag, H)
    # dgrad of c_fc, K = fc_out: dxg = d_fc W_fc[e]
    d_fc = bf(torch.randn(plan.max_rows, F, device="cuda", generator=g))
    exact, mag = _per_expert(d_fc[rows], grp, w_fc, E, transpose=False)
    _check(K().gemm_grouped_m(d_fc, w_fc, plan, b_mn=True)[rows], exact, mag, F)


# ---------------------------------------------------------------------------------------------------------------------
# K-grouped weight gradient
# ---------------------------------------------------------------------------------------------------------------------
CANARY = 12345.5


def _wgrad_ref(a, b, plan, M, N):
    off = plan.offsets.cpu().tolist()
    ex, mg = [], []
    for e in range(plan.E):
        s0, s1 = off[e], off[e + 1]
        ex.append(a[s0:s1].double().t() @ b[s0:s1].double())
        mg.append(a[s0:s1].double().abs().t() @ b[s0:s1].double().abs())
    return torch.stack(ex), torch.stack(mg), [off[e + 1] - off[e] for e in range(plan.E)]


@pytest.mark.parametrize("T,E,k,M,N", [(300, 3, 2, 72, 80), (1000, 6, 2, 200, 144), (777, 20, 4, 136, 200),
                                       (64, 1, 1, 48, 24), (4096, 12, 8, 848, 160)])
def test_grouped_k_wgrad_over_m_and_n_tails(T, E, k, M, N):
    """out3[e] (+)= a_e^T b_e in fp32: overwrite (beta 0: an expert without rows is written as zeros over its own [M, N])
    and accumulate (beta 1: it keeps its values); the canary after the buffer stays"""
    g = torch.Generator(device="cuda").manual_seed(T + M + N)
    empty = (1,) if k < E - 2 else ()
    plan = _plan(T, E, k, g, empty)
    a = bf(torch.randn(plan.max_rows, M, device="cuda", generator=g))
    b = bf(torch.randn(plan.max_rows, N, device="cuda", generator=g))
    a[plan.slot_of_row < 0] = 0  # padding rows are zero (combine_bwd / gather write zeros there)
    b[plan.slot_of_row < 0] = 0
    exact, mag, rows = _wgrad_ref(a, b, plan, M, N)
    n = E * M * N
    for beta in (0.0, 1.0):
        buf = torch.full((n + 64,), CANARY, device="cuda")
        out3 = buf[:n].view(E, M, N)
        init = torch.randn(E, M, N, device="cuda", generator=g)
        out3.copy_(init)
        K().gemm_grouped_k(a, b, plan, out3, beta=beta)
        torch.cuda.synchronize()
        assert bool((buf[n:] == CANARY).all())
        want = exact + (init.double() if beta else 0)
        bar = (max(rows) + 2) * F32_EPS * (mag + (init.double().abs() if beta else 0)) + 1e-30
        for e in range(E):
            if rows[e] == 0:
                assert torch.equal(out3[e], init[e] if beta else torch.zeros_like(init[e])), (beta, e)
                continue
            assert bool(((out3[e].double() - want[e]).abs() <= bar[e]).all()), (beta, e)


@pytest.mark.parametrize("M,N", [(72, 80), (136, 200), (200, 24)])
def test_grouped_k_wgrad_writes_nothing_between_rows_and_groups(M, N):
    """a row stride of N + 8 leaves eight canary columns after every row of every group, and canary rows after the last
    group: a tile that ran past row M or column N of its own group would overwrite one of them"""
    from dolomite_engine_b200 import _lib

    g = torch.Generator(device="cuda").manual_seed(M * N)
    E = 5
    plan = _plan(900, E, 2, g, empty=(2,))
    a = bf(torch.randn(plan.max_rows, M, device="cuda", generator=g))
    b = bf(torch.randn(plan.max_rows, N, device="cuda", generator=g))
    a[plan.slot_of_row < 0] = 0
    b[plan.slot_of_row < 0] = 0
    exact, mag, rows = _wgrad_ref(a, b, plan, M, N)
    ld = N + 8
    for beta in (0.0, 1.0):
        buf = torch.full((E * M + 3, ld), CANARY, device="cuda")
        view = buf[: E * M].view(E, M, ld)
        if beta:
            view[:, :, :N] = 0.5
        _lib.call("dolomite_b200_gemm_bf16_grouped_k", a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0),
                  buf.data_ptr(), ld, 1.0, beta, M, N, plan.max_rows, plan.offsets.data_ptr(), E, K()._stream())
        torch.cuda.synchronize()
        assert bool((view[:, :, N:] == CANARY).all()) and bool((buf[E * M :] == CANARY).all()), beta
        got = view[:, :, :N].double()
        want = exact + (0.5 if beta else 0.0)
        bar = (max(rows) + 2) * F32_EPS * (mag + (0.5 if beta else 0.0)) + 1e-30
        assert bool(((got - want).abs() <= bar).all()), beta
        assert bool((view[2, :, :N] == (0.5 if beta else 0.0)).all())  # the expert without rows


# ---------------------------------------------------------------------------------------------------------------------
# router kernels
# ---------------------------------------------------------------------------------------------------------------------
def _grid_logits(T, E, seed):
    """rows of distinct logits 0.25 apart (exact in bf16): no top-k ties"""
    g = np.random.default_rng(seed)
    grid = (np.arange(E) - E // 2) * 0.25
    return torch.from_numpy(np.stack([g.permutation(grid) for _ in range(T)]).astype(np.float32))


@pytest.mark.parametrize("E,k", [(1, 1), (3, 2), (6, 2), (12, 8), (20, 4), (60, 8)])
def test_router_kernels_for_any_expert_count(E, k):
    """route (top-k, weights, counts), load-balancing statistics and both router backwards against fp64, from the gate
    GEMM's output as moe.forward passes it (16-byte rows -> kernels.router_logits)"""
    T, T_real = 1000, 900
    lg = _grid_logits(T, E, E)
    gate_out = K().rows_empty(T, E, device="cuda")
    gate_out.copy_(lg)
    logits = K().router_logits(gate_out)
    plan = K().moe_route(logits, k)
    ref_idx = lg.topk(k, dim=-1).indices
    assert torch.equal(plan.sel_idx.long().cpu(), ref_idx)
    top = lg.double().gather(1, ref_idx)
    w_ref = torch.softmax(top, -1)
    assert bool(((plan.sel_w.double().cpu() - w_ref).abs() <= 8 * F32_EPS).all())
    assert torch.equal(plan.counts.cpu().long(), torch.bincount(ref_idx.flatten(), minlength=E))
    # statistics over the first T_real tokens
    acc = K().moe_aux_acc(E, "cuda")
    K().moe_aux_stats(logits, plan, T_real, acc)
    p = torch.softmax(lg[:T_real].double(), -1)
    assert torch.equal(acc[1].cpu().double(), torch.bincount(ref_idx[:T_real].flatten(), minlength=E).double())
    assert bool(((acc[0].cpu().double() - p.sum(0)).abs() <= (T_real + 8) * F32_EPS * p.sum(0) + 1e-30).all())
    # router backward: d logits of the top-k softmax, and with the load-balancing term
    dw = torch.randn(T, k, device="cuda")
    dl = K().router_grad(K().moe_router_bwd(plan, dw))
    w = plan.sel_w.double().cpu()
    d = dw.double().cpu()
    ref = torch.zeros(T, E, dtype=torch.float64).scatter(1, ref_idx, w * (d - (w * d).sum(-1, keepdim=True)))
    mag = torch.zeros(T, E, dtype=torch.float64).scatter(1, ref_idx, w * (d.abs() + (w * d).abs().sum(-1, keepdim=True)))
    bar = BF16_EPS * ref.abs() + 16 * F32_EPS * mag + 1e-30
    assert bool(((dl.double().cpu() - ref).abs() <= bar).all())
    assert dl.stride(0) % 8 == 0  # 16-byte rows for the gate GEMMs
    c = torch.rand(E, device="cuda")
    s = torch.tensor([0.7], device="cuda")
    dla = K().router_grad(K().moe_router_bwd_aux(logits, plan, dw, c, s, T_real))
    pa = torch.softmax(lg.double(), -1)
    cd = c.double().cpu()
    term = 0.7 * pa * (cd - (pa * cd).sum(-1, keepdim=True))
    term[T_real:] = 0
    term_mag = 0.7 * pa * (cd.abs() + (pa * cd.abs()).sum(-1, keepdim=True))
    term_mag[T_real:] = 0
    ref_a = ref + term
    bar = BF16_EPS * ref_a.abs() + 16 * F32_EPS * mag + 64 * F32_EPS * term_mag + 1e-30
    assert bool(((dla.double().cpu() - ref_a).abs() <= bar).all())


# ---------------------------------------------------------------------------------------------------------------------
# layers
# ---------------------------------------------------------------------------------------------------------------------
def _layer_model(cfg):
    from dolomite_engine_b200.hf_models import MoEDolomiteConfig, MoEDolomiteForCausalLM

    hf = MoEDolomiteConfig(vocab_size=256, n_embd=cfg.n_embd, n_layer=1, n_head=cfg.n_embd // 16, n_inner=cfg.n_inner,
                           num_experts=cfg.num_experts, num_experts_per_tok=cfg.num_experts_per_tok, attention_head_type="mha",
                           add_bias=cfg.add_bias, position_embedding_type="rope", normalization_function="rmsnorm",
                           activation_function=cfg.activation_function, resid_pdrop=0, embd_pdrop=0, attn_pdrop=0)
    return MoEDolomiteForCausalLM(hf, seed=0)


@pytest.mark.parametrize("name", ["e3_k2", "e20_k4", "e1_k1"])
def test_moe_shapes_layer_matches_golden(golden_dir, name):
    """the reference's eager SparseMoE with E 3 / 20 / 1 and widths off multiples of 64: output, dx and every parameter
    gradient within rel-L2 2e-2, with the reference's routing (no near-ties at bf16 resolution)"""
    from dolomite_engine_b200 import moe

    fx = np.load(os.path.join(golden_dir, "moe_shapes_layer.npz"))
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
    assert rel_l2(saved[1], torch.from_numpy(fx[f"{name}/router_logits"])) < 1e-2
    assert rel_l2(y, torch.from_numpy(fx[f"{name}/y"])) < 2e-2
    dx = moe.backward(eng, eng.units[1], p, xc, bf(dy).cuda(), 1.0, saved)
    torch.cuda.synchronize()
    assert rel_l2(dx, torch.from_numpy(fx[f"{name}/grad:x"])) < 2e-2
    for n in params:
        got = eng.units[1].gviews[p + "mlp." + n[2:]]
        got = subsample(got.cpu()) if got.dim() == 3 else got
        assert rel_l2(got, torch.from_numpy(fx[f"{name}/grad:{n[2:]}"])) < 2e-2, n


# ---------------------------------------------------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------------------------------------------------
def _model(name, params, padding_free=True, **kw):
    from dolomite_engine_b200.hf_models import MoEDolomiteForCausalLM

    m = MoEDolomiteForCausalLM(hf_config(name, **kw), seed=None, use_padding_free_transformer=padding_free)
    m.load_state_dict(params)
    return m


def _fixture(golden_dir, name):
    fx = np.load(os.path.join(golden_dir, f"moe_shapes_model_{name}.npz"))
    cfg, params = model_params(fx, name)
    return fx, cfg, params


def _grad_errors(grads, ref):
    return [(n, round(rel_l2(grads[n], ref[n]), 4)) for n in grads if rel_l2(grads[n], ref[n]) > 3e-2]


@pytest.mark.parametrize("name", list(MODELS))
def test_model_packed_logits_loss_and_grads_match_oracle(golden_dir, name):
    """the fixture's packed ragged batch: logits, loss and every gradient against the oracle in bf16 with the GPU's expert
    choices pinned; the loss also against the reference's fp32 value"""
    fx, ocfg, params = _fixture(golden_dir, name)
    model = _model(name, params)
    model.assume_unit_loss_grad = True
    tokens = fx["packed_tokens"]
    inp, labels = O.split_tokens(tokens)
    b = O.prepare_model_inputs(inp.copy(), 7, True, True)
    args = (torch.from_numpy(b["input_ids"]).cuda(), torch.from_numpy(b["position_ids"]).cuda(),
            torch.from_numpy(b["cu_seqlens"]).cuda(), b["max_seqlen"])
    model.engine.zero_grad()
    loss = model.forward_pretraining_loss(*args, torch.from_numpy(np.ascontiguousarray(labels).reshape(-1)).cuda())
    routing = {f"transformer.h.{i}.mlp.": layer[-1][0].sel_idx.long().cpu() for i, layer in enumerate(model.engine._saved["layers"])}
    loss.backward()
    torch.cuda.synchronize()
    grads = {n: u.gviews[n].clone() for n, u, _ in model.engine.named_views()}
    logits = model(input_ids=args[0], position_ids=args[1], cu_seqlens=args[2], max_seqlen=args[3]).logits.float().cpu().detach()
    O.FORCED_ROUTING.clear()
    O.FORCED_ROUTING.update(routing)
    try:
        p_req = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        loss_ref, logits_ref = O.pretraining_loss(p_req, ocfg, tokens, 7, True, True, bf16=True)
        loss_ref.backward()
    finally:
        O.FORCED_ROUTING.clear()
    assert rel_l2(logits, logits_ref.detach()) < 1e-2
    assert abs(loss.item() - loss_ref.item()) / loss_ref.item() < 1e-3
    assert abs(loss.item() - float(fx["packed_loss"])) / float(fx["packed_loss"]) < 1e-2
    bad = _grad_errors(grads, {k: v.grad for k, v in p_req.items()})
    assert not bad, bad


def _padded_docs(fx):
    ids, mask = fx["padded_tokens"], fx["padded_mask"]
    docs = [ids[r][mask[r].astype(bool)].tolist() for r in range(ids.shape[0])]
    return ids * mask, mask, np.where(mask == 1, ids, -100), docs


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


@pytest.mark.parametrize("name", list(MODELS))
def test_model_padded_loss_and_grads_match_oracle(golden_dir, name):
    fx, ocfg, params = _fixture(golden_dir, name)
    model = _model(name, params, padding_free=False)
    ids, mask, labels, docs = _padded_docs(fx)
    out, routing, grads = _run_padded(model, ids, mask, labels)
    T_real = int(mask.sum())
    loss_ref, _, grads_ref = _oracle_padded(params, ocfg, docs, [r[:T_real] for r in routing])
    assert abs(out.loss.item() - loss_ref.item()) / loss_ref.item() < 1e-3
    assert abs(out.loss.item() - float(fx["padded_loss"])) / float(fx["padded_loss"]) < 1e-2
    bad = _grad_errors(grads, grads_ref)
    assert not bad, bad


@pytest.mark.parametrize("name", list(MODELS))
def test_model_load_balancing_loss_and_router_logits(golden_dir, name):
    """output_router_logits=True on the padded batch: each layer's router logits are a contiguous [B*S, E], zero at
    padding, the reference's values at real tokens; aux_loss against the reference's value and the oracle's; loss and
    every gradient with the term against the oracle"""
    fx, ocfg, params = _fixture(golden_dir, name)
    model = _model(name, params, padding_free=False, router_aux_loss_coef=1.0)
    ids, mask, labels, docs = _padded_docs(fx)
    out, routing, grads = _run_padded(model, ids, mask, labels, flag=True)
    keep = torch.from_numpy(mask.reshape(-1) == 1)
    E = ocfg.num_experts
    assert len(out.router_logits) == ocfg.n_layer
    for layer, r in enumerate(out.router_logits):
        assert tuple(r.shape) == (mask.size, E) and r.is_contiguous()
        r = r.float().cpu()
        assert bool((r[~keep] == 0).all())
        assert rel_l2(r[keep], torch.from_numpy(fx[f"padded_router_logits:{layer}"])) < 1e-2, layer
    assert abs(out.aux_loss.item() - float(fx["padded_aux"])) / float(fx["padded_aux"]) < 2e-2
    T_real = int(mask.sum())
    loss_ref, aux_ref, grads_ref = _oracle_padded(params, ocfg, docs, [r[:T_real] for r in routing], coef=1.0, with_aux=True)
    assert abs(out.aux_loss.item() - aux_ref.item()) / aux_ref.item() < 1e-3
    assert abs(out.loss.item() - loss_ref.item()) / loss_ref.item() < 1e-3
    bad = _grad_errors(grads, grads_ref)
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


@pytest.mark.parametrize("name", list(MODELS))
def test_model_steps_are_bit_identical_across_runs_and_checkpointing(golden_dir, name):
    _, _, params = _fixture(golden_dir, name)
    model = _model(name, params)
    la, ga = _packed_step(model)
    lb, gb = _packed_step(model)
    model.engine.checkpoint_every = 1
    lc, gc = _packed_step(model)
    model.engine.checkpoint_every = None
    for loss, g in ((lb, gb), (lc, gc)):
        assert torch.equal(loss, la)
        assert all(torch.equal(g[n], ga[n]) for n in ga), [n for n in ga if not torch.equal(g[n], ga[n])]
    assert all(bool(torch.isfinite(v).all()) for v in ga.values())


@pytest.mark.parametrize("name", list(MODELS))
def test_model_with_dropout_trains(golden_dir, name):
    _, _, params = _fixture(golden_dir, name)
    model = _model(name, params, resid_pdrop=0.1, embd_pdrop=0.1, attn_pdrop=0.1)
    assert model.engine.has_dropout
    model.engine.training = True
    loss, grads = _packed_step(model)
    assert torch.isfinite(loss).all()
    for n, v in grads.items():
        assert bool(torch.isfinite(v).all()), n
    assert grads["transformer.h.0.mlp.c_fc.weight"].abs().max() > 0


def test_fp8_mode_trains_with_a_bf16_router_for_six_experts(golden_dir):
    """E = 6: the attention linears run in FP8, the router (6 x 160) stays bf16, and the loss falls"""
    from dolomite_engine_b200.fp8 import fp8_autocast

    _, _, params = _fixture(golden_dir, "e6_swiglu")
    model = _model("e6_swiglu", params)
    eng = model.engine
    eng.enable_fp8()
    assert "transformer.h.0.attn.c_attn.weight" in eng.fp8.names
    assert not any(n.endswith("mlp.gate.weight") for n in eng.fp8.names)
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


@pytest.mark.parametrize("name", list(MODELS))
def test_greedy_decoding_equals_stepwise_argmax(golden_dir, name):
    _, _, params = _fixture(golden_dir, name)
    params = dict(params)
    params["transformer.wte.weight"] = params["transformer.wte.weight"] * 20  # logits with clear argmaxes (tied head)
    model = _model(name, params, padding_free=False)
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
