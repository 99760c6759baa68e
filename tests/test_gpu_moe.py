"""GPU parity of the MoE path (router, dispatch plan, grouped wgmma GEMMs, combine) against the oracle's eager
SparseMoE restatement and the reference-derived golden layer (tests/golden/moe_layer.npz).
Tolerances follow tests/hf_models/single_gpu/hf_models/scattermoe_test.py:38-48 (bf16: atol 2e-3 on logits)."""

import os

import numpy as np
import pytest
import torch

import oracle.dolomite_oracle as O

pytestmark = pytest.mark.gpu


def K():
    from dolomite_engine_b200 import kernels

    return kernels


def bf(x):
    return x.to(torch.bfloat16)


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


@pytest.mark.parametrize("T,E,k", [(96, 8, 2), (1000, 8, 2), (300, 16, 4), (5, 8, 1), (257, 64, 8)])
def test_route_and_plan_bookkeeping(T, E, k):
    g = torch.Generator().manual_seed(0)
    logits = bf(torch.randn(T, E, generator=g))
    plan = K().moe_route(logits.cuda(), k)
    torch.cuda.synchronize()
    w_ref, idx_ref, _ = O.moe_route(torch.zeros(T, 1), torch.zeros(E, 1), k) if False else (None, None, None)
    lf = logits.float()
    tv, ti = lf.topk(k, dim=-1)
    sel = plan.sel_idx.cpu().long()
    # selected experts: identical value multiset per token (ties may pick a different but equal-valued expert)
    assert torch.equal(torch.gather(lf, 1, sel).sort(-1).values, tv.sort(-1).values)
    w_ref = torch.softmax(torch.gather(lf, 1, sel), dim=-1)
    assert torch.allclose(plan.sel_w.cpu(), w_ref, atol=1e-6)
    counts = plan.counts.cpu().numpy()
    assert np.array_equal(counts, np.bincount(sel.reshape(-1).numpy(), minlength=E))  # bit exact (moe/base.py:158-164)
    off = plan.offsets.cpu().numpy()
    assert off[0] == 0 and np.all(off % 256 == 0)  # segments padded to CTA-pair super tiles
    assert np.array_equal(np.diff(off), (counts + 255) // 256 * 256)
    ros, sor = plan.row_of_slot.cpu().numpy(), plan.slot_of_row.cpu().numpy()
    assert len(set(ros.tolist())) == T * k  # every slot has its own row
    assert np.array_equal(sor[ros], np.arange(T * k))  # inverse maps
    flat = sel.reshape(-1).numpy()
    assert np.all(ros >= off[flat]) and np.all(ros < off[flat] + counts[flat])  # row inside its expert segment
    assert (sor >= 0).sum() == T * k
    tor = plan.token_of_row.cpu().numpy()
    assert np.array_equal(tor[ros], np.arange(T * k) // k) and np.all(tor[sor < 0] == 0)  # gather index of the fused load
    tg = plan.tile_group.cpu().numpy()
    for i, gidx in enumerate(tg):
        row = i * 128
        assert gidx == (-1 if row >= off[-1] else np.searchsorted(off, row, side="right") - 1)


def test_grouped_gemms_vs_per_expert_matmul():
    g = torch.Generator().manual_seed(1)
    T, E, k, H, F = 700, 8, 2, 128, 256
    x = bf(torch.randn(T, H, generator=g))
    logits = bf(torch.randn(T, E, generator=g))
    w = bf(torch.randn(E, F, H, generator=g) * 0.1)
    plan = K().moe_route(logits.cuda(), k)
    xg = K().moe_gather(x.cuda(), plan)
    y = K().gemm_grouped_m(xg, w.cuda(), plan, b_mn=False)
    torch.cuda.synchronize()
    off = plan.offsets.cpu().numpy()
    cnt = plan.counts.cpu().numpy()
    sor = plan.slot_of_row.cpu().numpy()
    xg_c, y_c = xg.float().cpu(), y.float().cpu()
    for e in range(E):
        rows = slice(off[e], off[e] + cnt[e])
        assert torch.equal(xg_c[rows], x.float()[sor[rows] // k])  # gather is exact
        assert torch.all(xg_c[off[e] + cnt[e] : off[e + 1]] == 0)  # padding rows are zero
        ref = xg_c[rows] @ w[e].float().t()
        assert rel_l2(y_c[rows], ref) < 5e-3
    # dgrad form: D = dY W[e]   (W stored [E, F, H] read MN-major)
    dy = K().gemm_grouped_m(y, w.cuda(), plan, b_mn=True)
    for e in range(E):
        rows = slice(off[e], off[e] + cnt[e])
        assert rel_l2(dy.float().cpu()[rows], y_c[rows] @ w[e].float()) < 5e-3
    # wgrad form: dW[e] += dY_e^T X_e, accumulated twice == 2x
    dw = torch.zeros(E, F, H, device="cuda")
    K().gemm_grouped_k(y, xg, plan, dw)
    once = dw.clone()
    K().gemm_grouped_k(y, xg, plan, dw)
    assert torch.allclose(dw, 2 * once, rtol=1e-5, atol=1e-4)
    for e in range(E):
        rows = slice(off[e], off[e] + cnt[e])
        assert rel_l2(once[e], y_c[rows].t() @ xg_c[rows]) < 1e-4


@pytest.mark.parametrize("F,H", [(256, 128), (512, 384)])  # one CTA-pair super tile / several tiles with a ragged last column block
def test_expert_wgrad_overwrite_writes_zeros_for_experts_without_tokens(F, H):
    """engine.zero_grad() does not clear the expert weight gradients: the first K-grouped GEMM of a window runs with beta = 0
    and must define EVERY expert's slice -- also of experts that received no token (empty contraction range)"""
    g = torch.Generator().manual_seed(3)
    T, E, k = 600, 8, 2
    logits = torch.randn(T, E, generator=g)
    logits[:, 3] = -1e4  # never among the top-2
    logits[:, 6] = -2e4
    plan = K().moe_route(bf(logits).cuda(), k)
    cnt = plan.counts.cpu().numpy()
    assert cnt[3] == 0 and cnt[6] == 0 and cnt.sum() == T * k
    x = bf(torch.randn(T, H, generator=g))
    xg = K().moe_gather(x.cuda(), plan)
    y = bf(torch.randn(plan.max_rows, F, generator=g)).cuda()
    acc = torch.zeros(E, F, H, device="cuda")
    K().gemm_grouped_k(y, xg, plan, acc)  # accumulate form into a cleared buffer = the reference result
    dw = torch.full((E, F, H), float("nan"), device="cuda")
    K().gemm_grouped_k(y, xg, plan, dw, beta=0.0)
    torch.cuda.synchronize()
    assert torch.equal(dw, acc)  # same tiles, same arithmetic; no stale value (NaN) survives
    assert torch.all(dw[3] == 0) and torch.all(dw[6] == 0)
    # accumulate form leaves the slices of the empty experts alone
    K().gemm_grouped_k(y, xg, plan, dw)
    assert torch.all(dw[3] == 0) and torch.allclose(dw, 2 * acc, rtol=1e-5, atol=1e-4)


def _moe_cfgs():
    from dolomite_engine_b200.hf_models import MoEDolomiteConfig

    kw = dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_head=8, n_inner=192, attention_head_type="mha",
              add_bias=False, num_experts=8, num_experts_per_tok=2)
    ocfg = O.OracleConfig(**kw)
    cfg = MoEDolomiteConfig(position_embedding_type="rope", normalization_function="rmsnorm", activation_function="swiglu",
                            resid_pdrop=0, embd_pdrop=0, attn_pdrop=0, eos_token_id=7, **kw)
    return cfg, ocfg


@pytest.mark.parametrize("T,H,N,E,k", [(1000, 256, 512, 8, 2), (4096, 2048, 1024, 8, 2), (37, 64, 264, 16, 4)])
def test_gather_on_load_equals_gather_then_gemm(T, H, N, E, k):
    """grouped expert GEMM with the token gather fused into its operand load (rows copied by the producer warp) == gather kernel + grouped GEMM,
    bit for bit on every real row; CTA-pair and single-CTA grids (the reference: scattermoe parallel_linear, moe/scatter.py:38-49)"""
    g = torch.Generator(device="cuda").manual_seed(5)
    x = bf(torch.randn(T, H, device="cuda", generator=g))
    w = bf(torch.randn(E, N, H, device="cuda", generator=g) * 0.05)
    plan = K().moe_route(bf(torch.randn(T, E, device="cuda", generator=g)), k)
    real = plan.slot_of_row >= 0
    for flags in (K().GEMM_TMA_STORE, K().GEMM_TMA_STORE | 8):  # default (CTA pair) / single-CTA kernel
        ref = K().gemm_grouped_m(K().moe_gather(x, plan), w, plan, b_mn=False, flags=flags)
        got = K().gemm_grouped_m_gather(x, w, plan, flags=flags)
        assert torch.equal(got[real], ref[real]), flags
    # and against fp64 on a few rows
    rows = torch.nonzero(real)[:: max(1, int(real.sum()) // 9)].flatten()[:8]
    tg = plan.tile_group.cpu()
    for r in rows.tolist():
        e = int(tg[r // 128])
        exact = x[int(plan.token_of_row[r])].double() @ w[e].double().t()
        assert torch.allclose(got[r].double(), exact, atol=2e-2, rtol=2e-2)


def test_moe_layer_matches_golden(golden_dir):
    """one SparseMoE layer, reference-derived fixture: y within bf16 tolerance, expert histogram bit exact"""
    from dolomite_engine_b200 import moe
    from dolomite_engine_b200.hf_models import MoEDolomiteConfig, MoEDolomiteForCausalLM

    fx = np.load(os.path.join(golden_dir, "moe_layer.npz"))
    cfg = MoEDolomiteConfig(vocab_size=256, n_embd=64, n_layer=1, n_head=4, n_inner=128, num_experts=8, num_experts_per_tok=2,
                            attention_head_type="mha", add_bias=False, position_embedding_type="rope",
                            normalization_function="rmsnorm", activation_function="swiglu", resid_pdrop=0, embd_pdrop=0,
                            attn_pdrop=0)
    model = MoEDolomiteForCausalLM(cfg, seed=0)
    sd = model.state_dict()
    sd["transformer.h.0.mlp.gate.weight"] = torch.from_numpy(fx["gate"])
    sd["transformer.h.0.mlp.c_fc.weight"] = torch.from_numpy(fx["c_fc"])
    sd["transformer.h.0.mlp.c_proj.weight"] = torch.from_numpy(fx["c_proj"])
    model.load_state_dict(sd)
    eng = model.engine
    x = bf(torch.from_numpy(fx["x"])).cuda()
    zero = torch.zeros_like(x)
    y, saved = moe.forward(eng, eng.units[1], "transformer.h.0.", x, zero, 1.0)
    torch.cuda.synchronize()
    ref = torch.from_numpy(fx["y"])
    assert rel_l2(y, ref) < 2e-2
    assert (y.float().cpu() - ref).abs().max() < 4 * 2.0**-8 * ref.abs().max() + 5e-3  # every element within ~4 bf16 ulp of the largest
    # bf16 router logits can reorder near-ties; the histogram must still sum to T*k
    assert int(saved[0].counts.sum().item()) == x.shape[0] * 2


@pytest.mark.parametrize("ragged", [False, True])
def test_moe_model_logits_loss_and_grads_match_oracle(ragged):
    from dolomite_engine_b200.hf_models import MoEDolomiteForCausalLM

    cfg, ocfg = _moe_cfgs()
    params = O.init_params(ocfg, seed=42)
    model = MoEDolomiteForCausalLM(cfg, seed=None)
    model.load_state_dict(params)
    model.assume_unit_loss_grad = True
    rng = np.random.default_rng(3)
    tokens = rng.integers(0, ocfg.vocab_size, size=(2, 97), dtype=np.int64)
    tokens[0, 30] = 7
    tokens[1, 60] = 7
    inp, labels = O.split_tokens(tokens)
    b = O.prepare_model_inputs(inp.copy(), 7, ragged, ragged)
    args = (torch.from_numpy(b["input_ids"]).cuda(), torch.from_numpy(b["position_ids"]).cuda(),
            torch.from_numpy(b["cu_seqlens"]).cuda(), b["max_seqlen"])
    # GPU forward first; its expert choices are pinned in the oracle (near-tied bf16 router logits may flip the
    # top-k, which is a property of the precision, not of the kernels -- the reference's own sort is unstable too)
    model.engine.zero_grad()
    lab = torch.from_numpy(np.ascontiguousarray(labels).reshape(-1)).cuda()
    loss = model.forward_pretraining_loss(*args, lab)
    routing = {f"transformer.h.{i}.mlp.": layer[-1][0].sel_idx.long().cpu() for i, layer in enumerate(model.engine._saved["layers"])}
    loss.backward()
    out = model(input_ids=args[0], position_ids=args[1], cu_seqlens=args[2], max_seqlen=args[3])
    logits = out.logits.float().cpu().detach()
    O.FORCED_ROUTING.clear()
    O.FORCED_ROUTING.update(routing)
    try:
        p_req = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        loss_ref, logits_ref = O.pretraining_loss(p_req, ocfg, tokens, 7, ragged, ragged, bf16=True)
        loss_ref.backward()
        # how often does the oracle's own (unpinned) choice agree with the GPU's?
        O.FORCED_ROUTING.clear()
        _, free_logits = O.pretraining_loss(params, ocfg, tokens, 7, ragged, ragged)
    finally:
        O.FORCED_ROUTING.clear()
    assert rel_l2(logits, logits_ref.detach()) < 1e-2
    assert abs(loss.item() - loss_ref.item()) / loss_ref.item() < 1e-3
    assert rel_l2(logits, free_logits.detach()) < 5e-2  # unpinned fp32 routing: only a few tokens may flip experts
    bad = []
    for pname, unit, spec in model.engine.named_views():
        e = rel_l2(unit.gviews[pname], p_req[pname].grad)
        if e > 3e-2:
            bad.append((pname, round(e, 4)))
    assert not bad, bad


def test_lazy_gradient_clearing_leaves_no_stale_expert_gradients():
    """zero_grad() does not touch the big weight-gradient buffers (the first wgrad GEMM of the window overwrites them): the
    gradients of batch B must not depend on what an earlier window (batch A) left in the buffers"""
    from dolomite_engine_b200.hf_models import MoEDolomiteForCausalLM

    cfg, ocfg = _moe_cfgs()
    model = MoEDolomiteForCausalLM(cfg, seed=None)
    model.load_state_dict(O.init_params(ocfg, seed=42))
    model.assume_unit_loss_grad = True
    eng = model.engine
    rng = np.random.default_rng(11)

    def run(tokens):
        inp, labels = O.split_tokens(tokens)
        b = O.prepare_model_inputs(inp.copy(), 7, False, False)
        eng.zero_grad()
        loss = model.forward_pretraining_loss(torch.from_numpy(b["input_ids"]).cuda(), torch.from_numpy(b["position_ids"]).cuda(),
                                              torch.from_numpy(b["cu_seqlens"]).cuda(), b["max_seqlen"],
                                              torch.from_numpy(np.ascontiguousarray(labels).reshape(-1)).cuda())
        loss.backward()
        torch.cuda.synchronize()
        return {n: u.gviews[n].clone() for n, u, _ in eng.named_views()}

    tok_a = rng.integers(0, ocfg.vocab_size, size=(2, 97), dtype=np.int64)
    tok_b = rng.integers(0, ocfg.vocab_size, size=(2, 97), dtype=np.int64)
    g1 = run(tok_b)  # buffers still hold the zeros of their allocation
    run(tok_a)
    g2 = run(tok_b)  # buffers hold batch A's gradients
    # not bit-equal: dQ tiles, router split-K partials and embedding rows are reduced with fp32 atomics (order-dependent
    # rounding, which now and then moves a bf16 activation gradient by one ulp: ~1e-5 relative on a whole tensor); a stale
    # buffer would show up as an O(1) relative difference
    for n in g1:
        assert rel_l2(g1[n], g2[n]) < 1e-3, n
