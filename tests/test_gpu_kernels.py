"""GPU parity tests: every CUDA kernel, called through the C ABI, against the CPU oracle on seeded inputs; plus
size-independent properties at the benchmark's full sizes (C2: T=8192, H=2560, F=10240, V=49152, S=4096, hd=80)."""

import math

import numpy as np
import pytest
import torch

import oracle.dolomite_oracle as O

pytestmark = pytest.mark.gpu

BF16_EPS = 2.0**-8  # one bf16 ulp relative


def K():
    from dolomite_engine_b200 import kernels

    return kernels


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def bf(x):
    return x.to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,H", [(1, 64), (37, 256), (200, 2560), (5, 8192)])
def test_rmsnorm_fwd_bwd(T, H):
    g = torch.Generator().manual_seed(0)
    x = bf(torch.randn(T, H, generator=g))
    w = bf(1 + 0.1 * torch.randn(H, generator=g))
    dy = bf(torch.randn(T, H, generator=g))
    y, rstd = K().rmsnorm_fwd(x.cuda(), w.cuda(), 1e-5)
    ref = O.rmsnorm(x.float(), w.float(), 1e-5, bf16=True)
    # same rounding points as the reference -> at most one bf16 ulp apart (rsqrt approximation)
    assert (y.float().cpu() - ref).abs().max() <= 2 * BF16_EPS * ref.abs().max()
    assert rel_l2(y, ref) < 1e-3
    xf = x.float().requires_grad_(True)
    wf = w.float().requires_grad_(True)
    O.rmsnorm(xf, wf, 1e-5).backward(dy.float())
    dw = torch.zeros(H, device="cuda")
    dx = K().rmsnorm_bwd(dy.cuda(), x.cuda(), w.cuda(), rstd, dw)
    assert rel_l2(dx, xf.grad) < 5e-3 and rel_l2(dw, wf.grad) < 5e-3


@pytest.mark.parametrize("ng,g,hd", [(4, 1, 64), (32, 1, 80), (2, 4, 128), (1, 4, 32)])
def test_rope_bit_exact_with_reference_rounding(ng, g, hd):
    gen = torch.Generator().manual_seed(1)
    T, npos = 96, 256
    qkv = bf(torch.randn(T, ng * (g + 2) * hd, generator=gen))
    cos, sin = O.rope_tables(hd, npos, 10000, bf16=True)
    pos = torch.randint(0, npos, (T,), generator=gen)
    v = qkv.float().view(T, ng, g + 2, hd)
    ref = v.clone()
    ref[:, :, : g + 1] = O.apply_rope(v[:, :, : g + 1], cos[pos][:, None, None], sin[pos][:, None, None], bf16=True)
    out = K().rope_qk_inplace(qkv.cuda().clone(), ng, g, hd, bf(cos).cuda(), bf(sin).cuda(), pos.cuda())
    assert torch.equal(out.float().cpu().view(T, ng, g + 2, hd), ref)  # bit exact, v slots untouched
    back = K().rope_qk_inplace(out.clone(), ng, g, hd, bf(cos).cuda(), bf(sin).cuda(), pos.int().cuda(), inverse=True)
    assert rel_l2(back, qkv) < 2e-2  # rotation is orthogonal: inverse(forward(x)) ~ x


def test_swiglu_fwd_bwd():
    g = torch.Generator().manual_seed(2)
    x = bf(torch.randn(77, 512, generator=g))
    dy = bf(torch.randn(77, 256, generator=g))
    y = K().swiglu_fwd(x.cuda())
    ref = O.activation(x.float(), "swiglu", bf16=True)
    assert (y.float().cpu() - ref).abs().max() <= 4 * BF16_EPS * ref.abs().max()
    xf = x.float().requires_grad_(True)
    O.activation(xf, "swiglu").backward(dy.float())
    dx = K().swiglu_bwd(dy.cuda(), x.cuda())
    assert rel_l2(dx, xf.grad) < 5e-3
    # fused variant: identical dx, plus the bias gradient of the producing linear (column sums of the bf16 dx),
    # accumulated on top of what is already in the buffer; ragged row / column-tile counts
    for T, F in [(77, 256), (1000, 328), (8, 8)]:
        x2, dy2 = bf(torch.randn(T, 2 * F, generator=g)).cuda(), bf(torch.randn(T, F, generator=g)).cuda()
        plain = K().swiglu_bwd(dy2, x2)
        db = torch.full((2 * F,), 0.5, device="cuda")
        fused = K().swiglu_bwd(dy2, x2, bias_grad_accum=db)
        assert torch.equal(fused, plain)
        want = 0.5 + plain.float().sum(0)
        assert torch.allclose(db, want, rtol=1e-5, atol=1e-4), (T, F, (db - want).abs().max().item())


def test_embedding_exact_and_grad():
    g = torch.Generator().manual_seed(3)
    wte = bf(torch.randn(512, 64, generator=g))
    ids = torch.randint(0, 512, (300,), generator=g)
    assert torch.equal(K().embedding_fwd(ids.cuda(), wte.cuda()).cpu(), wte[ids])
    dout = bf(torch.randn(300, 64, generator=g))
    dw = torch.zeros(512, 64, device="cuda")
    K().embedding_bwd(ids.cuda(), dout.cuda(), dw)
    ref = torch.zeros(512, 64).index_add_(0, ids, dout.float())
    assert torch.allclose(dw.cpu(), ref, atol=1e-5)


@pytest.mark.parametrize("T,V", [(1, 64), (50, 2048), (9, 49152)])
def test_cross_entropy_fwd_bwd(T, V):
    g = torch.Generator().manual_seed(4)
    logits = bf(torch.randn(T, V, generator=g) * 3)
    labels = torch.randint(0, V, (T,), generator=g)
    if T > 4:
        labels[::5] = -100
    lf = logits.float().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(lf, labels, ignore_index=-100)
    ref.backward()
    loss, loss_tok, dl = K().cross_entropy_fwd_bwd(logits.cuda(), labels.cuda())
    assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item()) + 1e-6
    assert rel_l2(dl, lf.grad) < 5e-3
    # property: every gradient row sums to ~0 (softmax - onehot), ignored rows are exactly 0
    rows = dl.float().sum(-1).cpu()
    assert rows.abs().max() < 2e-2 / max(1, (labels != -100).sum().item())
    assert torch.all(dl[labels.cuda() == -100] == 0)


@pytest.mark.parametrize("M,N,Kd,a_mn,b_mn", [(128, 256, 64, False, False), (300, 520, 328, False, False),
                                              (200, 264, 136, False, True), (136, 72, 400, True, True), (64, 8, 8, True, False)])
def test_gemm_vs_oracle(M, N, Kd, a_mn, b_mn):
    g = torch.Generator().manual_seed(5)
    A = bf(torch.randn(M, Kd, generator=g))
    B = bf(torch.randn(N, Kd, generator=g))
    bias = bf(torch.randn(N, generator=g))
    ref = O.linear(A.float(), B.float(), bias.float(), bf16=True)
    a = (A.t().contiguous() if a_mn else A).cuda()
    b = (B.t().contiguous() if b_mn else B).cuda()
    # bit0: bf16 D without C; bit2 / bit3: CTA-pair flags (accepted, no effect on sm_90)
    for flags in (0, 1, 4, 5, 8, 9):
        out = K().gemm(a, b, a_mn=a_mn, b_mn=b_mn, bias=bias.cuda(), flags=flags)
        # fp32 accumulation order differs from the CPU: allow one bf16 ulp of the result magnitude
        assert (out.float().cpu() - ref).abs().max() <= 2 * BF16_EPS * ref.abs().max()
    out32 = K().gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32)
    assert torch.allclose(out32.cpu(), A.float() @ B.float().t(), atol=1e-3, rtol=1e-4)


def test_gemm_epilogue_alpha_beta_accumulate():
    g = torch.Generator().manual_seed(6)
    A, B = bf(torch.randn(160, 96, generator=g)), bf(torch.randn(264, 96, generator=g))
    C = torch.randn(160, 264, generator=g)
    d = C.cuda().clone()
    K().gemm(A.cuda(), B.cuda(), out=d, c=d, alpha=0.5, beta=1.0)
    assert torch.allclose(d.cpu(), C + 0.5 * (A.float() @ B.float().t()), atol=1e-3, rtol=1e-4)


def test_gemm_tile_schedules_are_bit_identical():
    """the `gemm_dynamic` option (a tile-scheduling choice of other GPU generations, accepted on sm_90) never changes the
    arithmetic: outputs are bit-identical for every operand layout / epilogue flag, with many more tiles than SMs"""
    g = torch.Generator().manual_seed(12)
    default = K().get_option("gemm_dynamic")
    cases = [(4096, 4096, 512, False, False, 5, torch.bfloat16), (1024, 3072, 1024, False, True, 5, torch.bfloat16),
             (640, 512, 2048, True, True, 4, torch.float32), (4096 + 64, 2048, 256, False, False, 8, torch.bfloat16),
             (300, 520, 328, False, False, 5, torch.bfloat16), (100, 2560, 2560, False, False, 0, torch.bfloat16)]
    try:
        for M, N, Kd, a_mn, b_mn, flags, dt in cases:
            A, B = bf(torch.randn(M, Kd, generator=g)), bf(torch.randn(N, Kd, generator=g))
            a = (A.t().contiguous() if a_mn else A).cuda()
            b = (B.t().contiguous() if b_mn else B).cuda()
            outs = []
            for dyn in (0, 1):
                K().set_option("gemm_dynamic", dyn)
                outs.append(K().gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=dt, flags=flags if dt == torch.bfloat16 else flags & ~1))
            assert torch.equal(outs[0], outs[1]), (M, N, Kd, a_mn, b_mn, flags)
            ref = A.float() @ B.float().t()
            assert rel_l2(outs[1], ref) < 5e-3
    finally:
        K().set_option("gemm_dynamic", default)


@pytest.mark.parametrize("M,N,Kd", [(8, 2048, 4096), (264, 520, 1024)])
def test_gemm_split_k_accumulate(M, N, Kd):
    """D (fp32) += A^T B with the contraction split over several CTAs (fp32 vector atomics): the MoE gate weight gradient
    (E = 8 output rows, the whole token stream as contraction; moe.py backward)"""
    g = torch.Generator().manual_seed(11)
    A, B = bf(torch.randn(Kd, M, generator=g) * 0.1), bf(torch.randn(Kd, N, generator=g) * 0.1)
    C = torch.randn(M, N, generator=g)
    default = K().get_option("gemm_dynamic")
    for dyn in (0, 1):  # both values of the scheduling option
        try:
            K().set_option("gemm_dynamic", dyn)
            d = C.cuda().clone()
            K().gemm(A.cuda(), B.cuda(), a_mn=True, b_mn=True, out=d, c=d, beta=1.0, flags=K().GEMM_SPLITK_ACCUMULATE)
        finally:
            K().set_option("gemm_dynamic", default)
        ref = C + A.float().t() @ B.float()
        assert torch.allclose(d.cpu(), ref, atol=2e-3, rtol=1e-4), dyn


def _attn_inputs(lens, ng, g, hd, seed=7):
    gen = torch.Generator().manual_seed(seed)
    T = sum(lens)
    qkv = bf(torch.randn(T, ng * (g + 2) * hd, generator=gen))
    dout = bf(torch.randn(T, ng * g * hd, generator=gen))
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return qkv, dout, cu


@pytest.mark.parametrize("lens,ng,g,hd", [([128], 2, 1, 64), ([100, 37, 300, 1, 129], 4, 1, 64), ([200, 130, 515], 2, 1, 80),
                                          ([300, 77, 260], 2, 4, 128), ([150, 250], 1, 4, 32), ([1], 1, 1, 16)])
def test_attention_fwd_bwd_vs_oracle(lens, ng, g, hd):
    qkv, dout, cu = _attn_inputs(lens, ng, g, hd)
    T = qkv.shape[0]
    scale = 1.0 / math.sqrt(hd)
    cfg = O.OracleConfig(n_embd=ng * g * hd, n_head=ng * g, num_key_value_heads=ng,
                         attention_head_type="mha" if g == 1 else "gqa")
    x = qkv.float().requires_grad_(True)
    q, k, v = O.split_qkv_activations(x, cfg)
    ref = O.packed_causal_attention(q, k, v, cu, scale)
    ref.backward(dout.float())
    out, lse = K().attn_varlen_fwd(qkv.cuda(), torch.from_numpy(cu).cuda(), max(lens), ng, g, hd, scale)
    assert rel_l2(out, ref) < 6e-3
    if hd >= 64:  # every forward kernel (single-buffer / split softmax with two or four threads per row) of the head_dim
        default_split = K().get_option("attn_fwd_split")
        for split in (0, 2, 3):
            try:
                K().set_option("attn_fwd_split", split)
                out2, lse2 = K().attn_varlen_fwd(qkv.cuda(), torch.from_numpy(cu).cuda(), max(lens), ng, g, hd, scale)
            finally:
                K().set_option("attn_fwd_split", default_split)
            assert rel_l2(out2, ref) < 6e-3, split
            assert torch.allclose(lse2, lse, atol=2e-3, rtol=1e-4), split
    # head_dim <= 80 runs the pipelined backward, larger head dims the serial one: both are covered by the parameter list
    dqkv = K().attn_varlen_bwd(dout.cuda(), qkv.cuda(), out, lse, torch.from_numpy(cu).cuda(), max(lens), ng, g, hd, scale)
    assert rel_l2(dqkv, x.grad) < 1.2e-2
    if hd in (64, 80):  # the other variants of the pipelined backward (0 = round-1 softmax warps, 1 = lean; default 2)
        for variant in (0, 1):
            try:
                K().set_option("attn_bwd_variant", variant)
                dq2 = K().attn_varlen_bwd(dout.cuda(), qkv.cuda(), out, lse, torch.from_numpy(cu).cuda(), max(lens), ng, g, hd, scale)
            finally:
                K().set_option("attn_bwd_variant", 2)
            assert rel_l2(dq2, x.grad) < 1.2e-2, variant


# ------------------------------------------------------------------------------------------------
# full-size (C2) properties
# ------------------------------------------------------------------------------------------------
def test_full_size_gemm_spot_checks():
    T, H, F = 8192, 2560, 10240
    g = torch.Generator(device="cuda").manual_seed(8)
    x = bf(torch.randn(T, H, device="cuda", generator=g))
    w = bf(torch.randn(2 * F, H, device="cuda", generator=g) * 0.02)
    y = K().gemm(x, w, out_dtype=torch.float32)
    rows = torch.randint(0, T, (16,), generator=torch.Generator().manual_seed(9))
    cols = torch.randint(0, 2 * F, (16,), generator=torch.Generator().manual_seed(10))
    exact = (x[rows.cuda()].double().cpu() @ w[cols.cuda()].double().cpu().t())
    got = y[rows.cuda()][:, cols.cuda()].double().cpu()
    assert torch.allclose(got, exact, atol=1e-3, rtol=1e-4)
    # checksum of checksums: sum_n y[m, n] == x[m] . (sum_n w[n])
    wsum = w.double().sum(0)
    assert torch.allclose(y[rows.cuda()].double().sum(-1).cpu(), (x[rows.cuda()].double() @ wsum).cpu(), atol=5e-2, rtol=1e-3)
    # wgrad form (both operands MN-major), fp32 accumulate twice == 2x
    dy = bf(torch.randn(T, 512, device="cuda", generator=g))
    dw = torch.zeros(512, H, device="cuda")
    K().gemm(dy, x, a_mn=True, b_mn=True, out=dw, c=dw, beta=1.0)
    once = dw.clone()
    K().gemm(dy, x, a_mn=True, b_mn=True, out=dw, c=dw, beta=1.0)
    assert torch.allclose(dw, 2 * once, rtol=1e-5, atol=1e-3)
    exact = dy[:, :8].double().t().cpu() @ x[:, :8].double().cpu()
    assert torch.allclose(once[:8, :8].double().cpu(), exact, atol=5e-2, rtol=1e-3)


@pytest.mark.parametrize("tma_epilogue", [False, True])
def test_block_weight_gradients_in_one_launch_and_fp32_tile_epilogues(tma_epilogue):
    """gemm_wgrad_multi (the four weight gradients of a block in one persistent launch, TMA store / reduce-add epilogue)
    == four separate GEMMs == fp64 products on sampled entries; overwrite and accumulate forms; ragged M / N edges.
    Also: the fp32 TMA epilogue and the per-thread epilogue of the single-problem GEMM agree bit for bit."""
    g = torch.Generator(device="cuda").manual_seed(21)
    T = 2048 + 64  # not a multiple of the 64-row contraction block
    shapes = [(2560, 1024), (520, 2560), (264, 264), (7680, 328)]  # (M = out features, N = in features)
    probs, refs = [], []
    for i, (M, N) in enumerate(shapes):
        dy = bf(torch.randn(T, M, device="cuda", generator=g))
        x = bf(torch.randn(T, N, device="cuda", generator=g))
        acc = i % 2 == 1
        dw = torch.randn(M, N, device="cuda", generator=g) if acc else torch.full((M, N), float("nan"), device="cuda")
        ref = (dw.clone() if acc else torch.zeros(M, N, device="cuda"))
        alpha = 1.0 if i != 2 else 0.5
        probs.append((dy, x, dw, alpha, acc))
        refs.append((ref, dy, x, alpha))
    K().set_option("gemm_f32_tma_epilogue", int(tma_epilogue))
    try:
        K().gemm_wgrad_multi(probs)
        torch.cuda.synchronize()
    finally:
        K().set_option("gemm_f32_tma_epilogue", 0)
    for (dy, x, dw, alpha, acc), (ref, _, _, _) in zip(probs, refs):
        sep = ref.clone()
        if acc:
            K().gemm(dy, x, a_mn=True, b_mn=True, out=sep, c=sep, alpha=alpha, beta=1.0, flags=K().GEMM_DIRECT_EPILOGUE)
        else:
            K().gemm(dy, x, a_mn=True, b_mn=True, out=sep, alpha=alpha, flags=K().GEMM_DIRECT_EPILOGUE)
        assert torch.isfinite(dw).all()
        # same tiles, same fp32 accumulation order; only the final add differs (L2 reduce-add vs register add): <= 1 ulp
        assert torch.allclose(dw, sep, rtol=1e-6, atol=1e-5), (dw - sep).abs().max()
        rows = torch.randint(0, dw.shape[0], (12,), generator=torch.Generator().manual_seed(3)).cuda()
        cols = torch.randint(0, dw.shape[1], (12,), generator=torch.Generator().manual_seed(4)).cuda()
        exact = alpha * (dy[:, rows].double().t() @ x[:, cols].double()) + ref[rows][:, cols].double()
        assert torch.allclose(dw[rows][:, cols].double(), exact, atol=2e-2, rtol=1e-3)
    # single-problem GEMM: TMA tile epilogue (default) vs per-thread epilogue
    dy, x = probs[0][0], probs[0][1]
    a = torch.empty(2560, 1024, device="cuda")
    b = torch.empty(2560, 1024, device="cuda")
    K().gemm(dy, x, a_mn=True, b_mn=True, out=a, flags=K().GEMM_F32_TMA_EPILOGUE)
    K().gemm(dy, x, a_mn=True, b_mn=True, out=b, flags=K().GEMM_DIRECT_EPILOGUE)
    assert torch.equal(a, b)


def test_full_size_attention_properties():
    S, B, nh, hd = 4096, 2, 32, 80
    T = S * B
    g = torch.Generator(device="cuda").manual_seed(11)
    qkv = bf(torch.randn(T, nh * 3 * hd, device="cuda", generator=g))
    v = qkv.view(T, nh, 3, hd)
    v[:, :, 2] = 1.0  # V = ones -> every output element must be 1 (softmax rows sum to one)
    cu = torch.arange(0, T + 1, S, dtype=torch.int32, device="cuda")
    out, lse = K().attn_varlen_fwd(qkv, cu, S, nh, 1, hd, hd**-0.5)
    assert (out.float() - 1).abs().max() < 1e-2
    # first token of each document attends only to itself: lse == scale * q.k
    for d in range(B):
        q0 = v[d * S, :, 0].float()
        k0 = v[d * S, :, 1].float()
        assert torch.allclose(lse[:, d * S], (q0 * k0).sum(-1) * hd**-0.5, atol=2e-3, rtol=1e-4)
    # spot-check a few late rows against an exact CPU softmax
    for (t, h) in [(4095, 3), (5000, 17), (8191, 31)]:
        d0 = (t // S) * S
        q = v[t, h, 0].double().cpu()
        keys = v[d0 : t + 1, h, 1].double().cpu()
        s = (keys @ q) * hd**-0.5
        assert abs(lse[h, t].item() - torch.logsumexp(s, 0).item()) < 2e-3


def test_full_size_cross_entropy_properties():
    T, V = 8192, 49152
    g = torch.Generator(device="cuda").manual_seed(12)
    logits = bf(torch.randn(T, V, device="cuda", generator=g))
    labels = torch.randint(0, V, (T,), device="cuda", generator=g)
    keep = logits[:4].float().cpu()
    loss, loss_tok, dl = K().cross_entropy_fwd_bwd(logits, labels)
    ref = torch.nn.functional.cross_entropy(keep, labels[:4].cpu(), reduction="none")
    assert torch.allclose(loss_tok[:4].cpu(), ref, atol=1e-4, rtol=1e-5)
    assert abs(loss.item() - loss_tok.mean().item()) < 1e-5
    assert dl.float().sum(-1).abs().max().item() < 1e-5  # rows of (softmax - onehot)/T sum to zero


def test_optimizer_kernels_vs_torch():
    n = 100_003
    g = torch.Generator().manual_seed(13)
    p0, grad = torch.randn(n, generator=g), torch.randn(n, generator=g) * 0.1
    pr = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([pr], lr=1e-3, betas=(0.9, 0.95), eps=1e-10, weight_decay=0.1)
    p, m, v = p0.cuda(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    pb = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    ss, coef, norm = torch.zeros(1, device="cuda"), torch.empty(1, device="cuda"), torch.empty(1, device="cuda")
    K().sumsq_accum(grad.cuda(), ss)
    K().clip_coef(ss, 1.0, coef, norm)
    c = min(1.0, 1.0 / (grad.norm().item() + 1e-6))
    assert abs(norm.item() - grad.norm().item()) < 1e-3 and abs(coef.item() - c) < 1e-6
    for step in (1, 2, 3):
        pr.grad = grad * c
        opt.step()
        K().adamw_step(p, grad.cuda(), m, v, pb, 1e-3, 0.9, 0.95, 1e-10, 0.1, step, clip=coef)
    assert torch.allclose(p.cpu(), pr.data, atol=1e-6, rtol=1e-5)
    assert torch.equal(pb.cpu(), bf(p.cpu()))


@pytest.mark.parametrize("T,H,bias", [(1, 64, True), (37, 256, True), (200, 2560, False), (5, 8192, True)])
def test_layernorm_fwd_bwd(T, H, bias):
    """normalization_function layernorm = torch.nn.LayerNorm: fp32 statistics, one bf16 rounding (oracle.layernorm)"""
    g = torch.Generator().manual_seed(0)
    x = bf(torch.randn(T, H, generator=g) + 0.5)
    w = bf(1 + 0.1 * torch.randn(H, generator=g))
    b = bf(0.1 * torch.randn(H, generator=g)) if bias else None
    dy = bf(torch.randn(T, H, generator=g))
    dres = bf(torch.randn(T, H, generator=g))
    y, mean, rstd = K().layernorm_fwd(x.cuda(), w.cuda(), None if b is None else b.cuda(), 1e-5)
    ref = O.layernorm(x.float(), w.float(), None if b is None else b.float(), 1e-5, bf16=True)
    assert (y.float().cpu() - ref).abs().max() <= 2 * BF16_EPS * max(ref.abs().max().item(), 1.0)
    assert torch.allclose(mean.cpu(), x.float().mean(-1), atol=1e-5)
    xf = x.float().requires_grad_(True)
    wf = w.float().requires_grad_(True)
    bfp = b.float().requires_grad_(True) if bias else None
    O.layernorm(xf, wf, bfp, 1e-5).backward(dy.float())
    dw = torch.zeros(H, device="cuda")
    db = torch.zeros(H, device="cuda") if bias else None
    dx = K().layernorm_bwd(dy.cuda(), x.cuda(), w.cuda(), mean, rstd, dw, db, dx_add=dres.cuda())
    assert rel_l2(dx, xf.grad + dres.float()) < 5e-3 and rel_l2(dw, wf.grad) < 5e-3
    if bias:
        assert rel_l2(db, bfp.grad) < 1e-4


def test_gelu_tanh_fwd_bwd_and_fused_bias_gradient():
    """activation_function gelu_pytorch_tanh (non-GLU MLP, gpt_dolomite/mlp.py:45-50)"""
    g = torch.Generator().manual_seed(2)
    for T, F in [(77, 256), (1000, 328), (8, 8)]:
        x = bf(torch.randn(T, F, generator=g) * 2)
        dy = bf(torch.randn(T, F, generator=g))
        y = K().gelu_fwd(x.cuda())
        ref = O.activation(x.float(), "gelu_pytorch_tanh", bf16=True)
        assert (y.float().cpu() - ref).abs().max() <= 2 * BF16_EPS * max(ref.abs().max().item(), 1.0)
        xf = x.float().requires_grad_(True)
        O.activation(xf, "gelu_pytorch_tanh").backward(dy.float())
        plain = K().gelu_bwd(dy.cuda(), x.cuda())
        assert rel_l2(plain, xf.grad) < 5e-3
        db = torch.full((F,), 0.25, device="cuda")
        fused = K().gelu_bwd(dy.cuda(), x.cuda(), bias_grad_accum=db)
        assert torch.equal(fused, plain)
        want = 0.25 + plain.float().sum(0)
        assert torch.allclose(db, want, rtol=1e-5, atol=1e-4)


@pytest.mark.parametrize("lens,ng,g,hd", [([130, 0, 64, 0], 2, 1, 80), ([0, 5], 1, 2, 64), ([70, 200], 2, 1, 96),
                                          ([257], 1, 1, 80), ([127, 129, 128], 2, 1, 64)])
def test_attention_edge_cases_empty_documents_and_tile_boundaries(lens, ng, g, hd):
    """cu_seqlens with empty documents (consecutive equal entries, what `reset_attention_mask` produces for back-to-back
    EOS), lengths on either side of the 128-row tile boundary, head_dim 96"""
    qkv, dout, cu = _attn_inputs(lens, ng, g, hd, seed=11)
    scale = 1.0 / math.sqrt(hd)
    cfg = O.OracleConfig(n_embd=ng * g * hd, n_head=ng * g, num_key_value_heads=ng,
                         attention_head_type="mha" if g == 1 else "gqa")
    x = qkv.float().requires_grad_(True)
    q, k, v = O.split_qkv_activations(x, cfg)
    ref = O.packed_causal_attention(q, k, v, cu, scale)
    ref.backward(dout.float())
    cu_d = torch.from_numpy(cu).cuda()
    out, lse = K().attn_varlen_fwd(qkv.cuda(), cu_d, max(lens), ng, g, hd, scale)
    assert rel_l2(out, ref) < 6e-3
    dqkv = K().attn_varlen_bwd(dout.cuda(), qkv.cuda(), out, lse, cu_d, max(lens), ng, g, hd, scale)
    assert rel_l2(dqkv, x.grad) < 1.2e-2


def test_empty_and_single_row_inputs_are_accepted():
    """T = 0 launches nothing and returns; T = 1 works for every HBM kernel"""
    k = K()
    for T in (0, 1):
        x = torch.randn(T, 256, device="cuda").bfloat16()
        w = torch.ones(256, device="cuda").bfloat16()
        y, rstd = k.rmsnorm_fwd(x, w, 1e-5)
        assert tuple(y.shape) == (T, 256) and tuple(rstd.shape) == (T,)
        dw = torch.zeros(256, device="cuda")
        assert tuple(k.rmsnorm_bwd(x, x, w, rstd, dw).shape) == (T, 256)
        assert tuple(k.swiglu_fwd(torch.randn(T, 512, device="cuda").bfloat16()).shape) == (T, 256)
        assert tuple(k.gelu_fwd(torch.randn(T, 512, device="cuda").bfloat16()).shape) == (T, 512)
        ids = torch.zeros(T, dtype=torch.int64, device="cuda")
        assert tuple(k.embedding_fwd(ids, torch.randn(16, 64, device="cuda").bfloat16()).shape) == (T, 64)
    torch.cuda.synchronize()
