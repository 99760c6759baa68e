"""GPU: the bf16 GEMM's epilogue, which stages each output tile through shared memory and writes it with TMA stores
(reduce-adds for split-K) clipped by D's tensor map.

The cases are the ones that path makes new: D as a view whose row stride exceeds N, C aliasing D or separate from it, M
and N tails that do not fill a 64-row x 128-byte slab, bf16 and fp32 D with bias, alpha and beta, a K-grouped launch
with an expert that has no rows writing into a dirty buffer, and split-K."""

import pytest
import torch

pytestmark = pytest.mark.gpu

BF16_EPS = 2.0**-8
SENTINEL = -12345.0  # exactly representable in bf16 and fp32


def K():
    from dolomite_engine_b200 import kernels

    return kernels


def bf(x):
    return x.to(torch.bfloat16)


def _with_width(width, fn):
    old = K().get_option("gemm_tile_n")
    K().set_option("gemm_tile_n", width)
    try:
        return fn()
    finally:
        K().set_option("gemm_tile_n", old)


def _reference(A, B, b, C, alpha, beta):
    ref = A.double() @ B.double().t()
    if b is not None:
        ref = ref + b.double()
    ref = alpha * ref
    if C is not None:
        ref = ref + beta * C.double()
    return ref


def _check_accuracy(out, ref, dtype):
    out = out.double().cpu()
    if dtype == torch.bfloat16:
        assert (out - ref).abs().max() <= 2 * BF16_EPS * ref.abs().max()
    else:
        assert torch.allclose(out, ref, atol=1e-3, rtol=1e-4), (out - ref).abs().max()


# (M, N, K): M % 64 != 0 and N not a multiple of a slab's 64 bf16 / 32 fp32 columns (N % 8 == 0 only); the last shape has
# more tiles than SMs, so slabs are reused across tiles
SHAPES = [(200, 328, 136), (72, 8, 64), (1000, 1352, 200)]


@pytest.mark.parametrize("width", [128, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("shape", SHAPES)
def test_strided_view_tails_and_c_aliasing(shape, dtype, width):
    """D is a view into a larger buffer (row stride > N, rows below M): nothing outside the view is written.  C aliasing D
    and C in its own (differently strided) buffer give bit-identical results, which match fp64."""
    M, N, Kd = shape
    g = torch.Generator().manual_seed(M + N + Kd)
    A, B = bf(torch.randn(M, Kd, generator=g)), bf(torch.randn(N, Kd, generator=g))
    b = bf(torch.randn(N, generator=g))
    C = torch.randn(M, N, generator=g).to(dtype)
    alpha, beta = 0.75, -0.5
    a, bm, bias = A.cuda(), B.cuda(), b.cuda()
    pad_cols, pad_rows = 24, 70

    def run(alias):
        big = torch.full((M + pad_rows, N + pad_cols), SENTINEL, dtype=dtype, device="cuda")
        out = big[:M, :N]
        if alias:
            out.copy_(C.cuda())
            c = out
        else:
            cbig = torch.full((M, N + 40), float("nan"), dtype=dtype, device="cuda")
            c = cbig[:, :N]
            c.copy_(C.cuda())
        K().gemm(a, bm, out=out, c=c, alpha=alpha, beta=beta, bias=bias)
        torch.cuda.synchronize()
        return big

    big_alias = _with_width(width, lambda: run(True))
    big_sep = _with_width(width, lambda: run(False))
    assert torch.equal(big_alias, big_sep)
    assert torch.all(big_alias[:M, N:] == SENTINEL) and torch.all(big_alias[M:] == SENTINEL)
    _check_accuracy(big_alias[:M, :N], _reference(A, B, b, C, alpha, beta), dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_no_c_with_bias_overwrites_dirty_output(dtype):
    """without C the epilogue never reads D: a NaN-filled output is fully defined by (A B^T + bias) * alpha"""
    M, N, Kd = 264, 200, 328
    g = torch.Generator().manual_seed(7)
    A, B = bf(torch.randn(M, Kd, generator=g)), bf(torch.randn(N, Kd, generator=g))
    b = bf(torch.randn(N, generator=g))
    outs = []
    for width in (128, 256):
        out = torch.full((M, N), float("nan"), dtype=dtype, device="cuda")
        _with_width(width, lambda: K().gemm(A.cuda(), B.cuda(), out=out, alpha=2.0, bias=b.cuda()))
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    _check_accuracy(outs[0], _reference(A, B, b, None, 2.0, 0.0), dtype)


def test_k_grouped_empty_expert_into_dirty_buffer():
    """expert weight gradients (K-grouped, rank-3 output): an expert without rows gets an all-zero slice stored from a
    zeroed slab when the launch overwrites, and keeps its slice when it accumulates"""
    g = torch.Generator().manual_seed(11)
    T, E, k, F, H = 500, 8, 2, 200, 328  # F, H not multiples of a slab
    logits = torch.randn(T, E, generator=g)
    logits[:, 5] = -1e4
    plan = K().moe_route(bf(logits).cuda(), k)
    cnt = plan.counts.cpu().numpy()
    assert cnt[5] == 0
    xg = K().moe_gather(bf(torch.randn(T, H, generator=g)).cuda(), plan)
    y = bf(torch.randn(plan.max_rows, F, generator=g)).cuda()
    dw = torch.full((E, F, H), float("nan"), device="cuda")
    K().gemm_grouped_k(y, xg, plan, dw, beta=0.0)
    torch.cuda.synchronize()
    assert torch.all(dw[5] == 0) and not torch.isnan(dw).any()
    off = plan.offsets.cpu().numpy()
    y_c, x_c = y.double().cpu(), xg.double().cpu()
    for e in range(E):
        rows = slice(off[e], off[e] + cnt[e])
        ref = y_c[rows].t() @ x_c[rows]
        assert torch.allclose(dw[e].double().cpu(), ref, atol=1e-3, rtol=1e-4)
    once = dw.clone()
    dw[5] = 3.0
    K().gemm_grouped_k(y, xg, plan, dw, beta=1.0)
    torch.cuda.synchronize()
    assert torch.all(dw[5] == 3.0)
    assert torch.allclose(dw[:5], 2 * once[:5], rtol=1e-5, atol=1e-4)


def test_split_k_accumulate():
    """split-K partial tiles are reduce-added into fp32 D (C == D, beta == 1) and clipped at the M and N tails"""
    M, N, Kd = 136, 200, 8192
    g = torch.Generator().manual_seed(13)
    A, B = bf(torch.randn(M, Kd, generator=g)), bf(torch.randn(N, Kd, generator=g))
    C = torch.randn(M, N, generator=g)
    big = torch.full((M + 8, N + 8), SENTINEL, device="cuda")
    out = big[:M, :N]
    out.copy_(C.cuda())
    K().gemm(A.cuda(), B.cuda(), out=out, c=out, alpha=0.5, beta=1.0, flags=K().GEMM_SPLITK_ACCUMULATE)
    torch.cuda.synchronize()
    assert torch.all(big[:M, N:] == SENTINEL) and torch.all(big[M:] == SENTINEL)
    _check_accuracy(out, _reference(A, B, None, C, 0.5, 1.0), torch.float32)
