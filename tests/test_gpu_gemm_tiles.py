"""GPU: the 128 x 256 output tile of the dense bf16 GEMM (wgmma m64n256k16) against the 128 x 128 tile and against fp64,
the same bits on fewer SMs (gemm_sm_margin), and the per-launch choice of the tile width.

Each output element sees the same k16 MMA sequence in the same order at both widths, so the results are bit-identical."""

import contextlib
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BF16_EPS = 2.0**-8  # one bf16 ulp relative


def K():
    from dolomite_engine_b200 import kernels

    return kernels


def bf(x):
    return x.to(torch.bfloat16)


@contextlib.contextmanager
def tile_n(width):
    old = K().get_option("gemm_tile_n")
    K().set_option("gemm_tile_n", width)
    try:
        yield
    finally:
        K().set_option("gemm_tile_n", old)


def at_both_widths(fn):
    outs = []
    for width in (128, 256):
        with tile_n(width):
            outs.append(fn())
    torch.cuda.synchronize()
    return outs


SM_MARGINS = (1, 37, 64)  # SMs left out of the persistent schedule: each worker then runs more tiles through the ring


def at_sm_margins(fn):
    """fn at both tile widths with each gemm_sm_margin (0 is the library default)"""
    outs = []
    old = K().get_option("gemm_sm_margin")
    try:
        for margin in SM_MARGINS:
            K().set_option("gemm_sm_margin", margin)
            outs.extend(at_both_widths(fn))
    finally:
        K().set_option("gemm_sm_margin", old)
    return outs


# (M, N, K, D dtype, bias, (alpha, beta) or None for no C).  M tails (M % 128 != 0), N % 256 in {8, 128, 136}, K % 64 != 0;
# the last case has more tiles than SMs at both widths, so every CTA runs several tiles through the stage ring.
CASES = [
    (200, 264, 328, torch.bfloat16, True, None),
    (328, 384, 200, torch.float32, False, (0.5, 1.0)),
    (520, 392, 136, torch.bfloat16, True, (0.75, 0.5)),
    (136, 136, 72, torch.float32, True, (1.0, 0.0)),
    (2112, 2440, 520, torch.bfloat16, True, None),
    (2112, 2440, 520, torch.float32, False, (2.0, -1.0)),
]


def _operands(M, N, Kd, d_dtype, bias, ab, seed):
    g = torch.Generator().manual_seed(seed)
    A = bf(torch.randn(M, Kd, generator=g))
    B = bf(torch.randn(N, Kd, generator=g))
    b = bf(torch.randn(N, generator=g)) if bias else None
    C = torch.randn(M, N, generator=g).to(d_dtype) if ab is not None else None
    return A, B, b, C


def _reference(A, B, b, C, ab):
    ref = A.double() @ B.double().t()
    alpha, beta = ab if ab is not None else (1.0, 0.0)
    if b is not None:
        ref = ref + b.double()
    ref = alpha * ref
    if C is not None:
        ref = ref + beta * C.double()
    return ref


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_tile_widths_bit_identical_and_accurate(a_mn, b_mn, case):
    M, N, Kd, d_dtype, bias, ab = CASES[case]
    A, B, b, C = _operands(M, N, Kd, d_dtype, bias, ab, seed=100 + case)
    a = (A.t().contiguous() if a_mn else A).cuda()
    bm = (B.t().contiguous() if b_mn else B).cuda()
    alpha, beta = ab if ab is not None else (1.0, 0.0)

    def run():
        out = torch.empty(M, N, dtype=d_dtype, device="cuda")
        c = None
        if C is not None:
            out.copy_(C.cuda())
            c = out
        return K().gemm(a, bm, a_mn=a_mn, b_mn=b_mn, out=out, c=c, alpha=alpha, beta=beta,
                        bias=None if b is None else b.cuda())

    o128, o256 = at_both_widths(run)
    assert torch.equal(o128, o256), (M, N, Kd, a_mn, b_mn, (o128.float() - o256.float()).abs().max().item())
    for i, o in enumerate(at_sm_margins(run)):
        assert torch.equal(o, o128), (M, N, Kd, a_mn, b_mn, SM_MARGINS[i // 2])

    ref = _reference(A, B, b, C, ab)
    for out in (o128, o256):
        out = out.double().cpu()
        if d_dtype == torch.bfloat16:
            # the oracle tolerance of the bf16 GEMM: one rounding of the result, fp32 accumulation in another order
            assert (out - ref).abs().max() <= 2 * BF16_EPS * ref.abs().max()
        else:
            assert torch.allclose(out, ref, atol=1e-3, rtol=1e-4), (out - ref).abs().max()


def test_wgrad_multi_tile_widths_bit_identical_and_accurate():
    """four weight gradients of unequal sizes in one launch, two overwriting and two accumulating"""
    g = torch.Generator().manual_seed(21)
    T = 328
    shapes = [(384, 264), (200, 520), (136, 136), (520, 392)]
    alphas = [1.0, 0.5, 2.0, 0.25]
    accumulate = [False, True, False, True]
    dys = [bf(torch.randn(T, m, generator=g)) for m, _ in shapes]
    xs = [bf(torch.randn(T, n, generator=g)) for _, n in shapes]
    dw0 = [torch.randn(m, n, generator=g) for m, n in shapes]

    def run():
        dws = [w.cuda() for w in dw0]
        K().gemm_wgrad_multi([(dy.cuda(), x.cuda(), dw, al, acc)
                              for dy, x, dw, al, acc in zip(dys, xs, dws, alphas, accumulate)])
        return dws

    w128, w256 = at_both_widths(run)
    margins = at_sm_margins(run)
    for q in range(len(shapes)):
        assert torch.equal(w128[q], w256[q]), q
        assert all(torch.equal(w[q], w128[q]) for w in margins), q
        ref = alphas[q] * (dys[q].double().t() @ xs[q].double()) + (dw0[q].double() if accumulate[q] else 0.0)
        for w in (w128[q], w256[q]):
            assert torch.allclose(w.double().cpu(), ref, atol=1e-3, rtol=1e-4), (q, (w.double().cpu() - ref).abs().max())


def test_automatic_tile_choice():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert K().get_option("gemm_tile_n") == 0, "the library default is the automatic choice"
    margin = K().get_option("gemm_sm_margin")
    workers = sms - margin

    # 4096 x 20480 (the MLP c_fc forward of C2): 640 tiles of 128 x 256, both widths fill their waves
    width, cost = K().gemm_tile_n([(4096, 20480)])
    assert width == 256
    assert 1.0 < cost < 2.0, "a 128 x 256 tile does twice the work of a 128 x 128 one"

    # 4096 x 2560 (attention / MLP c_proj forward and the dgrads of C2): 640 tiles of 128 x 128 but 320 of 128 x 256; on
    # 132 workers 5 waves against 3, so the wide tile wins iff c_256 / c_128 < 5 / 3
    w128 = math.ceil(32 * 20 / workers)
    w256 = math.ceil(32 * 10 / workers)
    width, cost = K().gemm_tile_n([(4096, 2560)])
    assert width == (256 if w256 * cost < w128 else 128), (width, cost, w128, w256)

    # one tile either way: the narrow tile is cheaper
    assert K().gemm_tile_n([(128, 200)])[0] == 128
    # a weight-gradient launch counts the tiles of all its problems
    width, _ = K().gemm_tile_n([(7680, 2560), (2560, 2560), (20480, 2560), (2560, 10240)])
    t128 = 60 * 20 + 20 * 20 + 160 * 20 + 20 * 80
    t256 = 60 * 10 + 20 * 10 + 160 * 10 + 20 * 40
    assert width == (256 if math.ceil(t256 / workers) * cost < math.ceil(t128 / workers) else 128)

    for forced in (128, 256):
        with tile_n(forced):
            assert K().gemm_tile_n([(4096, 2560)])[0] == forced
            assert K().gemm_tile_n([(128, 200)])[0] == forced
    from dolomite_engine_b200 import _lib

    with pytest.raises(_lib.DolomiteB200Error, match="gemm_tile_n"):
        K().set_option("gemm_tile_n", 192)
    assert K().get_option("gemm_tile_n") == 0
