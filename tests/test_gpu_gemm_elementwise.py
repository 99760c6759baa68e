"""GPU: every bf16 and fp8 GEMM instance, through every entry point that runs it, element by element.

The cases are those of tests/gemm_instances.py (test_gemm_sass.py checks on the CPU that they reach every built
instance).  Each case runs twice:

- random inputs (N(0, 1); rows and columns scaled by 2^+-6; rows built to cancel, so that exact results lie near 0)
  against the fp64 product of the kernel's own bf16 / fp8 inputs, with a bar per element that follows the kernel's
  rounding points (below);
- exact-arithmetic inputs (small halves or integers, power-of-two scales, alpha and beta), where every fp32 partial sum
  of the pipeline is exact, so D must equal the fp64 result rounded once to D's type, bit for bit.  A misplaced row,
  column, k-block, bias pair, C chunk or group fails at zero tolerance, and split-K loses its nondeterminism.

The bar of an element.  Products are exact in fp32 (8 x 8 and 4 x 4 significand bits).  One tensor-core step sums
m = 16 (bf16 k16) or 32 (fp8 k32) products with the accumulator; each of those m + 1 addends is aligned to the largest
and kept to the accumulator's width, so it loses less than u_acc times the largest, which is at most S = sum_k |a_k b_k|.
The width is what the probe tests measure (J_BF16, J_FP8 bits below the leading one: u_acc = 2^-J).  Over n steps and
fp32 promotions (the split accumulator's adds, split-K's reduce-adds) the accumulator is off by at most
(m + 1) n u_acc S.  The epilogue (s acc + bias) alpha + beta C adds one fp32 rounding of its own magnitude per
operation, and a bf16 D one rounding of up to 2^-8 of its value.  No bar is a fraction of a tensor-wide norm.

Exact invariants: the L2 eviction hints on and off, gemm_wgrad_multi / gemm_fp8_wgrad_multi against the same problems
run alone and in another order, row-strided operand views against contiguous ones, D's padding columns
[N, round_up(N, 16 B)) written as zeros and nothing after them, two runs giving the same bits.
"""

import pytest
import torch

from gemm_instances import CASES, HINT_SHAPE
from test_fp8 import FP8_MAX, dequantize_ref, quantize_ref

pytestmark = pytest.mark.gpu

U32 = 2.0**-24  # fp32 rounding to nearest
BF16_U = 2.0**-8  # bf16 rounding to nearest: 8 significand bits, so up to 2^-8 of the value (not 2^-9)
# Accumulator width of one tensor-core step: the largest j for which a product 2^-j next to a product 1.0 survives
# (test_accumulator_bits_*).  u_acc = 2^-J bounds what each aligned addend loses, relative to the largest.
J_BF16 = 23
J_FP8 = 13
STEP_TERMS = {"bf16": 16 + 1, "fp8": 32 + 1}  # addends of one tensor-core step: the products and the accumulator

DISTS = ("normal", "scaled", "cancel")
# name -> (bias, C: None | "separate" | "alias", alpha of the random inputs, alpha of the exact inputs, beta)
EPILOGUES = {
    "plain": (False, None, 1.0, 1.0, 0.0),
    "bias": (True, None, 1.0, 1.0, 0.0),
    "c_separate": (False, "separate", 1.0, 1.0, 1.0),
    "bias_c_alias": (True, "alias", 0.75, 2.0, -1.0),
    "bias_c_half": (True, "separate", 1.25, 0.5, 0.5),
}
DTYPES = (torch.bfloat16, torch.float32)

# largest err / bar per (entry point, instance), printed at the end of the module
WORST: dict = {}


def K():
    from dolomite_engine_b200 import kernels

    return kernels


@pytest.fixture(scope="module", autouse=True)
def _report():
    from dolomite_engine_b200 import build

    build.build()
    yield
    for (entry, inst, d), r in sorted(WORST.items()):
        print(f"ERRBAR {entry:18s} {inst:28s} D {d}: {r:.3e}")


class _option:
    def __init__(self, key, value):
        self.key, self.value = key, value

    def __enter__(self):
        self.old = K().get_option(self.key)
        K().set_option(self.key, self.value)

    def __exit__(self, *exc):
        K().set_option(self.key, self.old)


def bf(x):
    return x.to(torch.bfloat16)


def _up(n, m):
    return -(-n // m) * m


def _strided(x, fill):
    """x in a buffer whose row stride exceeds its width by at least 8 elements (16-byte aligned rows); the columns
    after x hold `fill` (NaN, or the fp8 NaN bits 0x7f), which the kernels must never read"""
    rows, cols = x.shape
    ld = _up(cols, 16) + 16
    buf = torch.full((rows, ld), fill, dtype=x.dtype, device="cuda")
    buf[:, :cols] = x
    return buf[:, :cols]


def _out_buffer(M, N, dtype):
    """D as a NaN-filled view [M, N] of a buffer with three more rows and 8 more columns than the 16-byte round-up of N"""
    per = 4 if dtype == torch.float32 else 8
    buf = torch.full((M + 3, _up(N, per) + 8), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[:M, :N]


def _check_padding(buf, M, N):
    """the TMA store writes whole 16-byte segments: columns [N, round_up(N, 16 B)) are zero, nothing else is touched"""
    rn = _up(N, 4 if buf.dtype == torch.float32 else 8)
    assert bool((buf[:M, N:rn] == 0).all()), "padding columns of D"
    assert bool(buf[:M, rn:].isnan().all()) and bool(buf[M:].isnan().all()), "D written outside its rows / segments"


def _record(case, got, err, bar):
    ratio = (err / (bar + 1e-30)).max().item()
    key = (case["entry"], case["instance"], "bf16" if got.dtype == torch.bfloat16 else "fp32")
    WORST[key] = max(WORST.get(key, 0.0), ratio)
    return ratio


def _check_bar(case, got, ref, bar, what):
    assert bool(torch.isfinite(got).all()), what
    err = (got.double() - ref).abs()
    ratio = _record(case, got, err, bar)
    assert bool((err <= bar + 1e-30).all()), (what, ratio)


def _acc_bar(kind, steps, mag):
    return STEP_TERMS[kind] * steps * 2.0 ** -(J_BF16 if kind == "bf16" else J_FP8) * mag


def _finish_bar(bar32, ref, dtype):
    return bar32 + (BF16_U * (ref.abs() + bar32) if dtype == torch.bfloat16 else 0.0)


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def _bf16_random(rows, cols, dist, g):
    x = torch.randn(rows, cols, device="cuda", generator=g)
    if dist == "scaled":
        x = x * 2.0 ** torch.randint(-6, 7, (rows, 1), device="cuda", generator=g).float()
    return bf(x)


def _cancel(A, B):
    """even rows of A cancel over the paired columns [0, h) and [h, 2h) of the contraction, rows 1 mod 4 nearly cancel
    (their second half is the negated first one times 1 + 2^-7, rounded to bf16)"""
    h = A.shape[1] // 2
    if h == 0:
        return A, B
    A, B = A.clone(), B.clone()
    B[:, h : 2 * h] = B[:, :h]
    A[::2, h : 2 * h] = -A[::2, :h]
    A[1::4, h : 2 * h] = bf(-A[1::4, :h].float() * (1 + 2.0**-7))
    return A, B


def _halves(shape, g, lim=2):
    return torch.randint(-2 * lim, 2 * lim + 1, shape, device="cuda", generator=g).double() / 2


def _bf16_operands(M, N, Kd, dist, g):
    """A [M, K], B [N, K] in bf16; dist "exact": halves in [-2, 2]"""
    if dist == "exact":
        return bf(_halves((M, Kd), g)), bf(_halves((N, Kd), g))
    A, B = _bf16_random(M, Kd, dist, g), _bf16_random(N, Kd, dist, g)
    return _cancel(A, B) if dist == "cancel" else (A, B)


def _epilogue_inputs(M, N, dtype, dist, g):
    if dist == "exact":
        return bf(_halves((N,), g)), _halves((M, N), g).to(dtype)
    return bf(torch.randn(N, device="cuda", generator=g) * 0.5), torch.randn(M, N, device="cuda", generator=g).to(dtype)


# ---------------------------------------------------------------------------------------------------------------------
# dense bf16 GEMM and split-K
# ---------------------------------------------------------------------------------------------------------------------
def _dense_call(case, a, b, dtype, epi, dist, bias, C, flags=None):
    M, N, _ = case["shape"]
    has_bias, c_mode, alpha_r, alpha_x, beta = EPILOGUES[epi]
    alpha = alpha_x if dist == "exact" else alpha_r
    a_mn, b_mn = case["layout"]
    buf, out = _out_buffer(M, N, dtype)
    c = None
    if c_mode == "alias":
        out.copy_(C)
        c = out
    elif c_mode == "separate":
        c = _strided(C, float("nan"))
    K().gemm(a, b, a_mn=a_mn, b_mn=b_mn, out=out, c=c, alpha=alpha, beta=beta, bias=bias if has_bias else None,
             flags=flags)
    return buf, out, alpha, beta


def _contiguous(x):
    """a copy with row stride = width (x.contiguous() keeps the stride of a one-row view)"""
    return torch.empty(x.shape, dtype=x.dtype, device=x.device).copy_(x)


def _dense_operands(case, A, B):
    a_mn, b_mn = case["layout"]
    return _strided(A.t() if a_mn else A, float("nan")), _strided(B.t() if b_mn else B, float("nan"))


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c["entry"] == "gemm"])
@pytest.mark.parametrize("dist", DISTS + ("exact",))
def test_dense(name, dist):
    case = CASES[name]
    M, N, Kd = case["shape"]
    g = torch.Generator(device="cuda").manual_seed(case["seed"] * 10 + len(dist))
    A, B = _bf16_operands(M, N, Kd, dist, g)
    a, b = _dense_operands(case, A, B)
    exact = A.double() @ B.double().t()
    mag = A.double().abs() @ B.double().abs().t()
    steps = 4 * _up(Kd, 64) // 64
    with _option("gemm_tile_n", case["tile_n"]):
        for dtype in DTYPES:
            bias, C = _epilogue_inputs(M, N, dtype, dist, g)
            first = None
            for epi, (has_bias, c_mode, _, _, _) in EPILOGUES.items():
                buf, out, alpha, beta = _dense_call(case, a, b, dtype, epi, dist, bias, C)
                _check_padding(buf, M, N)
                bd = bias.double() if has_bias else 0.0
                cd = C.double() if c_mode else 0.0
                ref = alpha * (exact + bd) + beta * cd
                if dist == "exact":
                    assert torch.equal(out, ref.to(dtype)), (epi, dtype)
                    continue
                if first is None:
                    first = out.clone()
                mag_out = abs(alpha) * (mag + (bias.double().abs() if has_bias else 0.0)) + abs(beta) * (
                    C.double().abs() if c_mode else 0.0)
                bar32 = abs(alpha) * _acc_bar("bf16", steps, mag) + 3 * U32 * mag_out
                _check_bar(case, out, ref, _finish_bar(bar32, ref, dtype), (epi, dtype))
            if dist == "exact":
                continue
            # two runs give the same bits; so does a contiguous A and B where their rows can be (16-byte aligned)
            again = _dense_call(case, a, b, dtype, "plain", dist, bias, C)[1]
            assert torch.equal(again, first)
            a_mn, b_mn = case["layout"]
            if (M if a_mn else Kd) % 8 == 0 and (N if b_mn else Kd) % 8 == 0:
                ac = _contiguous(A.t() if a_mn else A)
                bc = _contiguous(B.t() if b_mn else B)
                assert torch.equal(_dense_call(case, ac, bc, dtype, "plain", dist, bias, C)[1], first)
            if case["shape"] == HINT_SHAPE:
                with _option("gemm_l2_hints", 0):
                    assert torch.equal(_dense_call(case, a, b, dtype, "plain", dist, bias, C)[1], first)


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c["entry"] == "gemm_splitk"])
@pytest.mark.parametrize("dist", DISTS + ("exact",))
def test_split_k(name, dist):
    """D (fp32) += alpha A B^T with the contraction split over CTAs whose partial tiles are reduce-added"""
    case = CASES[name]
    M, N, Kd = case["shape"]
    g = torch.Generator(device="cuda").manual_seed(case["seed"] * 10 + len(dist))
    A, B = _bf16_operands(M, N, Kd, dist, g)
    a, b = _dense_operands(case, A, B)
    _, C = _epilogue_inputs(M, N, torch.float32, dist, g)
    alpha = 0.5 if dist == "exact" else 0.75
    outs = []
    with _option("gemm_tile_n", case["tile_n"]):
        for _ in range(2):
            buf, out = _out_buffer(M, N, torch.float32)
            out.copy_(C)
            K().gemm(a, b, a_mn=case["layout"][0], b_mn=case["layout"][1], out=out, c=out, alpha=alpha, beta=1.0,
                     flags=K().GEMM_SPLITK_ACCUMULATE)
            _check_padding(buf, M, N)
            outs.append(out)
    ref = alpha * (A.double() @ B.double().t()) + C.double()
    if dist == "exact":
        for out in outs:  # exact partial sums: the order of the reduce-adds no longer matters
            assert torch.equal(out, ref.float())
        return
    mag = A.double().abs() @ B.double().abs().t()
    splits = 16  # at most; each adds one fp32 reduce-add
    bar = abs(alpha) * _acc_bar("bf16", 4 * _up(Kd, 64) // 64, mag) + (2 + splits) * U32 * (abs(alpha) * mag + C.double().abs())
    for out in outs:
        _check_bar(case, out, ref, bar, "split-K")


# ---------------------------------------------------------------------------------------------------------------------
# weight gradients of a block in one launch
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c["entry"] == "wgrad_multi"])
@pytest.mark.parametrize("dist", DISTS + ("exact",))
def test_wgrad_multi(name, dist):
    """dW_q (+)= alpha_q dY_q^T X_q for four problems in one launch; each equals the same problem run alone through
    gemm(a_mn=True, b_mn=True), and the launch gives the same bits with the problems in reverse order"""
    case = CASES[name]
    T = case["K"]
    g = torch.Generator(device="cuda").manual_seed(case["seed"] * 10 + len(dist))
    probs, refs = [], []
    for q, (M, N) in enumerate(case["problems"]):
        dY, X = _bf16_operands(M, N, T, dist, g)  # logical [M, T] and [N, T]; stored [T, M] and [T, N]
        alpha = 2.0 ** (q - 2) if dist == "exact" else 0.75 + 0.5 * q
        acc = q % 2 == 1
        dw0 = _halves((M, N), g).float() if dist == "exact" else torch.randn(M, N, device="cuda", generator=g)
        probs.append((_strided(dY.t(), float("nan")), _strided(X.t(), float("nan")), dw0, alpha, acc))
        refs.append((dY, X))

    def run(order):
        dws = [None] * len(probs)
        for q in order:
            dws[q] = probs[q][2].clone()
        K().gemm_wgrad_multi([(probs[q][0], probs[q][1], dws[q], probs[q][3], probs[q][4]) for q in order])
        return dws

    with _option("gemm_tile_n", case["tile_n"]):
        dws = run(range(len(probs)))
        rev = run(list(reversed(range(len(probs)))))
        for q, (dy, x, dw0, alpha, acc) in enumerate(probs):
            assert torch.equal(rev[q], dws[q]), q
            alone = dw0.clone()
            K().gemm(dy, x, a_mn=True, b_mn=True, out=alone, c=alone if acc else None, alpha=alpha, beta=1.0)
            assert torch.equal(alone, dws[q]), q
    for q, ((dY, X), (_, _, dw0, alpha, acc)) in enumerate(zip(refs, probs)):
        ref = alpha * (dY.double() @ X.double().t()) + (dw0.double() if acc else 0.0)
        if dist == "exact":
            assert torch.equal(dws[q], ref.float()), q
            continue
        mag = dY.double().abs() @ X.double().abs().t()
        bar = abs(alpha) * _acc_bar("bf16", 4 * _up(T, 64) // 64, mag) + 3 * U32 * (
            abs(alpha) * mag + (dw0.double().abs() if acc else 0.0))
        _check_bar(case, dws[q], ref, bar, q)


# ---------------------------------------------------------------------------------------------------------------------
# grouped expert GEMMs
# ---------------------------------------------------------------------------------------------------------------------
def _plan(T, E, k, seed):
    """routing with expert 1 receiving no tokens"""
    # each row a permutation of values 0.25 apart (exact in bf16): no top-k ties
    order = torch.rand(T, E, generator=torch.Generator().manual_seed(seed)).argsort(-1)
    logits = (order - E // 2).float() * 0.25
    logits[:, 1] = -1e4
    logits = bf(logits)
    plan = K().moe_route(logits.cuda(), k)
    counts = torch.bincount(logits.float().topk(k, -1).indices.flatten(), minlength=E)
    assert torch.equal(plan.counts.cpu().long(), counts)
    assert counts[1] == 0
    return plan


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c["entry"] in ("grouped_m", "grouped_m_gather")])
@pytest.mark.parametrize("dist", DISTS + ("exact",))
def test_grouped_m(name, dist):
    """expert forward (w3 [E, N, K]) or dgrad (w3 [E, K, N]) on the rows of each expert, with the per-expert bias row;
    gather-on-load equals the plain launch on the gathered rows"""
    case = CASES[name]
    T, E, k, Kd, N = case["moe"]
    b_mn = case["layout"][1]
    g = torch.Generator(device="cuda").manual_seed(case["seed"] * 10 + len(dist))
    plan = _plan(T, E, k, case["seed"])
    rows = torch.nonzero(plan.slot_of_row >= 0).flatten()
    grp = plan.tile_group[rows // 128].long()
    x, W = _bf16_operands(T, E * N, Kd, dist, g)  # tokens [T, K]; the experts' [N, K] weights stacked
    W = W.view(E, N, Kd)
    alpha = 0.5 if dist == "exact" else 0.75
    bias = _epilogue_inputs(1, E * N, torch.bfloat16, dist, g)[0].view(E, N) if case["bias"] else None
    with _option("gemm_tile_n", case["tile_n"]):
        if case["entry"] == "grouped_m_gather":
            out = K().gemm_grouped_m_gather(x, W, plan, alpha=alpha, bias=bias)
            plain = K().gemm_grouped_m(K().moe_gather(x, plan), W, plan, b_mn=False, alpha=alpha, bias=bias)
            assert torch.equal(out[rows], plain[rows])
            again = K().gemm_grouped_m_gather(x, W, plan, alpha=alpha, bias=bias)
        else:
            xg = K().moe_gather(x, plan)
            w3 = W.transpose(1, 2).contiguous() if b_mn else W
            out = K().gemm_grouped_m(xg, w3, plan, b_mn=b_mn, alpha=alpha, bias=bias)
            again = K().gemm_grouped_m(xg, w3, plan, b_mn=b_mn, alpha=alpha, bias=bias)
    assert torch.equal(out[rows], again[rows])
    xr = x[plan.token_of_row[rows].long()].double()
    exact = torch.zeros(rows.numel(), N, dtype=torch.float64, device="cuda")
    mag = torch.zeros_like(exact)
    for e in range(E):
        sel = grp == e
        exact[sel] = xr[sel] @ W[e].double().t()
        mag[sel] = xr[sel].abs() @ W[e].double().abs().t()
    bd = bias.double()[grp] if bias is not None else 0.0
    ref = alpha * (exact + bd)
    got = out[rows]
    if dist == "exact":
        assert torch.equal(got, ref.to(torch.bfloat16))
        return
    mag_out = abs(alpha) * (mag + (bd.abs() if bias is not None else 0.0))
    bar32 = abs(alpha) * _acc_bar("bf16", 4 * _up(Kd, 64) // 64, mag) + 2 * U32 * mag_out
    _check_bar(case, got, ref, _finish_bar(bar32, ref, torch.bfloat16), "grouped_m")


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c["entry"] == "grouped_k"])
@pytest.mark.parametrize("dist", DISTS + ("exact",))
def test_grouped_k(name, dist):
    """expert weight gradient out3[e] = alpha dY_e^T X_e (+ beta out3[e]) over each expert's rows; the expert without rows
    is written as zeros (overwrite) or keeps its values (accumulate)"""
    case = CASES[name]
    T, E, k, Kd, N = case["moe"]
    beta = case["beta"]
    g = torch.Generator(device="cuda").manual_seed(case["seed"] * 10 + len(dist))
    plan = _plan(T, E, k, case["seed"])
    # an expert whose rows reach the last 64-row k-block of its segment (padded to 256 rows): a tile that dropped its
    # last k-block would differ
    assert any(c % 256 > 192 for c in plan.counts.tolist()), plan.counts
    pad = plan.slot_of_row < 0
    dY, X = _bf16_operands(N, Kd, plan.max_rows, dist, g)  # logical [N, rows], [Kd, rows]: stored [rows, N], [rows, Kd]
    dY, X = dY.t().contiguous(), X.t().contiguous()
    dY[pad] = 0  # padding rows are zero (combine_bwd / gather write zeros there)
    X[pad] = 0
    alpha = 0.5 if dist == "exact" else 0.75
    init = _halves((E, N, Kd), g).float() if dist == "exact" else torch.randn(E, N, Kd, device="cuda", generator=g)
    outs = []
    for _ in range(2):
        out3 = init.clone()
        with _option("gemm_tile_n", case["tile_n"]):
            K().gemm_grouped_k(dY, X, plan, out3, alpha=alpha, beta=beta)
        outs.append(out3)
    assert torch.equal(outs[0], outs[1])
    out3 = outs[0]
    off = plan.offsets.cpu().tolist()
    for e in range(E):
        s0, s1 = off[e], off[e + 1]
        exact = dY[s0:s1].double().t() @ X[s0:s1].double()
        ref = alpha * exact + beta * init[e].double()
        if s1 == s0:
            assert torch.equal(out3[e], init[e] if beta else torch.zeros_like(init[e])), e
            continue
        if dist == "exact":
            assert torch.equal(out3[e], ref.float()), e
            continue
        mag = dY[s0:s1].double().abs().t() @ X[s0:s1].double().abs()
        bar = abs(alpha) * _acc_bar("bf16", 4 * _up(s1 - s0, 64) // 64, mag) + 3 * U32 * (
            abs(alpha) * mag + beta * init[e].double().abs())
        _check_bar(case, out3[e], ref, bar, e)


# ---------------------------------------------------------------------------------------------------------------------
# fp8
# ---------------------------------------------------------------------------------------------------------------------
def _quantize(x, scale, fmt):
    """fp8 bits of x on the device, cast on the CPU (whose conversion keeps the subnormals of both formats)"""
    return quantize_ref(x.cpu(), scale, fmt).cuda()


def _dequantize(q, fmt):
    return dequantize_ref(q.cpu(), fmt).cuda()


def _fp8_operand(rows, cols, fmt, dist, g):
    """-> (fp8 bits [rows, cols], their values, scale_inv).  Random: bf16 values quantised with the delayed-scaling scale
    of their amax; "scaled" rows span 2^+-3; "exact": integers in [-2, 2] with a power-of-two scale_inv."""
    if dist == "exact":
        v = torch.randint(-2, 3, (rows, cols), device="cuda", generator=g).double()
        return _quantize(v, 1.0, fmt), v, 0.5
    x = torch.randn(rows, cols, device="cuda", generator=g)
    if dist == "scaled":
        x = x * 2.0 ** torch.randint(-3, 4, (rows, 1), device="cuda", generator=g).float()
    x = bf(x)
    scale = FP8_MAX[fmt] / x.float().abs().max().item()
    q = _quantize(x, scale, fmt)
    return q, _dequantize(q, fmt), float(torch.tensor(1.0 / scale, dtype=torch.float32))


def _fp8_cancel(qa, qb):
    """the fp8 counterpart of _cancel: even rows of A negated (sign bit) over the second half, B's halves equal"""
    h = qa.shape[1] // 2
    qa, qb = qa.clone(), qb.clone()
    qb[:, h : 2 * h] = qb[:, :h]
    qa[::2, h : 2 * h] = qa[::2, :h] ^ 0x80
    return qa, qb


def _fp8_pair(M, N, Kd, fa, fb, dist, g):
    qa, _, sa = _fp8_operand(M, Kd, fa, dist, g)
    qb, _, sb = _fp8_operand(N, Kd, fb, dist, g)
    if dist == "cancel":
        qa, qb = _fp8_cancel(qa, qb)
    if dist == "exact":
        sa, sb = 4.0, 0.5
    return qa, qb, sa, sb


def _dev_scalar(v):
    return torch.tensor([v], dtype=torch.float32, device="cuda")


def _fp8_steps(case, Kd):
    kb = _up(Kd, 128) // 128
    return 4 * kb + (kb if case["split"] else 0)


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c["entry"] == "gemm_fp8"])
@pytest.mark.parametrize("dist", DISTS + ("exact",))
def test_fp8(name, dist):
    case = CASES[name]
    M, N, Kd = case["shape"]
    fa, fb, split = case["fa"], case["fb"], case["split"]
    g = torch.Generator(device="cuda").manual_seed(case["seed"] * 10 + len(dist))
    qa, qb, sa, sb = _fp8_pair(M, N, Kd, fa, fb, dist, g)
    A, B = _strided(qa, 0x7F), _strided(qb, 0x7F)
    SA, SB = _dev_scalar(sa), _dev_scalar(sb)
    s = sa * sb  # the fp64 product of the fp32 scales
    va, vb = _dequantize(qa, fa), _dequantize(qb, fb)
    exact = s * (va @ vb.t())
    mag = abs(s) * (va.abs() @ vb.abs().t())
    for dtype in DTYPES:
        bias, C = _epilogue_inputs(M, N, dtype, dist, g)
        first = None
        for epi, (has_bias, c_mode, alpha_r, alpha_x, beta) in EPILOGUES.items():
            alpha = alpha_x if dist == "exact" else alpha_r
            buf, out = _out_buffer(M, N, dtype)
            c = None
            if c_mode == "alias":
                out.copy_(C)
                c = out
            elif c_mode == "separate":
                c = _strided(C, float("nan"))
            K().gemm_fp8(A, fa, SA, B, fb, SB, out=out, c=c, alpha=alpha, beta=beta, bias=bias if has_bias else None,
                         split_accumulate=split)
            _check_padding(buf, M, N)
            bd = bias.double() if has_bias else 0.0
            cd = C.double() if c_mode else 0.0
            ref = alpha * (exact + bd) + beta * cd
            if dist == "exact":
                assert torch.equal(out, ref.to(dtype)), (epi, dtype)
                continue
            if first is None:
                first = out.clone()
                again = torch.empty_like(out)
                K().gemm_fp8(A, fa, SA, B, fb, SB, out=again, split_accumulate=split)
                assert torch.equal(again, first)
            mag_out = abs(alpha) * (mag + (bias.double().abs() if has_bias else 0.0)) + abs(beta) * (
                C.double().abs() if c_mode else 0.0)
            # the scale product s = sa * sb is one more fp32 rounding
            bar32 = abs(alpha) * _acc_bar("fp8", _fp8_steps(case, Kd), mag) + 4 * U32 * mag_out
            _check_bar(case, out, ref, _finish_bar(bar32, ref, dtype), (epi, dtype))


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c["entry"] == "fp8_wgrad_multi"])
@pytest.mark.parametrize("dist", DISTS + ("exact",))
def test_fp8_wgrad_multi(name, dist):
    """three fp8 weight gradients in one launch: each equals gemm_fp8 on the same problem alone, bit for bit, and the
    launch gives the same bits with the problems in reverse order"""
    case = CASES[name]
    fa, fb, split, T = case["fa"], case["fb"], case["split"], case["K"]
    g = torch.Generator(device="cuda").manual_seed(case["seed"] * 10 + len(dist))
    probs = []
    for q, (M, N) in enumerate(case["problems"]):
        qa, qb, sa, sb = _fp8_pair(M, N, T, fa, fb, dist, g)
        alpha = 2.0 ** (q - 1) if dist == "exact" else 0.75 + 0.5 * q
        dw0 = _halves((M, N), g).float() if dist == "exact" else torch.randn(M, N, device="cuda", generator=g)
        probs.append((_strided(qa, 0x7F), _dev_scalar(sa), _strided(qb, 0x7F), _dev_scalar(sb), dw0, alpha, q != 1, sa, sb))

    def run(order):
        dws = [None] * len(probs)
        for q in order:
            dws[q] = probs[q][4].clone()
        K().gemm_fp8_wgrad_multi([probs[q][:4] + (dws[q],) + probs[q][5:7] for q in order], dy_fmt=fa, x_fmt=fb,
                                 split_accumulate=split)
        return dws

    dws = run(range(len(probs)))
    rev = run(list(reversed(range(len(probs)))))
    for q, (a, SA, b, SB, dw0, alpha, acc, sa, sb) in enumerate(probs):
        assert torch.equal(rev[q], dws[q]), q
        alone = dw0.clone()
        K().gemm_fp8(a, fa, SA, b, fb, SB, out=alone, c=alone if acc else None, alpha=alpha, beta=1.0,
                     split_accumulate=split)
        assert torch.equal(alone, dws[q]), q
        va, vb = _dequantize(a, fa), _dequantize(b, fb)
        ref = alpha * sa * sb * (va @ vb.t()) + (dw0.double() if acc else 0.0)
        if dist == "exact":
            assert torch.equal(dws[q], ref.float()), q
            continue
        mag = abs(sa * sb) * (va.abs() @ vb.abs().t())
        bar = abs(alpha) * _acc_bar("fp8", _fp8_steps(case, T), mag) + 4 * U32 * (
            abs(alpha) * mag + (dw0.double().abs() if acc else 0.0))
        _check_bar(case, dws[q], ref, bar, q)


# ---------------------------------------------------------------------------------------------------------------------
# accumulator width of one tensor-core step
# ---------------------------------------------------------------------------------------------------------------------
def _survivors(big, got, j_of):
    """j -> whether big * (1 + 2^-j) came out above big; the values must be exactly big or big * (1 + 2^-j)"""
    seen = {}
    for idx, j in j_of.items():
        v = got[idx].item()
        assert v in (big, big * (1 + 2.0**-j)), (j, v)
        seen[j] = v != big
    return seen


def _largest_surviving(seen):
    j = max(j for j, s in seen.items() if s)
    assert all(seen[i] for i in seen if i <= j) and not any(seen[i] for i in seen if i > j), seen
    return j


def test_accumulator_bits_bf16():
    """one k16 step: row j of A is [1, 2^-j, 0, ...], B's row 0 is [1, 1, 0, ...]; D[j, 0] = 1 + 2^-j survives up to
    j = J_BF16, the bar's u_acc = 2^-J_BF16"""
    J = 40
    A = torch.zeros(J + 1, 16)
    A[:, 0] = 1.0
    A[:, 1] = torch.tensor([2.0**-j for j in range(J + 1)])
    B = torch.zeros(8, 16)
    B[0, :2] = 1.0
    D = K().gemm(bf(A).cuda(), bf(B).cuda(), out_dtype=torch.float32)
    j = _largest_surviving(_survivors(1.0, D[:, 0].cpu(), {(r,): r for r in range(J + 1)}))
    print(f"bf16 k16 step: 1 + 2^-j survives up to j = {j}")
    assert j == J_BF16


@pytest.mark.parametrize("split", [False, True])
def test_accumulator_bits_fp8(split):
    """one k32 step of e4m3 operands: a product 2^16 (2^8 * 2^8) next to one product 2^(16 - j), for j = 0 .. 34 (row r of
    A holds 2^8 and 2^(8 - r); B's rows hold 2^8 and 2^-9 or 2^8); the largest surviving j is J_FP8 with split and fast
    accumulation alike"""
    E4M3 = 0
    A = torch.zeros(128, 32, dtype=torch.float64)
    A[:18, 0] = 2.0**8
    A[:18, 1] = torch.tensor([2.0 ** (8 - r) for r in range(18)], dtype=torch.float64)
    B = torch.zeros(16, 32, dtype=torch.float64)
    B[0, 0], B[0, 1], B[1, 0], B[1, 1] = 2.0**8, 2.0**-9, 2.0**8, 2.0**8
    qa, qb = _quantize(A, 1.0, E4M3), _quantize(B, 1.0, E4M3)
    assert torch.equal(dequantize_ref(qa.cpu(), E4M3), A) and torch.equal(dequantize_ref(qb.cpu(), E4M3), B)
    one = _dev_scalar(1.0)
    D = K().gemm_fp8(qa, E4M3, one, qb, E4M3, one, out_dtype=torch.float32, split_accumulate=split).cpu()
    j_of = {(r, 0): 17 + r for r in range(18)}
    j_of.update({(r, 1): r for r in range(18)})
    j = _largest_surviving(_survivors(2.0**16, D, j_of))
    print(f"fp8 k32 step (split={split}): 1 + 2^-j survives up to j = {j}")
    assert j == J_FP8
