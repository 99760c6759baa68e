"""GPU: the small kernels of a training step -- norms, RoPE, embedding, reductions and elementwise ops, optimizer, MoE
dispatch -- element by element against plain high-precision restatements (fp64, or fp32 with the rounding points the
kernels document), at every template instance the host can choose (small_kernel_instances.INSTANCES) and at the edges
where such kernels go wrong: row tails, column-tile tails, duplicate ids, strided views, aliasing, odd lengths, special
values.  Bars are per element or per row.  `_le` records the largest error / bar ratio of each check (printed at the
end of the module with -s) so that later changes can see the margin they have."""

import math

import numpy as np
import pytest
import torch

import oracle.dolomite_oracle as O
from small_kernel_instances import INSTANCES, instances_of, rope_threads

pytestmark = pytest.mark.gpu

F32_EPS = 2.0**-24  # unit roundoff of fp32


def K():
    from dolomite_engine_b200 import kernels

    return kernels


def bf(x):
    return x.to(torch.bfloat16)


def num_sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    """one bf16 ulp at |x| (fp64; the smallest normal's ulp for zero and subnormals)"""
    a = x.double().abs().clamp_min(2.0**-126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def _inputs(T, H, dist, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, H, generator=g, dtype=torch.float64)
    if dist == "mean":  # a large common offset: LayerNorm's (x - mean) cancels, RMSNorm's rstd is set by the offset
        x = x + 64.0
    elif dist == "range":  # 2^-12 .. 2^12 within a row: rstd is set by a few large elements
        x = x * torch.exp2(torch.randint(-12, 13, (T, H), generator=g).double())
    w = 1 + 0.25 * torch.randn(H, generator=g, dtype=torch.float64)
    b = 0.5 * torch.randn(H, generator=g, dtype=torch.float64)
    dy = torch.randn(T, H, generator=g, dtype=torch.float64)
    dres = torch.randn(T, H, generator=g, dtype=torch.float64)
    return bf(x), bf(w), bf(b), bf(dy), bf(dres)


MARGINS: dict = {}


def _le(err, bar, key):
    """assert err <= bar element-wise and record the largest err / bar under `key`"""
    err, bar = torch.as_tensor(err).double().cpu(), torch.as_tensor(bar).double().cpu()
    ratio = (err / bar.clamp_min(1e-300)).max().item() if err.numel() else 0.0
    MARGINS[key] = max(MARGINS.get(key, 0.0), ratio)
    ok = err <= bar
    assert ok.all(), (key, ratio, torch.nonzero(~ok)[:4].tolist())


@pytest.fixture(scope="module", autouse=True)
def _report_margins():
    yield
    for key in sorted(MARGINS):
        print(f"margin {key}: {MARGINS[key]:.3g}")


def _assert_rows(got, ref, ulps, what):
    """every element within `ulps` bf16 ulps of its row's largest reference value (a per-row bar: no row or vector of a
    row can be off without failing)"""
    got, ref = got.double().cpu(), ref.double().cpu()
    _le((got - ref).abs(), ulps * bf16_ulp(ref.abs().amax(-1, keepdim=True)), what)


# ------------------------------------------------------------------------------------------------
# RMSNorm
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dist", ["normal", "mean", "range"])
@pytest.mark.parametrize("name", instances_of("rmsnorm_fwd_warp_kernel") + instances_of("rmsnorm_fwd_kernel"))
def test_rmsnorm_fwd_every_instance(name, dist):
    """y = bf16(w * bf16(x * rstd)): bit exact given the kernel's rstd (the rounding points of the reference); rstd within
    16 fp32 ulps of fp64; y within 2 bf16 ulps of the fp64-rstd chain (a rstd ulp can flip bf16(x * rstd)
    at a tie, and w moves that flip by up to two ulps of y)"""
    T, H = INSTANCES[name]
    x, w, _, _, _ = _inputs(T, H, dist, seed=H + T)
    y, rstd = K().rmsnorm_fwd(x.cuda(), w.cuda(), 1e-5)
    x64, w64 = x.double(), w.double()
    r64 = 1.0 / torch.sqrt(x64.pow(2).mean(-1) + 1e-5)
    _le((rstd.double().cpu() - r64).abs(), 16 * F32_EPS * r64, "rmsnorm_fwd/rstd")
    same = bf(w.float() * bf(x.float() * rstd.cpu()[:, None]).float())
    assert torch.equal(y.cpu(), same)
    chain = bf(w64 * bf(x64 * r64[:, None]).double())
    _le((y.double().cpu() - chain.double()).abs(), 2 * bf16_ulp(chain), "rmsnorm_fwd/chain")


def _rms_bwd_ref(x, w, dy, rstd_kernel):
    """fp64 autograd of w * (x * rsqrt(mean(x^2) + eps)) for dx; dw = sum_rows dy * bf16(x * rstd) -- the reference
    rounds the normalised x to bf16 before the weight multiplies it, with the kernel's rstd so that rounding is the same"""
    xr = x.double().requires_grad_(True)
    r = torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + 1e-5)
    (w.double() * (xr * r)).backward(dy.double())
    xn = bf(x.float() * rstd_kernel[:, None]).double()
    return xr.grad, (dy.double() * xn).sum(0), (dy.double() * xn).abs().sum(0)


BWD_SHAPES = sorted({INSTANCES[n] for n in instances_of("rmsnorm_bwd_kernel")} | {(3, 1024), (1700, 2560), (64, 4096)})


@pytest.mark.parametrize("dist", ["normal", "mean", "range"])
@pytest.mark.parametrize("with_add", [False, True])
@pytest.mark.parametrize("T,H", BWD_SHAPES)
def test_rmsnorm_bwd_every_instance(T, H, with_add, dist):
    """dx against fp64 autograd, per row (every element within 2 bf16 ulps of the row's largest value),
    with and without the residual gradient dx_add; dw accumulated onto a non-zero buffer, per column within
    (T / parts + 128) fp32 roundoffs of sum |dy * xn|"""
    x, w, _, dy, dres = _inputs(T, H, dist, seed=3 * H + T)
    xc, wc = x.cuda(), w.cuda()
    _, rstd = K().rmsnorm_fwd(xc, wc, 1e-5)
    dw0 = torch.randn(H, generator=torch.Generator().manual_seed(7))
    dw = dw0.cuda()
    dx = K().rmsnorm_bwd(dy.cuda(), xc, wc, rstd, dw, dx_add=dres.cuda() if with_add else None)
    gx, gw, gw_abs = _rms_bwd_ref(x, w, dy, rstd.cpu())
    ref = gx + dres.double() if with_add else gx
    _assert_rows(dx, ref, 2.0, "rmsnorm_bwd/dx")
    parts = min(T, 6 * num_sms())
    bound = (T / parts + 128) * F32_EPS * (gw_abs + dw0.double().abs()) + 1e-30
    _le((dw.double().cpu() - (dw0.double() + gw)).abs(), bound, "rmsnorm_bwd_every_instance/1")


# ------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dist", ["normal", "mean", "range"])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("name", instances_of("layernorm_fwd_kernel"))
def test_layernorm_fwd_every_instance(name, bias, dist):
    """y = bf16((x - mean) * rstd * w + b), fp32 statistics: mean within 16 fp32 roundoffs of mean |x| and rstd within 16
    of itself against fp64; y within 1 bf16 ulp of the fp64 value computed from the kernel's own statistics (one
    rounding) and within 2 of the all-fp64 chain, each plus 32 fp32 roundoffs of the magnitudes that cancel in
    (x - mean) and in the + b"""
    T, H = INSTANCES[name]
    x, w, b, _, _ = _inputs(T, H, dist, seed=5 * H + T)
    bb = b if bias else None
    y, mean, rstd = K().layernorm_fwd(x.cuda(), w.cuda(), None if bb is None else bb.cuda(), 1e-5)
    x64, w64 = x.double(), w.double()
    m64 = x64.mean(-1, keepdim=True)
    r64 = 1.0 / torch.sqrt((x64 - m64).pow(2).mean(-1, keepdim=True) + 1e-5)
    _le((mean.double().cpu()[:, None] - m64).abs(), 16 * F32_EPS * x64.abs().mean(-1, keepdim=True), "layernorm_fwd_every_instance/1")
    _le((rstd.double().cpu()[:, None] - r64).abs(), 16 * F32_EPS * r64, "layernorm_fwd_every_instance/2")
    b64 = bb.double() if bias else torch.zeros(H, dtype=torch.float64)
    cancel = 32 * F32_EPS * ((x64.abs() + x64.abs().mean(-1, keepdim=True)) * r64 * w64.abs() + b64.abs())
    own = (x64 - mean.double().cpu()[:, None]) * rstd.double().cpu()[:, None] * w64 + b64
    _le((y.double().cpu() - own).abs(), bf16_ulp(own) + cancel, "layernorm_fwd_every_instance/3")
    full = (x64 - m64) * r64 * w64 + b64
    _le((y.double().cpu() - full).abs(), 2 * bf16_ulp(full) + cancel, "layernorm_fwd_every_instance/4")


LN_BWD_SHAPES = sorted({INSTANCES[n] for n in instances_of("layernorm_bwd_kernel")} | {(1, 64), (1500, 2048)})


@pytest.mark.parametrize("dist", ["normal", "mean", "range"])
@pytest.mark.parametrize("with_add", [False, True])
@pytest.mark.parametrize("T,H", LN_BWD_SHAPES)
def test_layernorm_bwd_every_instance(T, H, with_add, dist):
    """dx, dw, db against fp64 autograd of torch.nn.functional.layer_norm: dx per row within 2 bf16 ulps of the row's
    largest value; dw / db accumulated onto non-zero buffers, per column within (T / parts + 144) fp32 roundoffs of
    sum |dy| * (|xhat| + rstd * (|x| + mean |x|) + 1) -- the fp32 (x - mean) enters xhat"""
    x, w, b, dy, dres = _inputs(T, H, dist, seed=7 * H + T)
    xc, wc = x.cuda(), w.cuda()
    _, mean, rstd = K().layernorm_fwd(xc, wc, b.cuda(), 1e-5)
    g = torch.Generator().manual_seed(9)
    dw0, db0 = torch.randn(H, generator=g), torch.randn(H, generator=g)
    dw, db = dw0.cuda(), db0.cuda()
    dx = K().layernorm_bwd(dy.cuda(), xc, wc, mean, rstd, dw, db, dx_add=dres.cuda() if with_add else None)
    xr = x.double().requires_grad_(True)
    wr = w.double().requires_grad_(True)
    br = b.double().requires_grad_(True)
    torch.nn.functional.layer_norm(xr, (H,), wr, br, 1e-5).backward(dy.double())
    ref = xr.grad + dres.double() if with_add else xr.grad
    _assert_rows(dx, ref, 2.0, "layernorm_bwd/dx")
    x64 = x.double()
    r64 = torch.rsqrt(x64.var(-1, unbiased=False, keepdim=True) + 1e-5)
    xhat = (x64 - x64.mean(-1, keepdim=True)) * r64
    parts = min(T, 6 * num_sms())
    mag = (dy.double().abs() * (xhat.abs() + r64 * (x64.abs() + x64.abs().mean(-1, keepdim=True)) + 1)).sum(0)
    bound = (T / parts + 144) * F32_EPS * mag
    _le((dw.double().cpu() - (dw0.double() + wr.grad)).abs(), bound + F32_EPS * dw0.double().abs(), "layernorm_bwd_every_instance/1")
    _le((db.double().cpu() - (db0.double() + br.grad)).abs(), bound + F32_EPS * db0.double().abs(), "layernorm_bwd_every_instance/2")


# ------------------------------------------------------------------------------------------------
# RoPE
# ------------------------------------------------------------------------------------------------
def _rope_case(ng, g, hd, T, n_pos, pos_dtype, tables, seed, pad=0):
    """packed qkv rows [T, ng * (g + 2) * hd] as a view of a buffer `pad` columns wider; positions include 0, n_pos - 1
    and ids past either end (clamped by the kernel)"""
    gen = torch.Generator().manual_seed(seed)
    W = ng * (g + 2) * hd
    buf = bf(torch.randn(T, W + pad, generator=gen))
    if tables == "reference":
        cos, sin = (bf(t) for t in O.rope_tables(hd, n_pos, 10000, bf16=True))
    else:  # halves differ: only the transpose rotation passes the backward check
        cos, sin = bf(torch.randn(n_pos, hd, generator=gen)), bf(torch.randn(n_pos, hd, generator=gen))
    pos = torch.randint(0, n_pos, (T,), generator=gen)
    edge = torch.tensor([0, n_pos - 1, n_pos, n_pos + 7, -3])[: T]
    pos[: edge.numel()] = edge
    return buf, cos, sin, pos.to(torch.int32 if pos_dtype == "int32_t" else torch.int64)


def _rope_ref(buf, cos, sin, pos, ng, g, hd, dy=None):
    """forward: O.apply_rope on the bf16 slots; backward: torch autograd through the same bf16 ops"""
    T = buf.shape[0]
    W = ng * (g + 2) * hd
    p = pos.long().clamp(0, cos.shape[0] - 1)
    c, s = cos[p][:, None, None], sin[p][:, None, None]
    x = buf[:, :W].reshape(T, ng, g + 2, hd)[:, :, : g + 1].clone().requires_grad_(dy is not None)
    y = O.apply_rope(x, c, s, bf16=True)
    if dy is None:
        return y
    y.backward(dy[:, :W].reshape(T, ng, g + 2, hd)[:, :, : g + 1].float())
    return x.grad


def _check_rope(ng, g, hd, T, pos_dtype, tables, pad, seed):
    n_pos = 64
    buf, cos, sin, pos = _rope_case(ng, g, hd, T, n_pos, pos_dtype, tables, seed, pad)
    W = ng * (g + 2) * hd
    cc, sc, pc = cos.cuda(), sin.cuda(), pos.cuda()
    for inverse in (False, True):
        dev = buf.cuda()
        K().rope_qk_inplace(dev[:, :W], ng, g, hd, cc, sc, pc, inverse=inverse)
        out = dev.cpu()
        slots = out[:, :W].reshape(T, ng, g + 2, hd)
        if inverse:
            want = bf(_rope_ref(buf, cos, sin, pos, ng, g, hd, dy=buf))
        else:
            want = bf(_rope_ref(buf, cos, sin, pos, ng, g, hd))
        assert torch.equal(slots[:, :, : g + 1], want), (inverse, (slots[:, :, : g + 1].float() - want.float()).abs().max())
        src = buf[:, :W].reshape(T, ng, g + 2, hd)
        assert torch.equal(slots[:, :, g + 1], src[:, :, g + 1])  # v slots untouched
        assert torch.equal(out[:, W:], buf[:, W:])  # columns past the slots untouched


LAYOUTS = {"mha": (4, 1), "gqa": (2, 4), "mqa": (1, 8)}


@pytest.mark.parametrize("hd", [32, 64, 80, 96, 128, 256])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("tables", ["reference", "random"])
def test_rope_forward_and_backward_bit_exact(layout, hd, tables):
    """forward bit exact with O.apply_rope(bf16=True); backward (inverse=1) bit identical to torch autograd through the
    same bf16 ops -- with the reference's cos/sin tables and with random tables whose halves differ"""
    ng, g = LAYOUTS[layout]
    _check_rope(ng, g, hd, 301, "int64_t", tables, pad=0, seed=hd + ng)


@pytest.mark.parametrize("name", instances_of("rope_kernel"))
def test_rope_every_instance_token_loop_and_strided_rows(name):
    """each instance (position id type x block size) at T below the grid and at T = q * grid + r with r odd and even: the
    blocks then run the two-token loop with and without its one-token tail; rows are a view of a wider buffer"""
    ng, g, hd, pos_dtype = INSTANCES[name]
    grid = num_sms() * (2048 // rope_threads(ng, g, hd))
    for T in (1, 6, 2 * grid + 3, 3 * grid + 2):
        _check_rope(ng, g, hd, T, pos_dtype, "random", pad=24, seed=T)


# ------------------------------------------------------------------------------------------------
# Embedding
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scale", [1.0, 3.5, 0.1])
@pytest.mark.parametrize("H", [8, 2560, 4096])
def test_embedding_fwd_exact(H, scale):
    """scale 1: a bit-exact copy of the row; else bf16(wte * scale) (fp32 product, one rounding); ids clamped to [0, V)"""
    g = torch.Generator().manual_seed(H)
    V = 300
    wte = bf(torch.randn(V, H, generator=g))
    ids = torch.randint(0, V, (517,), generator=g)
    ids[:4] = torch.tensor([0, V - 1, -2, V + 5])
    out = K().embedding_fwd(ids.cuda(), wte.cuda(), scale).cpu()
    rows = wte[ids.clamp(0, V - 1)]
    assert torch.equal(out, rows if scale == 1.0 else bf(rows.float() * scale))


def _embedding_ids(kind, T, V, g):
    if kind == "one_id":
        return torch.full((T,), 5, dtype=torch.int64)
    if kind == "far_duplicates":  # every id repeats 33, 257 and 1000 tokens later
        base = torch.randint(0, V, (T,), generator=g)
        for gap in (33, 257, 1000):
            base[gap::gap + 1] = base[: len(base[gap::gap + 1])]
        return base
    if kind == "large_vocab":
        return torch.randint(0, V, (T,), generator=g)
    ids = torch.randint(0, V, (T,), generator=g)  # "edges": ids 0, V - 1 and out of range
    ids[::97] = 0
    ids[1::89] = V - 1
    ids[2::101] = -1
    ids[3::103] = V + 2
    return ids


@pytest.mark.parametrize("H", [8, 2560, 4096])
@pytest.mark.parametrize("kind,T,V", [("one_id", 3000, 64), ("far_duplicates", 2000, 700), ("large_vocab", 150, 50257),
                                      ("edges", 1200, 500)])
def test_embedding_bwd_vs_fp64_index_add(kind, T, V, H):
    """dwte += scale * index_add(dout) onto a non-zero buffer, with scale = m_emb != 1: per element within (count + 2) fp32
    roundoffs of |dwte0| + scale * sum |dout| of its row (the sum runs in token order, one rounding per add); a second run on the same input is bit identical"""
    g = torch.Generator().manual_seed(T + H)
    scale = 12.0 if kind != "edges" else 1.0
    ids = _embedding_ids(kind, T, V, g).cuda()
    dout = bf(torch.randn(T, H, generator=g)).cuda()
    d0 = torch.randn(V, H, generator=torch.Generator(device="cuda").manual_seed(T), device="cuda")
    runs = []
    for _ in range(2):
        dw = d0.clone()
        K().embedding_bwd(ids, dout, dw, scale)
        runs.append(dw)
    assert torch.equal(runs[0], runs[1])
    # fp64 references on the device (torch's index_add, fp64: its atomics' order does not matter at this precision)
    cid = ids.clamp(0, V - 1)
    ref = d0.double().index_add(0, cid, dout.double() * scale)
    mag = d0.double().abs().index_add(0, cid, dout.double().abs() * scale)
    count = torch.bincount(cid, minlength=V).double()[:, None]
    _le((runs[0].double() - ref).abs(), (count + 2) * F32_EPS * mag, "embedding_bwd_vs_fp64_index_add/1")


# ------------------------------------------------------------------------------------------------
# Column sums, residual adds, scaling, casts
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [8, 248, 256, 264, 10248])
@pytest.mark.parametrize("T", [1, 7, 9, 8192])
def test_colsum_accum_vs_fp64(T, N):
    """out[n] += scale * sum_t x[t, n] (bias gradients): x a view with row stride > N, scale != 1, out non-zero; per column
    within (T + 24) fp32 roundoffs of |out0| + |scale| sum |x|; two runs bit identical"""
    g = torch.Generator(device="cuda").manual_seed(T * 7 + N)
    buf = bf(torch.randn(T, N + 24, device="cuda", generator=g))
    x = buf[:, :N]
    out0 = torch.randn(N, device="cuda", generator=g)
    scale = -0.37
    runs = []
    for _ in range(2):
        out = out0.clone()
        K().colsum_accum(x, out, scale)
        runs.append(out)
    assert torch.equal(runs[0], runs[1])
    ref = out0.double() + scale * x.double().sum(0)
    bound = (T + 24) * F32_EPS * (out0.double().abs() + abs(scale) * x.double().abs().sum(0))
    _le((runs[0].double() - ref).abs(), bound, "colsum_accum_vs_fp64/1")


@pytest.mark.parametrize("n", [8, 1000, 65544])
@pytest.mark.parametrize("alias", ["none", "a", "b"])
def test_add_scaled_bit_exact_and_aliasing(n, alias):
    """out = bf16(a + bf16(alpha * b)) with fp32 arithmetic; out may be a or b"""
    g = torch.Generator().manual_seed(n)
    a, b = bf(torch.randn(n, generator=g)), bf(torch.randn(n, generator=g) * 3)
    alpha = 0.7071
    want = bf(a.float() + bf(torch.tensor(alpha, dtype=torch.float32) * b.float()).float())
    ac, bc = a.cuda(), b.cuda()
    out = {"none": None, "a": ac, "b": bc}[alias]
    got = K().add_scaled(ac, bc, alpha, out=out)
    assert torch.equal(got.cpu(), want)


@pytest.mark.parametrize("s", [1.0, 0.3, -2.0])
def test_scale_by_device_scalar(s):
    """x = bf16(x * s): contiguous, and the rows of a rows_empty buffer (spare columns scaled too, the memory after the
    buffer untouched); s == 1 leaves the buffer bit for bit as it was (NaN and inf included)"""
    g = torch.Generator().manual_seed(1)
    sc = torch.tensor([s], device="cuda")
    x = bf(torch.randn(4104, generator=g))
    x[:3] = torch.tensor([float("nan"), float("inf"), -0.0])
    xc = x.cuda()
    K().scale_by_device_scalar(xc, sc)
    if s == 1.0:
        assert torch.equal(xc.cpu().view(torch.int16), x.view(torch.int16))
    else:  # NaN stays NaN (its payload is the kernel's canonical one)
        got, want = xc.cpu(), bf(x.float() * s)
        assert torch.isnan(got[0]) and torch.equal(got[1:].view(torch.int16), want[1:].view(torch.int16))
    rows, cols = 37, 2053  # the logits of an odd vocabulary: rows of 2056 columns
    big = bf(torch.randn(rows + 1, 2056, generator=g))
    dev = big.cuda()
    view = dev[:rows, :cols]
    assert view.stride(0) == 2056
    K().scale_by_device_scalar(view, sc)
    got = dev.cpu()
    want = big[:rows] if s == 1.0 else bf(big[:rows].float() * s)
    assert torch.equal(got[:rows].view(torch.int16), want.view(torch.int16))
    assert torch.equal(got[rows:].view(torch.int16), big[rows:].view(torch.int16))


def test_cast_f32_to_bf16_special_values():
    """bit exact with torch's round-to-nearest-even at ties, subnormals, +-inf, values near the bf16 maximum (and just
    past it: inf), at an odd length; NaN stays NaN"""
    g = torch.Generator().manual_seed(2)
    bits = torch.randint(-(2**31), 2**31 - 1, (50001,), generator=g, dtype=torch.int64).to(torch.int32)
    bits[::3] = (bits[::3] & ~0xFFFF) | 0x8000  # exact ties, both parities of the kept bit
    x = bits.view(torch.float32).clone()
    special = torch.tensor([0.0, -0.0, 1e-40, -1e-40, 1.4e-45, 2.0**-126, float("inf"), float("-inf"), 3.3895e38,
                            -3.3895e38, 3.39e38, 3.4e38, -3.4e38, 1.0 + 2.0**-8, 1.0 + 3 * 2.0**-8, float("nan")])
    x[: special.numel()] = special
    x = x[:50001]
    d = torch.empty(50001, dtype=torch.bfloat16, device="cuda")
    K().cast_f32_to_bf16(x.cuda(), d)
    got, want = d.cpu(), x.bfloat16()
    nan = torch.isnan(x)
    assert nan.sum() > 100 and torch.isnan(got[nan].float()).all()
    assert torch.equal(got[~nan].view(torch.int16), want[~nan].view(torch.int16))


def test_accum_bf16_into_f32():
    """d += scale * float(s): within one fp32 rounding of each of the product and the sum (fused or not) of fp64"""
    g = torch.Generator().manual_seed(3)
    n = 100_001
    s, d0 = bf(torch.randn(n, generator=g)), torch.randn(n, generator=g)
    for scale in (1.0, 0.125, -3.3):
        d = d0.cuda()
        K().accum_bf16_into_f32(s.cuda(), d, scale)
        prod = float(np.float32(scale)) * s.double()
        ref = d0.double() + prod
        _le((d.double().cpu() - ref).abs(), F32_EPS * (prod.abs() + ref.abs()), "accum_bf16_into_f32/1")


# ------------------------------------------------------------------------------------------------
# Optimizer
# ------------------------------------------------------------------------------------------------
def _adamw64(p, g, m, v, lr, b1, b2, eps, wd, step, cc):
    """the header's formula in fp64: p -= lr / bc1 * m / (sqrt(v) / sqrt(bc2) + eps) after p *= 1 - lr * wd"""
    gi = g * cc
    p = p * (1 - lr * wd)
    m = b1 * m + (1 - b1) * gi
    v = b2 * v + (1 - b2) * gi * gi
    bc1, bc2 = 1 - b1**step, 1 - b2**step
    p = p - lr / bc1 * (m / (torch.sqrt(v) / math.sqrt(bc2) + eps))
    return p, m, v


ADAM_CASES = [  # (bf16 copy, clip coefficient, weight decay, first step)
    (True, 0.37, 0.1, 1),
    (False, None, 0.0, 1),
    (True, None, 0.0, 10**6 - 19),
    (False, 0.9, 0.1, 10**6 - 19),
]


@pytest.mark.parametrize("case", range(len(ADAM_CASES)))
@pytest.mark.parametrize("n", [4096, 4097, 4098, 4099])
def test_adamw_vector_and_scalar_paths(n, case):
    """20 steps against fp64 (per element: p within 20 * 2^-22 * (|p| + 100 lr), m and v within 20 * 2^-22 of the
    element's largest |g| and g^2) and against torch.optim.AdamW on CPU (rtol 1e-5, atol 1e-6); the 16-byte
    vector body (aligned shard) and the scalar path (a [1:] view, as a muP segment slice gives) agree bit for bit, the
    bf16 copy is bf16(p) bit for bit.  n = 0..3 (mod 4) covers the scalar tail of the vector path"""
    with_pb, clip, wd, step0 = ADAM_CASES[case]
    lr, b1, b2, eps = 1e-3, 0.9, 0.95, 1e-8
    gen = torch.Generator().manual_seed(n + case)
    p0 = torch.randn(n, generator=gen)
    grads = [torch.randn(n, generator=gen) * 0.1 * (1 + i % 3) for i in range(20)]
    states = {}
    for path in ("vector", "scalar"):
        off = 0 if path == "vector" else 1
        bufs = [torch.zeros(n + off, device="cuda") for _ in range(4)]
        p, g, m, v = (b[off:] for b in bufs)
        assert (p.data_ptr() % 16 == 0) == (path == "vector")
        p.copy_(p0.cuda())
        pb = torch.empty(n + off, dtype=torch.bfloat16, device="cuda")[off:] if with_pb else None
        coef = torch.tensor([clip], device="cuda") if clip is not None else None
        for i in range(20):
            g.copy_(grads[i].cuda())
            K().adamw_step(p, g, m, v, pb, lr, b1, b2, eps, wd, step0 + i, clip=coef)
        states[path] = (p.cpu(), m.cpu(), v.cpu(), None if pb is None else pb.cpu())
    for a, b in zip(states["vector"], states["scalar"]):
        assert (a is None and b is None) or torch.equal(a, b)
    p, m, v, pb = states["vector"]
    if with_pb:
        assert torch.equal(pb, bf(p))
    cc = 1.0 if clip is None else float(np.float32(clip))
    p64, m64, v64 = p0.double(), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    for i in range(20):
        p64, m64, v64 = _adamw64(p64, grads[i].double(), m64, v64, lr, b1, b2, eps, wd, step0 + i, cc)
    gmax = torch.stack([gr.abs() for gr in grads]).amax(0).double() * cc  # per element
    _le((p.double() - p64).abs(), 20 * 2.0**-22 * (p64.abs() + 100 * lr), "adamw_vector_and_scalar_paths/1")
    _le((m.double() - m64).abs(), 20 * 2.0**-22 * gmax, "adamw_vector_and_scalar_paths/2")
    _le((v.double() - v64).abs(), 20 * 2.0**-22 * gmax**2, "adamw_vector_and_scalar_paths/3")
    pr = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([pr], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
    for i in range(20):
        pr.grad = grads[i] * cc
        if i == 0 and step0 > 1:  # torch counts its own steps: start it where the kernel starts
            opt.state[pr]["step"] = torch.tensor(float(step0 - 1))
            opt.state[pr]["exp_avg"] = torch.zeros(n)
            opt.state[pr]["exp_avg_sq"] = torch.zeros(n)
        opt.step()
    assert torch.allclose(p, pr.data, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("n", [1, 3, 4, 5, 1000, 262145, 1048576 + 7, 3_000_001])
def test_sumsq_accum_vs_fp64_and_bit_identical_runs(n):
    """out[0] += sum(g^2) onto a non-zero out: within (n / 262144 + 64) fp32 roundoffs of the fp64 sum; n past 1024 blocks x 256 threads x 4 leaves partial blocks with empty tails; two runs bit identical"""
    g = torch.randn(n, generator=torch.Generator().manual_seed(n)) * 0.01
    runs = []
    for _ in range(2):
        out = torch.tensor([2.5], device="cuda")
        K().sumsq_accum(g.cuda(), out)
        runs.append(out.cpu())
    assert torch.equal(runs[0], runs[1])
    ref = 2.5 + g.double().pow(2).sum().item()
    _le(torch.tensor(abs(runs[0].item() - ref)), (n / 262144 + 64) * F32_EPS * ref, "sumsq")


@pytest.mark.parametrize("sumsq,max_norm", [(0.25, 1.0), (1.0, 1.0), (16.0, 1.0), (0.0, 1.0), (float("inf"), 1.0),
                                            (float("nan"), 1.0), (16.0, 0.0), (2.0e6, 0.5)])
def test_clip_coef_matches_torch_clamp(sumsq, max_norm):
    """coef = torch.clamp(max_norm / (norm + 1e-6), max=1) bit for bit in fp32 -- NaN for a NaN norm, as the reference's
    clip_grad_norm_ gives (the NaN then reaches every parameter); 1 when clipping is off (max_norm 0)"""
    s = torch.tensor([sumsq], device="cuda")
    coef, norm = torch.empty(1, device="cuda"), torch.empty(1, device="cuda")
    K().clip_coef(s, max_norm, coef, norm)
    n32 = torch.sqrt(torch.tensor(sumsq, dtype=torch.float32))
    want = torch.clamp(torch.tensor(max_norm, dtype=torch.float32) / (n32 + 1e-6), max=1.0) if max_norm > 0 else torch.tensor(1.0)
    assert torch.equal(norm.cpu()[0], n32) or (math.isnan(sumsq) and torch.isnan(norm).all())
    if math.isnan(sumsq):
        assert torch.isnan(coef).all()
    else:
        assert torch.equal(coef.cpu()[0], want), (coef.item(), want.item())


# ------------------------------------------------------------------------------------------------
# MoE dispatch
# ------------------------------------------------------------------------------------------------
def _stable_topk(lf: torch.Tensor, k: int) -> torch.Tensor:
    """torch.topk's order (NaN first, then descending) with ties to the lowest index"""
    a = lf.numpy()
    idx = np.arange(a.shape[1])
    out = np.empty((a.shape[0], k), dtype=np.int64)
    for t in range(a.shape[0]):
        nan = np.isnan(a[t])
        out[t] = np.lexsort((idx, -np.where(nan, 0, a[t]), ~nan))[:k]
    return torch.from_numpy(out)


@pytest.mark.parametrize("k", [1, 2, 8])
@pytest.mark.parametrize("E", [8, 33, 256])
def test_moe_route_ties_infinities_and_nan(E, k):
    """rows of tied logits, rows that must choose -inf logits, rows with NaN (which ranks highest, as in torch.topk):
    every chosen index is a distinct expert in [0, E), in rank order with ties to the lowest index, the value multiset is
    torch.topk's, the histogram is bincount; finite rows' weights are the fp32 softmax of the chosen logits"""
    if k > E:
        pytest.skip("k > E")
    g = torch.Generator().manual_seed(E * 10 + k)
    T = 600
    lf = torch.randint(-3, 4, (T, E), generator=g).float()  # many ties
    lf[T // 2 :] = bf(torch.randn(T - T // 2, E, generator=g)).float()
    lf[0] = float("-inf")  # all -inf
    lf[1] = float("-inf")
    lf[1, E - 1] = 2.0  # one finite logit, the rest -inf
    lf[2, E // 2] = float("nan")
    lf[3] = float("nan")
    lf[4, :: max(1, E // 3)] = float("nan")
    lf[5] = -0.0
    lf[5, ::2] = 0.0
    plan = K().moe_route(bf(lf).cuda(), k)
    sel = plan.sel_idx.cpu().long()
    assert ((sel >= 0) & (sel < E)).all()
    assert all(len(set(r.tolist())) == k for r in sel)
    assert torch.equal(sel, _stable_topk(lf, k))
    got_v = torch.gather(lf, 1, sel).sort(-1).values
    want_v = lf.topk(k, dim=-1).values.sort(-1).values
    assert torch.equal(got_v.isnan(), want_v.isnan()) and torch.equal(got_v[~got_v.isnan()], want_v[~want_v.isnan()])
    assert np.array_equal(plan.counts.cpu().numpy(), np.bincount(sel.reshape(-1).numpy(), minlength=E))
    finite = torch.isfinite(torch.gather(lf, 1, sel)).all(-1)
    w_ref = torch.softmax(torch.gather(lf, 1, sel), dim=-1)
    assert torch.allclose(plan.sel_w.cpu()[finite], w_ref[finite], atol=1e-6)


def _moe_setup(T, E, k, H, seed):
    g = torch.Generator().manual_seed(seed)
    logits = bf(torch.randn(T, E, generator=g))
    plan = K().moe_route(logits.cuda(), k)
    yg = bf(torch.randn(plan.max_rows, H, generator=g))
    return g, plan, yg


MOE_SHAPES = [(T, E, k) for E in (8, 33, 256) for k in (1, 2, 8) for T in (1, 2000) if k <= E]


@pytest.mark.parametrize("T,E,k", MOE_SHAPES)
def test_moe_combine_vs_reference_rounding(T, E, k):
    """out = c + alpha * sum_j bf16(w_j) * Y_g[row_j] with the reference's rounding points (_compute_experts: bf16 gates,
    bf16 products, bf16 index_add; the residual add of the block): bit exact for k <= 2 with and without c; for k = 8 the
    kernel sums in fp32 and rounds once, within one bf16 ulp of the fp64 sum of the products"""
    H = 264  # 33 vectors: lane 0 of each warp does two
    g, plan, yg = _moe_setup(T, E, k, H, seed=T + E + k)
    c = bf(torch.randn(T, H, generator=g))
    rows = plan.row_of_slot.cpu().long().view(T, k)
    gates = bf(plan.sel_w.cpu()).view(T, k, 1)
    prods = bf(yg[rows] * gates)  # [T, k, H]: bf16(y * bf16(w)), one rounding each
    acc = prods[:, 0].float()
    for j in range(1, k):
        acc = acc + prods[:, j].float()
    ycu = yg.cuda()
    plain = K().moe_combine(ycu, plan).cpu()
    if k <= 2:
        assert torch.equal(plain, bf(acc))  # == zeros.index_add(0, batch_index, prods) in bf16
        half = torch.tensor(0.5, dtype=torch.float32)
        assert torch.equal(K().moe_combine(ycu, plan, alpha=0.5).cpu(), bf(half * acc))
    else:
        exact = prods.double().sum(1)
        tol = bf16_ulp(exact) + k * F32_EPS * prods.double().abs().sum(1)
        _le((plain.double() - exact).abs(), tol, "moe_combine_vs_reference_rounding/1")
    alpha = torch.tensor(0.37, dtype=torch.float32)
    res = K().moe_combine(ycu, plan, c=c.cuda(), alpha=0.37).cpu()
    assert torch.equal(res, bf(c.float() + bf(alpha * bf(acc).float()).float()))  # residual + bf16(m * moe_out)


@pytest.mark.parametrize("T,E,k", MOE_SHAPES)
def test_moe_combine_bwd_token_sum_router_bwd(T, E, k):
    """autograd of _compute_experts and of the router softmax: dY_g = bf16(dy * bf16(w)) bit exact (alpha 1) and within
    one bf16 ulp of bf16(bf16(dy * alpha) * bf16(w)) (alpha != 1), padding rows exactly 0; dw = alpha <dy, Y_g> within
    (H / 8 + 8) fp32 roundoffs of the fp64 dot; token sums bit exact for k <= 2, within one bf16 ulp of fp64 for k = 8;
    router dlogits: unselected experts exactly 0, selected within one bf16 ulp of the fp64 softmax backward"""
    H = 264
    g, plan, yg = _moe_setup(T, E, k, H, seed=3 * T + E + k)
    dy = bf(torch.randn(T, H, generator=g))
    ycu, dcu = yg.cuda(), dy.cuda()
    sor = plan.slot_of_row.cpu().long()
    nrows = int(plan.offsets[-1])
    real = sor[:nrows] >= 0
    slots = sor[:nrows][real]
    gate = bf(plan.sel_w.cpu().view(-1))[slots][:, None]
    for alpha in (1.0, 0.37):
        dyg, dw = K().moe_combine_bwd(dcu, ycu, plan, alpha=alpha)
        dyg, dw = dyg.cpu()[:nrows], dw.cpu().view(-1)
        assert torch.all(dyg[~real] == 0)
        tok = dy[slots // k]
        if alpha == 1.0:
            assert torch.equal(dyg[real], bf(tok * gate))
        else:  # the kernel rounds dy * (w * alpha) once, the reference bf16(dy * alpha) first: up to 2 ulps apart
            ref = bf(bf(tok.float() * alpha) * gate)
            _le((dyg[real].double() - ref.double()).abs(), 2 * bf16_ulp(ref), "moe_combine_bwd_token_sum_router_bwd/1")
        terms = tok.double() * yg[:nrows][real].double()
        exact = alpha * terms.sum(-1)
        _le((dw[slots].double() - exact).abs(), (H / 8 + 8) * F32_EPS * alpha * terms.abs().sum(-1), "moe_combine_bwd_token_sum_router_bwd/2")
    # token sums: dx[t] = sum_j dX_g[row_j]
    dxg = bf(torch.randn(plan.max_rows, H, generator=g))
    dx = K().moe_token_sum(dxg.cuda(), plan).cpu()
    parts = dxg[plan.row_of_slot.cpu().long().view(T, k)]
    if k <= 2:
        acc = parts[:, 0].float() + (parts[:, 1].float() if k == 2 else 0)
        assert torch.equal(dx, bf(acc))
    else:
        exact = parts.double().sum(1)
        _le((dx.double() - exact).abs(), bf16_ulp(exact) + k * F32_EPS * parts.double().abs().sum(1), "moe_combine_bwd_token_sum_router_bwd/3")
    # router: softmax-over-selected backward to dense bf16 dlogits
    dws = torch.randn(T, k, generator=g)
    dl = K().moe_router_bwd(plan, dws.cuda()).cpu().double()
    sel = plan.sel_idx.cpu().long()
    w = plan.sel_w.cpu().double()
    want = w * (dws.double() - (w * dws.double()).sum(-1, keepdim=True))
    mask = torch.zeros(T, E, dtype=torch.bool).scatter_(1, sel, True)
    assert torch.all(dl[~mask] == 0)
    got = torch.gather(dl, 1, sel)
    tol = bf16_ulp(want) + 4 * k * F32_EPS * w * (w * dws.double()).abs().sum(-1, keepdim=True)
    _le((got - want).abs(), tol, "moe_combine_bwd_token_sum_router_bwd/4")
