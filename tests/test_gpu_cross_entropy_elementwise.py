"""GPU: every instance of the row-resident cross-entropy kernel (ce_act_instances.CE_CASES) element by element against an
fp64 restatement computed from the kernel's own bf16 logits: lse, loss_tok, p and dlogits = (p - onehot) * logit_scale *
grad_scale / n_valid.

The bars follow the kernel's rounding points (csrc/elementwise.cu, ce_rows_kernel): scale2 = logit_scale * log2(e)
rounded to fp32 (the reference uses that fp32 value, so it is no error), the FMA argument x * scale2 - m (one rounding:
2^-24 of |x * scale2| + |m|), ex2.approx.ftz and lg2.approx (the PTX ISA's bounds: 2^-22 relative, flushed below 2^-126;
2^-22 absolute in log2 units), the fp32 sum of the exponentials (8 * NV terms per thread, then 5 shuffle levels, then 8
warps, then SPLIT cluster ranks), and the final rounding (bf16 for dlogits, fp32 for loss_tok).  dlogits must be one of
the bf16 values its fp64 interval admits; loss_tok within its bar.  Invariants are checked with bit equality."""

import math

import numpy as np
import pytest
import torch

from ce_act_instances import CE_CASES, ce_instance, ce_split

pytestmark = pytest.mark.gpu

U = 2.0**-24
EX2_REL = 2.0**-22  # ex2.approx.ftz.f32: maximum relative error (PTX ISA), results below 2^-126 flushed to 0
LG2_ABS = 2.0**-22  # lg2.approx.f32: maximum absolute error in log2 units (PTX ISA)
TINY = 2.0**-126
LOG2E_F32 = float(np.float32(1.4426950408889634))
LN2_F32 = float(np.float32(0.6931471805599453))


def K():
    from dolomite_engine_b200 import kernels

    return kernels


def num_sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def f32(v):
    return float(np.float32(v))


def rn_bf16(v: torch.Tensor) -> torch.Tensor:
    """round-to-nearest-even of fp64 values to bf16 (bf16 subnormals, overflow to inf), exactly"""
    a = v.double().cpu().numpy()
    with np.errstate(invalid="ignore", over="ignore"):
        m, ex = np.frexp(a)
        q = np.ldexp(1.0, np.maximum(ex - 8, -133))
        r = np.round(a / q) * q
        r = np.where(np.abs(r) >= 2.0**128, np.copysign(np.inf, a), r)
        r = np.where(np.isfinite(a), r, a)
    return torch.from_numpy(r)


def nv_of(name: str) -> int:
    return int(name.split("<")[1].split(",")[0])


MARGINS: dict = {}


@pytest.fixture(scope="module", autouse=True)
def _report_margins():
    yield
    for key in sorted(MARGINS):
        print(f"margin {key}: {MARGINS[key]:.3g}")


def _note(key, ratio):
    MARGINS[key] = max(MARGINS.get(key, 0.0), float(ratio))


# ---------------------------------------------------------------------------------------------------------------------
# reference
# ---------------------------------------------------------------------------------------------------------------------
def reference(x, labels, ignore_index, logit_scale, grad_scale, V, n_valid):
    """fp64 (loss_tok, its bar, dlogits lo / hi, valid rows) of the rows of x [T, V] (bf16 values) as the kernel computes
    them; n_valid is the whole call's count of labels != ignore_index"""
    name = ce_instance(V)
    nv, split = nv_of(name), ce_split(V)
    scale2 = f32(f32(logit_scale) * LOG2E_F32)
    xd = x.double()
    valid = labels != ignore_index
    gs = f32(f32(grad_scale) / n_valid) if n_valid else 0.0
    gmul = f32(gs * f32(logit_scale))
    a = xd * scale2  # exact x * scale2 (the max of the fp32-rounded products is the kernel's m)
    m = a.float().double().amax(1, keepdim=True)
    arg = a - m
    terms = torch.exp2(arg)
    s = terms.sum(1, keepdim=True)
    depth = 8 * nv + 5 + 3 + split
    fin = torch.isfinite(xd)
    # the FMA rounds the exact x * scale2 - m once
    e_s = (terms * (math.log(2) * U * torch.where(fin, arg.abs(), torch.zeros_like(a)) + EX2_REL)).sum(1, keepdim=True)
    e_s = e_s + depth * U * s + V * TINY
    lse2 = m + torch.log2(s)  # log2 units, the kernel's m
    e_lse2 = U * lse2.abs() + e_s / (s * math.log(2)) + LG2_ABS
    lab = labels.clamp(0, V - 1).unsqueeze(1)
    xl = a.gather(1, lab)
    loss = (lse2 - xl) * LN2_F32
    e_loss = LN2_F32 * (e_lse2 + U * xl.abs() + U * (lse2 - xl).abs()) + U * loss.abs()
    # dlogits: p = ex2(fma(x, scale2, -lse2)); (p - onehot) * gmul, bf16
    parg = a - lse2
    p = torch.exp2(parg)
    e_arg = e_lse2 + U * (torch.where(fin, parg.abs(), torch.zeros_like(a)) + e_lse2)
    e_p = p * (torch.exp2(e_arg) - 1 + EX2_REL * torch.exp2(e_arg)) + TINY
    onehot = torch.zeros_like(p).scatter_(1, lab, 1.0)
    g = (p - onehot) * gmul
    e_g = (e_p + U * (p - onehot).abs()) * abs(gmul) + U * g.abs()
    lo, hi = g - e_g, g + e_g
    ign = ~valid
    lo[ign], hi[ign] = 0.0, 0.0
    return loss.squeeze(1), e_loss.squeeze(1), lo, hi, valid


def check_rows(x, labels, ignore_index, ls, gs, loss_tok, dl, key, rows=None):
    """per-element checks of the rows `rows` (all by default) of one call's loss_tok / dlogits"""
    V = x.shape[1]
    T = x.shape[0]
    sel = torch.arange(T) if rows is None else torch.as_tensor(rows)
    lab = labels.cpu()
    n_all = int((lab != ignore_index).sum())
    loss, e_loss, lo, hi, valid = reference(x[sel].cpu(), lab[sel], ignore_index, ls, gs, V, n_all)
    lt = loss_tok.cpu().double()[sel]
    assert bool((lt[~valid] == 0).all()), key
    err = (lt - loss).abs()[valid]
    bar = e_loss[valid]
    if err.numel():
        _note("loss_tok/" + key, (err / bar).max())
        assert bool((err <= bar).all()), (key, (err / bar).max().item())
    g = dl.cpu().double()[sel]
    blo, bhi = rn_bf16(lo), rn_bf16(hi)
    ok = (g >= blo) & (g <= bhi)
    if not bool(ok.all()):
        i = tuple(torch.nonzero(~ok)[0].tolist())
        raise AssertionError(f"{key}: {int((~ok).sum())} dlogits outside the admissible bf16 values; first at {i}: "
                             f"{g[i].item()!r} not in [{blo[i].item()!r}, {bhi[i].item()!r}]")
    width = ((hi - lo) / 2 + (rn_bf16(hi) - rn_bf16(lo)).abs() / 2).clamp_min(2.0**-133)
    _note("dlogits/" + key, ((g - (lo + hi) / 2).abs() / (width + (lo + hi).abs() * 2.0**-9)).max())


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
ROW_KINDS = ["normal", "peaked", "dominant", "equal", "masked", "huge"]


def ce_rows(T, V, ls, seed):
    """bf16 [T, V] logits: rows of N(0, 1), N(0, 64), one dominant logit, all equal, -inf entries (a masked vocabulary),
    magnitudes up to |x * logit_scale| ~ 2^29, in turn.  (Above ~2^31 the FMA argument x * scale2 - m of the largest logit
    is its fp32 rounding residual, up to half an ulp of m: past 128 in log2 units, ex2 of it is inf and so is the loss --
    a limit of the kernel's log2-domain FMA, documented in kernels.cross_entropy_fwd_bwd.)"""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(T, V, generator=gen)
    for r in range(T):
        kind = ROW_KINDS[r % len(ROW_KINDS)]
        if kind == "peaked":
            x[r] *= 8
        elif kind == "dominant":
            x[r, int(torch.randint(0, V, (1,), generator=gen))] = 60.0 / ls
        elif kind == "equal":
            x[r] = 1.75
        elif kind == "masked":
            x[r, torch.rand(V, generator=gen) < 0.3] = -math.inf
        elif kind == "huge":
            x[r] = x[r] * torch.exp2(torch.randint(0, 27, (V,), generator=gen).float()) / ls
    return x.bfloat16()


def ce_labels(T, V, ignore_index, seed, x=None):
    """labels at 0, V - 1, the tail vector and the first / last column of each cluster rank's slice; ignored rows single,
    alternating and in runs, the first and the last row included"""
    gen = torch.Generator().manual_seed(seed + 1)
    lab = torch.randint(0, V, (T,), generator=gen)
    split = ce_split(V)
    v8 = (V + 7) // 8
    per = -(-v8 // split)
    special = [0, V - 1, 8 * (v8 - 1), V - 2 if V > 1 else 0]
    for r in range(split):
        special += [min(V - 1, 8 * r * per), min(V, 8 * min(v8, (r + 1) * per)) - 1]
    for i, c in enumerate(special):
        if 1 + 2 * i < T:
            lab[1 + 2 * i] = c
    ign = torch.zeros(T, dtype=torch.bool)
    ign[0] = True
    ign[T - 1] = True
    if T > 40:
        ign[20:30:2] = True  # alternating
        ign[32:38] = True  # a run
    lab[ign] = ignore_index
    if x is not None:  # a label on a masked (-inf) logit would make the loss infinite
        rows = torch.arange(T)
        bad = (~ign) & torch.isinf(x[rows, lab.clamp(0, V - 1)].float())
        x[rows[bad], lab[bad]] = 0.0
    return lab


SCALES = [(1.0, 1.0), (0.625, 1.5), (1 / 16, 2.0**-10)]


def _call(x, labels, ignore_index, ls, gs, ld=None):
    """out-of-place call on a copy of x in rows of `ld` (the dlogits buffer of the same strides is NaN-filled)"""
    T, V = x.shape
    ld = ld or -(-V // 8) * 8
    buf = torch.full((T, ld), math.nan, dtype=torch.bfloat16, device="cuda")
    buf[:, :V] = x.cuda()
    lg = buf[:, :V]
    dbuf = torch.full((T, ld), math.nan, dtype=torch.bfloat16, device="cuda")
    loss, loss_tok, _ = K().cross_entropy_fwd_bwd(lg, labels.cuda(), ignore_index=ignore_index, logit_scale=ls,
                                                  grad_scale=gs, dlogits=dbuf[:, :V])
    return loss, loss_tok, dbuf


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CE_CASES))
def test_every_instance_per_element(name):
    """T = 67 rows of every kind with labels at the slice edges and ignored rows, per element; tail lanes written 0,
    columns past round_up(V, 8) untouched, the mean within its depth bar of the fp64 mean of the kernel's own loss_tok,
    the count exact, in place == out of place, two runs the same bits"""
    k = sorted(CE_CASES).index(name)
    for V in CE_CASES[name][:2]:
        ls, gs = SCALES[(k + V) % len(SCALES)]
        T = 67
        ignore_index = 5 if k % 3 == 0 and V > 5 else -100  # a valid class id as ignore_index
        x = ce_rows(T, V, ls, seed=V)
        labels = ce_labels(T, V, ignore_index, seed=V, x=x)
        v8 = -(-V // 8) * 8
        ld = v8 + 8
        loss, loss_tok, dbuf = _call(x, labels, ignore_index, ls, gs, ld=ld)
        key = f"{name}"
        dl = dbuf[:, :V]
        assert ce_instance(V) == name
        check_rows(x, labels, ignore_index, ls, gs, loss_tok, dl, key)
        # TAIL lanes are written 0, the columns after them keep their NaN fill
        assert bool((dbuf[:, V:v8] == 0).all()), key
        assert bool(dbuf[:, v8:].isnan().all()), key
        # count and mean
        n = int((labels != ignore_index).sum())
        assert K().cross_entropy_count(labels.cuda(), ignore_index)[0].item() == n
        lt = loss_tok.double().cpu()
        depth = -(-T // 1024) + 10
        want = lt.sum() / n
        bar = depth * U * lt.abs().sum() / n + U * abs(want) + 1e-300
        _note("mean/" + key, abs(loss.item() - want) / bar)
        assert abs(loss.item() - want) <= bar
        # in place == out of place; two runs the same bits
        buf = torch.full((T, ld), math.nan, dtype=torch.bfloat16, device="cuda")
        buf[:, :V] = x.cuda()
        loss2, loss_tok2, dl2 = K().cross_entropy_fwd_bwd(buf[:, :V], labels.cuda(), ignore_index=ignore_index,
                                                          logit_scale=ls, grad_scale=gs)
        assert torch.equal(dl2.view(torch.int16), dl.view(torch.int16))
        assert torch.equal(loss_tok2.view(torch.int32), loss_tok.view(torch.int32)) and torch.equal(loss2, loss)
        _, loss_tok3, dbuf3 = _call(x, labels, ignore_index, ls, gs, ld=ld)
        assert torch.equal(dbuf3[:, :v8].view(torch.int16), dbuf[:, :v8].view(torch.int16))
        assert torch.equal(loss_tok3.view(torch.int32), loss_tok.view(torch.int32))


@pytest.mark.parametrize("name", sorted(CE_CASES))
def test_every_instance_many_rows_per_cluster(name):
    """T >= 8 x the clusters of the launch, so the row loop of every SPLIT runs many times (the DSMEM exchange buffer is
    reused with no third cluster barrier): sampled rows per element, and every sampled row == the same row alone (T = 1)"""
    V = CE_CASES[name][0]
    split = ce_split(V)
    clusters = 2 * num_sms() // split
    T = max(8 * clusters + 3, 2200 if split > 1 else 0)
    gen = torch.Generator().manual_seed(V + 7)
    x = (torch.randn(T, V, generator=gen) * 4).bfloat16()
    labels = torch.randint(0, V, (T,), generator=gen)
    labels[::7] = -100
    ls, gs = 0.625, 1.5
    loss, loss_tok, dbuf = _call(x, labels, -100, ls, gs)
    dl = dbuf[:, :V]
    rows = sorted({0, 1, clusters - 1, clusters, clusters + 1, T // 2, T - 2, T - 1} | set(range(3, T, 97)))
    check_rows(x, labels, -100, ls, gs, loss_tok, dl, f"{name}/many", rows=rows)
    n = int((labels != -100).sum())
    g_alone = f32(f32(gs) / n)  # the batch's grad_scale / n_valid: the same fp32 divisor for one row with n_valid = 1
    for r in rows[:: max(1, len(rows) // 8)]:
        if labels[r] == -100:
            continue
        _, lt1, d1 = _call(x[r : r + 1], labels[r : r + 1], -100, ls, g_alone)
        assert torch.equal(lt1.view(torch.int32), loss_tok[r : r + 1].view(torch.int32)), (name, r)
        assert torch.equal(d1[:, :V].view(torch.int16), dl[r : r + 1].view(torch.int16)), (name, r)


@pytest.mark.parametrize("V", [2048, 49152, 65536, 131072])
def test_row_strided_logits_equal_contiguous(V):
    """logits in rows of ld > V give the bits of contiguous logits (single CTA, 24-vector, 2- and 4-CTA clusters)"""
    T = 33
    gen = torch.Generator().manual_seed(V)
    x = (torch.randn(T, V, generator=gen) * 3).bfloat16()
    labels = torch.randint(0, V, (T,), generator=gen)
    labels[4] = -100
    a = K().cross_entropy_fwd_bwd(x.cuda(), labels.cuda(), logit_scale=0.625, grad_scale=1.5)
    buf = torch.zeros(T, V + 64, dtype=torch.bfloat16, device="cuda")
    buf[:, :V] = x.cuda()
    b = K().cross_entropy_fwd_bwd(buf[:, :V], labels.cuda(), logit_scale=0.625, grad_scale=1.5)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))
    assert torch.equal(a[2].view(torch.int16), b[2].contiguous().view(torch.int16))


@pytest.mark.parametrize("V", [2051, 65536, 128259])
def test_all_rows_ignored(V):
    """every row ignored: loss 0, every gradient exactly 0 (tail lanes included), no NaN"""
    T = 9
    x = (torch.randn(T, V) * 3).bfloat16()
    labels = torch.full((T,), -100)
    loss, loss_tok, dbuf = _call(x, labels, -100, 1.0, 1.0)
    v8 = -(-V // 8) * 8
    assert loss.item() == 0.0 and bool((loss_tok == 0).all())
    assert bool((dbuf[:, :v8] == 0).all())


# ---------------------------------------------------------------------------------------------------------------------
# exact case: zero logits at V = 2^k.  m = 0, every term ex2(0) = 1, s = 2^k exactly, lse2 = lg2(2^k) = k, p = ex2(-k) =
# 2^-k: exact if ex2.approx of an integer and lg2.approx of a power of two are exact on the device, which the probe checks
# ---------------------------------------------------------------------------------------------------------------------
def _zero_case(V, T, ls, gs):
    x = torch.zeros(T, V, dtype=torch.bfloat16)
    labels = torch.arange(T) * 13 % V
    return x, labels, _call(x, labels, -100, ls, gs)


def _exact_probe() -> tuple:
    """loss_tok of a zero row at V = 2048 against 11 * ln2 in fp32, and its non-label gradient against 2^-11 exactly"""
    x, labels, (loss, loss_tok, dbuf) = _zero_case(2048, 1, 1.0, 1.0)
    lt = loss_tok[0].item()
    g = dbuf[0, 1].float().item()
    return lt == f32(11.0 * LN2_F32), g == 2.0**-11, (lt, g)


@pytest.fixture(scope="module")
def ex2_lg2_exact():
    a, b, _ = _exact_probe()
    return a and b


def test_probe_ex2_lg2_exact_at_integers_and_powers_of_two():
    """ex2.approx(-11) = 2^-11 and lg2.approx(2048) = 11 exactly (seen through the kernel): the exact case below relies
    on it"""
    a, b, got = _exact_probe()
    assert a and b, got


@pytest.mark.parametrize("V", [2048, 16384, 32768, 65536, 131072])
def test_zero_logits_exact(V, ex2_lg2_exact):
    """p = 2^-k, loss_tok = the kernel's fp32 k * ln2, dlogits = the fp64 value rounded once, bit for bit ((4,1), (8,1),
    (16,1), (16,2), (16,4)); n_valid = 16 (a power of two)"""
    if not ex2_lg2_exact:
        pytest.skip("ex2.approx / lg2.approx are not exact at these arguments (test_probe_ex2_lg2_exact...)")
    k = int(math.log2(V))
    T = 16
    ls, gs = 0.625, 1.5
    x, labels, (loss, loss_tok, dbuf) = _zero_case(V, T, ls, gs)
    assert bool((loss_tok.cpu().double() == f32(k * LN2_F32)).all()), loss_tok[:2].tolist()
    assert loss.item() == f32(k * LN2_F32)
    gmul = f32(f32(f32(gs) / T) * f32(ls))
    p = 2.0**-k
    want = torch.full((T, V), f32(p * gmul), dtype=torch.float64)
    want[torch.arange(T), labels] = f32(f32(p - 1.0) * gmul)
    assert torch.equal(dbuf[:, :V].cpu().double(), rn_bf16(want))
