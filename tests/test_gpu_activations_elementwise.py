"""GPU: every instance of the MLP activation kernels (ce_act_instances.ACT_CASES) element by element against an fp64
restatement of its functor, with the rounding points the functors document.

Each functor's fp32 value is bounded by a running error bound (EV below): every fp32 operation of the CUDA expression is
replayed in fp64 and adds its rounding error (half an ulp) or the CUDA Math API's documented ulp bound of the function it
calls, and errors carried in from the operands are propagated through the terms' own magnitudes (so that where a result
cancels -- silu' near -1.278, 1 + erf near -1 -- the bound is that of the terms, not of the small result).  The kernel's
fp32 value therefore lies in [v - e, v + e], and its bf16 output must equal bf16(w) for some w in that interval: the one
correct rounding wherever [v - e, v + e] holds no bf16 rounding midpoint, either neighbour where it does.  GLU's inner
bf16(f(g)) and the eager roundings of Laplace, SoftSign and TanhShrink are rounding points of their own: the admissible
bf16 values there are carried through the (monotone) rest of the expression.

The piecewise-linear functors (relu, relu2, relu6, hardtanh, hardshrink, softshrink) are exact in fp32 for bf16
inputs, plain and GLU, forward and backward: their results must equal the fp64 result rounded once (with GLU's inner
rounding), bit for bit.  MARGINS records the largest error / bar ratio of each check (printed at the end with -s)."""

import math

import numpy as np
import pytest
import torch

import act_oracle
from ce_act_instances import ACT_CASES, ACT_IDS, ACT_NAMES, GLU, PLAIN, SIGMOID_GLU, forms_of

pytestmark = pytest.mark.gpu

U = 2.0**-24  # fp32 unit roundoff: one rounding adds at most U * |result|
TINY = 2.0**-126  # absolute bar for results below the normal range (__expf / ex2.approx.ftz, __fdividef's 0)
F32_MAX = float(np.finfo(np.float32).max)
EXACT = {"relu", "relu2", "relu6", "hardtanh", "hardshrink", "softshrink"}


def K():
    from dolomite_engine_b200 import kernels

    return kernels


def f32(c: float) -> float:
    """the fp32 constant the CUDA source spells as `c` (fp32 literal)"""
    return float(np.float32(c))


# ---------------------------------------------------------------------------------------------------------------------
# bf16 rounding of fp64 values, exactly (round to nearest even, bf16 subnormals, overflow to inf)
# ---------------------------------------------------------------------------------------------------------------------
def rn_bf16(v: torch.Tensor) -> torch.Tensor:
    a = v.double().cpu().numpy()
    with np.errstate(invalid="ignore", over="ignore"):
        m, ex = np.frexp(a)  # a = m * 2^ex, 0.5 <= |m| < 1
        q = np.ldexp(1.0, np.maximum(ex - 8, -133))  # bf16 quantum at |a| (8 significant bits, subnormal quantum 2^-133)
        r = np.round(a / q) * q  # exact in fp64; np.round is round-half-even
        r = np.where(np.abs(r) >= 2.0**128, np.copysign(np.inf, a), r)
        r = np.where(np.isfinite(a), r, a)
    return torch.from_numpy(r)


def f32_of(v: torch.Tensor) -> torch.Tensor:
    """fp32 rounding of fp64 values (exact: one IEEE conversion), back in fp64"""
    return v.float().double()


# ---------------------------------------------------------------------------------------------------------------------
# running error bounds: EV(v, e) is the fp64 value of an fp32 expression and a bound on |fp32 result - v|
# ---------------------------------------------------------------------------------------------------------------------
def _ovf(v, e):
    """an fp32 intermediate past the fp32 range is inf / NaN in the kernel: the bound is void there (e = inf marks it)"""
    return torch.where((v.abs() + e > F32_MAX) | torch.isnan(e), torch.full_like(e, math.inf), e)


class EV:
    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e

    @staticmethod
    def _r(v, e):  # one fp32 rounding of a result whose operands carry an error e
        return EV(v, _ovf(v, e + U * (v.abs() + e)))

    def __add__(a, b):
        b = b if isinstance(b, EV) else EV(torch.full_like(a.v, f32(b)))
        return EV._r(a.v + b.v, a.e + b.e)

    __radd__ = __add__

    def __neg__(a):
        return EV(-a.v, a.e)

    def __sub__(a, b):
        return a + (-(b if isinstance(b, EV) else EV(torch.full_like(a.v, f32(b)))))

    def __rsub__(a, b):
        return (-a) + b

    def __mul__(a, b):
        if not isinstance(b, EV):  # an fp32 constant
            c = f32(b)
            return EV._r(a.v * c, a.e * abs(c))
        return EV._r(a.v * b.v, a.v.abs() * b.e + b.v.abs() * a.e + a.e * b.e)

    __rmul__ = __mul__

    def div(a, b, fast=False):
        """a / b (IEEE, correctly rounded) or __fdividef(a, b) (2 ulp; 0 for 2^126 < |b| < 2^128)"""
        b = b if isinstance(b, EV) else EV(torch.full_like(a.v, f32(b)))
        v = a.v / b.v
        den = (b.v.abs() - b.e).clamp_min(0)
        e = (a.e + v.abs() * b.e) / den
        if not fast:
            return EV._r(v, e)
        e = e + 4 * U * (v.abs() + e)
        big = (b.v.abs() + b.e) > 2.0**126
        return EV(v, _ovf(v, torch.where(big, torch.maximum(e, v.abs() + e), e)))


def _fn(a: EV, f, dmax, ulps):
    """fp32 math function with an `ulps` bound (k ulp <= 2k U |result|) and |f'| <= dmax(lo, hi) on [v - e, v + e]"""
    v = f(a.v)
    e_in = dmax(a.v - a.e, a.v + a.e) * a.e
    e_in = torch.where(a.e > 0, e_in, torch.zeros_like(e_in))
    return EV(v, _ovf(v, e_in + 2 * ulps * U * (v.abs() + e_in)))


def _exp_d(lo, hi):
    return torch.exp(hi)


def _away0(lo, hi):  # smallest |t| on [lo, hi]
    return torch.where((lo <= 0) & (hi >= 0), torch.zeros_like(lo), torch.minimum(lo.abs(), hi.abs()))


def expf(a):  # CUDA Math API: 2 ulp
    return _fn(a, torch.exp, _exp_d, 2)


def expm1f(a):  # 1 ulp
    return _fn(a, torch.expm1, _exp_d, 1)


def erff(a):  # 2 ulp
    return _fn(a, torch.erf, lambda lo, hi: 2 / math.sqrt(math.pi) * torch.exp(-_away0(lo, hi) ** 2), 2)


def tanhf(a):  # 2 ulp
    return _fn(a, torch.tanh, lambda lo, hi: 1 - torch.tanh(_away0(lo, hi)) ** 2, 2)


def log1pf(a):  # 1 ulp
    return _fn(a, torch.log1p, lambda lo, hi: 1 / (1 + lo).clamp_min(1e-300), 1)


def fast_expf(a):
    """__expf: 2 + floor(|1.173 x|) ulp (CUDA Math API), flushed to 0 below 2^-126 (ex2.approx.ftz)"""
    v = torch.exp(a.v)
    e_in = torch.where(a.e > 0, torch.exp(a.v + a.e) * a.e, torch.zeros_like(v))
    ulps = 2 + torch.floor((1.173 * a.v).abs())
    return EV(v, _ovf(v, e_in + 2 * ulps * U * (v.abs() + e_in) + TINY))


def sigmoidf_(x):  # __fdividef(1, 1 + __expf(-x))
    return EV(torch.ones_like(x.v)).div(1.0 + fast_expf(-x), fast=True)


def tanh_fast(z):  # 1 - __fdividef(2, 1 + __expf(2z))
    return 1.0 - EV(torch.full_like(z.v, 2.0)).div(1.0 + fast_expf(2.0 * z), fast=True)


def where(c, a: EV, b: EV) -> EV:
    return EV(torch.where(c, a.v, b.v), torch.where(c, a.e, b.e))


def const(x, c) -> EV:
    return EV(torch.full_like(x.v, f32(c)))


# ---------------------------------------------------------------------------------------------------------------------
# the functors of csrc/elementwise.cu (namespace act), operation by operation.  f returns an EV, or for the functors
# with eager bf16 roundings inside f an interval (lo, hi) of fp32 values computed exactly from the admissible
# intermediate roundings.  x is an EV of the exact bf16 inputs.
# ---------------------------------------------------------------------------------------------------------------------
SELU_S, SELU_AS = 1.0507009873554804934193349852946, 1.0507009873554804934193349852946 * 1.6732632423543772848170429916717
LAPLACE_MU, LAPLACE_DEN = f32(0.70703125), f32(0.282095 * 1.4142135623730951)


def _np32(t):
    return t.double().cpu().numpy().astype(np.float32)


def _iv_bf16(ev: EV):
    """bf16 candidates of one rounding point: [bf16(v - e), bf16(v + e)]"""
    return rn_bf16(ev.v - ev.e), rn_bf16(ev.v + ev.e)


def _elu(s, a_s):
    return (lambda x: where(x.v <= 0, expm1f(x) * a_s, x * s),
            lambda x: where(x.v <= 0, expf(x) * a_s, const(x, s)))


def _gelu_f(x):
    return (x * 0.5) * (1.0 + erff(x * 0.70710678118654752))


def _gelu_d(x):
    return (1.0 + erff(x * 0.70710678118654752)) * 0.5 + (x * 0.39894228040143268) * expf((x * -0.5) * x)


def _gelu_tanh_z(x):
    return (x + ((x * 0.044715) * x) * x) * 0.7978845608028654


def _gelu_tanh_f(x):
    return (x * 0.5) * (1.0 + tanh_fast(_gelu_tanh_z(x)))


def _gelu_tanh_d(x):
    t = tanh_fast(_gelu_tanh_z(x))
    dz = (1.0 + (x * float(np.float32(3) * np.float32(0.044715))) * x) * 0.7978845608028654
    return (1.0 + t) * 0.5 + ((x * 0.5) * (1.0 - t * t)) * dz


def _hardsigmoid_f(x):
    t = x + 3.0
    c = EV(t.v.clamp(0, 6), torch.where((t.v > 0) & (t.v < 6), t.e, torch.zeros_like(t.e)))
    return c.div(6.0)


def _hardswish_f(x):
    t = x + 3.0
    c = EV(t.v.clamp(0, 6), torch.where((t.v > 0) & (t.v < 6), t.e, torch.zeros_like(t.e)))
    return (x * c).div(6.0)


def _laplace_f(x):
    """0.5 * bf16(1 + bf16(erff(bf16(bf16(x - mu) / den))))"""
    xs = _np32(x.v)
    z = _np32(rn_bf16(torch.from_numpy((xs - np.float32(LAPLACE_MU)).astype(np.float64))))
    z = rn_bf16(torch.from_numpy((z / np.float32(LAPLACE_DEN)).astype(np.float64)))
    lo, hi = _iv_bf16(erff(EV(z)))
    post = lambda e: 0.5 * rn_bf16(f32_of(1.0 + e))  # noqa: E731  (1 + e in fp32, then bf16)
    return post(lo), post(hi)


def _laplace_d(x):
    z = (x - 0.707107).div(LAPLACE_DEN)
    return expf((-z) * z) * f32(np.float32(0.56418958354775629) / np.float32(LAPLACE_DEN))


def _logsigmoid_f(x):
    m = EV(x.v.clamp(max=0))
    return m - log1pf(expf(-EV(x.v.abs())))


def _logsigmoid_d(x):
    z = expf(-EV(x.v.abs()))
    q = z.div(1.0 + z)
    return where(x.v < 0, 1.0 - q, q)


def _mish_f(x):
    return x * tanhf(log1pf(expf(x)))


def _mish_d(x):
    t = tanhf(log1pf(expf(x)))
    return t + (x * EV(torch.ones_like(x.v)).div(1.0 + expf(-x))) * (1.0 - t * t)


def _silu_d(x):
    s = sigmoidf_(x)
    return s * (1.0 + x * (1.0 - s))


def _softplus_f(x):
    return where(x.v > 20, x, log1pf(expf(x)))


def _softplus_d(x):
    z = expf(x)
    return where(x.v > 20, const(x, 1.0), z.div(z + 1.0))


def _softsign_f(x):
    """x / bf16(|x| + 1): both fp32 operations correctly rounded, so the fp32 value is known exactly"""
    xs = _np32(x.v)
    d = _np32(rn_bf16(torch.from_numpy((np.abs(xs) + np.float32(1)).astype(np.float64))))
    with np.errstate(invalid="ignore"):
        q = torch.from_numpy((xs / d).astype(np.float64))
    return q, q


def _softsign_d(x):
    a = 1.0 + EV(x.v.abs())
    return EV(torch.ones_like(x.v)).div(a * a)


def _tanhshrink_f(x):
    """x - bf16(tanhf(x)): the fp32 difference of x and each admissible bf16 tanh"""
    lo, hi = _iv_bf16(tanhf(x))
    return f32_of(x.v - hi), f32_of(x.v - lo)


def _tanhshrink_d(x):
    t = tanhf(x)
    return t * t


def _sigmoid_d(x):
    s = sigmoidf_(x)
    return s * (1.0 - s)


def _exact(fn):
    return lambda x: EV(fn(x.v))


FUNCTORS = {  # name -> (f, d); d always returns an EV
    "celu": _elu(1.0, 1.0), "elu": _elu(1.0, 1.0), "selu": _elu(SELU_S, SELU_AS),
    "gelu": (_gelu_f, _gelu_d), "gelu_tanh": (_gelu_tanh_f, _gelu_tanh_d),
    "hardshrink": (_exact(lambda v: torch.where(v.abs() <= 0.5, torch.zeros_like(v), v)),
                   _exact(lambda v: (v.abs() > 0.5).double())),
    "hardsigmoid": (_hardsigmoid_f, lambda x: where((x.v > -3) & (x.v < 3), const(x, np.float32(1) / np.float32(6)),
                                                    const(x, 0.0))),
    "hardswish": (_hardswish_f, lambda x: where(x.v <= -3, const(x, 0.0),
                                                where(x.v < 3, x.div(3.0) + 0.5, const(x, 1.0)))),
    "hardtanh": (_exact(lambda v: v.clamp(-1, 1)), _exact(lambda v: ((v > -1) & (v < 1)).double())),
    "laplace": (_laplace_f, _laplace_d),
    "leaky_relu": (lambda x: where(x.v > 0, x, x * 0.01), lambda x: where(x.v > 0, const(x, 1.0), const(x, 0.01))),
    "log_sigmoid": (_logsigmoid_f, _logsigmoid_d),
    "mish": (_mish_f, _mish_d),
    "relu": (_exact(lambda v: v.clamp_min(0)), _exact(lambda v: (v > 0).double())),
    "relu2": (_exact(lambda v: v.clamp_min(0) ** 2), _exact(lambda v: 2 * v.clamp_min(0))),
    "relu6": (_exact(lambda v: v.clamp(0, 6)), _exact(lambda v: ((v > 0) & (v < 6)).double())),
    "sigmoid": (sigmoidf_, _sigmoid_d),
    "silu": (lambda x: x * sigmoidf_(x), _silu_d),
    "softplus": (_softplus_f, _softplus_d),
    "softshrink": (_exact(lambda v: torch.where(v > 0.5, v - 0.5, torch.where(v < -0.5, v + 0.5, torch.zeros_like(v)))),
                   _exact(lambda v: (v.abs() > 0.5).double())),
    "softsign": (_softsign_f, _softsign_d),
    "tanh": (tanhf, lambda x: 1.0 - tanhf(x) * tanhf(x)),
    "tanhshrink": (_tanhshrink_f, _tanhshrink_d),
}
# the per-functor bound, as the table above builds it: the functions each one calls and their documented bounds
BOUND_SOURCES = {
    "celu/elu/selu": "expm1f 1 ulp (f), expf 2 ulp (f')", "gelu": "erff 2 ulp, expf 2 ulp (f')",
    "gelu_tanh": "__expf 2 + floor(1.173 |2z|) ulp, __fdividef 2 ulp", "laplace": "erff 2 ulp (f), expf 2 ulp (f')",
    "log_sigmoid / mish / softplus": "expf 2 ulp, log1pf 1 ulp, tanhf 2 ulp", "sigmoid / silu": "__expf, __fdividef",
    "tanh / tanhshrink": "tanhf 2 ulp", "hardsigmoid / hardswish / leaky_relu / softsign": "IEEE roundings only",
    "relu / relu2 / relu6 / hardtanh / hardshrink / softshrink": "exact",
}


def _interval(r):
    """(lo, hi) fp64 bounds of an fp32 value from an EV or an interval; below 2^-126 an absolute TINY"""
    lo, hi = (r.v - r.e, r.v + r.e) if isinstance(r, EV) else r
    return lo - TINY * (lo.abs() < TINY), hi + TINY * (hi.abs() < TINY)


def _overflow(r) -> torch.Tensor:
    """elements whose fp64 replay leaves the fp32 range (the bound says nothing there)"""
    lo, hi = _interval(r)
    return ~(torch.isfinite(lo) & torch.isfinite(hi)) | (lo.abs() > F32_MAX) | (hi.abs() > F32_MAX)


def _prod_iv(a, lo, hi):
    """interval of fl32(a * w), w in [lo, hi], a exact"""
    p, q = a * lo, a * hi
    lo2, hi2 = torch.minimum(p, q), torch.maximum(p, q)
    return lo2 - U * lo2.abs(), hi2 + U * hi2.abs()


# ---------------------------------------------------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------------------------------------------------
MARGINS: dict = {}


@pytest.fixture(scope="module", autouse=True)
def _report_margins():
    yield
    for key in sorted(MARGINS):
        print(f"margin {key}: {MARGINS[key]:.3g}")


def _admissible(got, lo, hi, key, skip=None):
    """got (bf16) must lie in [bf16(lo), bf16(hi)]; records err / bar with bar = half the width of that range + half an
    ulp (1.0 means the kernel is at the edge of what its documented error bounds admit)"""
    g = got.double().cpu()
    blo, bhi = rn_bf16(lo), rn_bf16(hi)
    ok = (g >= blo) & (g <= bhi)
    if skip is not None:
        ok |= skip
    mid = (lo + hi) / 2
    with np.errstate(invalid="ignore"):
        _, ex = np.frexp(torch.maximum(lo.abs(), hi.abs()).numpy())
    ulp = torch.from_numpy(np.ldexp(1.0, np.maximum(ex - 8, -133)))
    bar = ((hi - lo) / 2).clamp_min(0) + ulp  # |got - mid| of an admissible bf16 value is below this
    chk = skip if skip is not None else torch.zeros_like(ok)
    r = ((g - mid).abs() / bar)[~chk & torch.isfinite(g)]
    MARGINS[key] = max(MARGINS.get(key, 0.0), r.max().item() if r.numel() else 0.0)
    if not bool(ok.all()):
        i = torch.nonzero(~ok)[0].tolist()
        raise AssertionError(f"{key}: {int((~ok).sum())} elements outside [bf16(lo), bf16(hi)]; first at {i}: got "
                             f"{g[tuple(i)].item()!r}, admissible [{blo[tuple(i)].item()!r}, {bhi[tuple(i)].item()!r}], "
                             f"fp64 interval [{lo[tuple(i)].item()!r}, {hi[tuple(i)].item()!r}]")


def _eq_nan(got, want, key):
    g, w = got.double().cpu(), want.double().cpu()
    ok = (g == w) | (torch.isnan(g) & torch.isnan(w))
    assert bool(ok.all()), (key, torch.nonzero(~ok)[:4].tolist(), g[~ok][:4].tolist(), w[~ok][:4].tolist())


def _torch_ref_fwd(x, act_id, form):
    """torch's own functions on fp64 CPU tensors, rounded once: the values at NaN / inf and where the fp32 replay overflows"""
    return rn_bf16(act_oracle.apply(x.double(), act_id, form, bf16=False)) if form != GLU else None


def fwd_reference(x, act_id, form):
    """(lo, hi) fp64 bounds of y's exact value before its final rounding, and the elements outside the bound's domain"""
    name = ACT_NAMES[act_id]
    f = FUNCTORS[name][0]
    W = x.shape[1]
    if form == PLAIN:
        r = f(EV(x.double()))
        return (*_interval(r), _overflow(r))
    u, g = x[:, : W // 2].double(), x[:, W // 2 :].double()
    r = f(EV(g))
    lo, hi = _interval(r)
    if form == SIGMOID_GLU:  # u * f(g), one rounding
        return (*_prod_iv(u, lo, hi), _overflow(r))
    a_lo, a_hi = rn_bf16(lo), rn_bf16(hi)  # GLU: u * bf16(f(g)), the product exact in fp32
    p, q = u * a_lo, u * a_hi
    return torch.minimum(p, q), torch.maximum(p, q), _overflow(r)


def bwd_reference(dy, x, act_id, form):
    """(lo, hi, overflow) of dx's exact value before its rounding: plain dy * f'(x); GLU [dy * f(g) | (dy * u) * f'(g)]"""
    f, d = FUNCTORS[ACT_NAMES[act_id]]
    dyd = dy.double()
    if form == PLAIN:
        r = d(EV(x.double()))
        return (*_prod_iv(dyd, *_interval(r)), _overflow(r))
    W = x.shape[1]
    u, g = x[:, : W // 2].double(), x[:, W // 2 :].double()
    rf, rd = f(EV(g)), d(EV(g))
    lo1, hi1 = _prod_iv(dyd, *_interval(rf))
    lo2, hi2 = _prod_iv(dyd * u, *_interval(rd))  # dy * u: exact in fp32
    return torch.cat([lo1, lo2], 1), torch.cat([hi1, hi2], 1), torch.cat([_overflow(rf), _overflow(rd)], 1)


# The piecewise-linear functors: every fp32 product of bf16 values here has at most 24 significant bits, so each fp32
# operation is exact (f32_of only turns an overflow into inf, as the kernel's fp32 arithmetic does) and the result is the
# fp64 value rounded once.
def exact_reference_fwd(x, act_id, form):
    f = FUNCTORS[ACT_NAMES[act_id]][0]
    if form == PLAIN:
        return rn_bf16(f32_of(f(EV(x.double())).v))
    W = x.shape[1]
    inner = rn_bf16(f32_of(f(EV(x[:, W // 2 :].double())).v))
    return rn_bf16(f32_of(x[:, : W // 2].double() * inner))


def exact_reference_bwd(dy, x, act_id, form):
    f, d = FUNCTORS[ACT_NAMES[act_id]]
    dyd = dy.double()
    if form == PLAIN:
        return rn_bf16(f32_of(dyd * f32_of(d(EV(x.double())).v)))
    W = x.shape[1]
    u, g = x[:, : W // 2].double(), x[:, W // 2 :].double()
    du = f32_of(dyd * f32_of(f(EV(g)).v))
    dg = f32_of(f32_of(dyd * u) * f32_of(d(EV(g)).v))
    return rn_bf16(torch.cat([du, dg], 1))


def _same_bits(a, b) -> bool:
    return torch.equal(a.contiguous().view(torch.int16 if a.dtype == torch.bfloat16 else torch.int32),
                       b.contiguous().view(torch.int16 if b.dtype == torch.bfloat16 else torch.int32))


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
KINKS = [0.0, 0.5, -0.5, 1.0, -1.0, 3.0, -3.0, 6.0, -6.0, 20.0, 20.125, 0.70703125, -1.278]


def _special_pool():
    vals = []
    for k in KINKS:
        b = torch.tensor([k]).bfloat16()
        vals.append(b.float().item())
        if k == 0:
            vals += [2.0**-133, -(2.0**-133)]  # the two bf16 neighbours of 0: the smallest subnormals
            continue
        bits = b.view(torch.int16)
        for step in (-1, 1):  # the two bf16 neighbours (sign and magnitude: +-1 on the bits of a nonzero value)
            vals.append((bits + step).view(torch.bfloat16).float().item())
    vals += [0.0, -0.0]
    sat = torch.logspace(math.log10(8), 2, 40).tolist()
    huge = torch.logspace(1, math.log10(3e38), 40).tolist()
    vals += sat + [-v for v in sat] + huge + [-v for v in huge]
    return torch.tensor(vals).bfloat16()


def act_inputs(T, F, form, seed, special=0.2):
    """x [T, W]: rows of N(0, s^2) for s in (0.5, 3, 30) in turn, a fraction `special` of the (gate) elements replaced by
    kinks and their neighbours, +-0, saturation (8..100) and huge (10..3e38) magnitudes; GLU up-projections of mixed sign
    and magnitude (2^-8 .. 2^8); dy of mixed magnitude"""
    gen = torch.Generator().manual_seed(seed)
    sig = torch.tensor([0.5, 3.0, 30.0])[torch.arange(T) % 3].unsqueeze(1)
    g = torch.randn(T, F, generator=gen) * sig
    pool = _special_pool()
    pick = torch.rand(T, F, generator=gen) < special
    g = torch.where(pick, pool[torch.randint(0, pool.numel(), (T, F), generator=gen)].float(), g).bfloat16()
    if form == PLAIN:
        x = g
    else:
        u = (torch.randn(T, F, generator=gen) * torch.exp2(torch.randint(-8, 9, (T, F), generator=gen).float())).bfloat16()
        x = torch.cat([u, g], 1)
    dy = (torch.randn(T, F, generator=gen) * torch.exp2(torch.randint(-4, 5, (T, F), generator=gen).float())).bfloat16()
    return x, dy


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------
PAIRS = sorted({(i, f) for i, f, _ in ACT_CASES.values()})


def _pid(p):
    return f"{ACT_NAMES[p[0]]}-{['plain', 'glu', 'sigmoid_glu'][p[1]]}"


def _check_fwd(x, y, act_id, form, key):
    name = ACT_NAMES[act_id]
    if name in EXACT:
        _eq_nan(y, exact_reference_fwd(x, act_id, form), key + "/exact")
        MARGINS[key + "/exact"] = 0.0
        return
    lo, hi, ov = fwd_reference(x, act_id, form)
    if form != GLU and bool(ov.any()):
        # an fp32 intermediate overflows: the kernel must give torch's value there, from its fp32 (bf16 tensor) or its
        # fp64 functions (they differ where torch's own fp32 order overflows)
        g = y.cpu().double()[ov]
        t32 = act_oracle.apply(x.float(), act_id, form, bf16=True).double()[ov]
        t64 = _torch_ref_fwd(x, act_id, form)[ov]
        ok = (g == t32) | (g == t64) | (torch.isnan(g) & (torch.isnan(t32) | torch.isnan(t64)))
        assert bool(ok.all()), (key + "/overflow", g[~ok][:4].tolist(), t32[~ok][:4].tolist(), t64[~ok][:4].tolist())
    _admissible(y, lo, hi, key, skip=ov)


def _check_bwd(dy, x, dx, act_id, form, key):
    name = ACT_NAMES[act_id]
    if name in EXACT:
        _eq_nan(dx, exact_reference_bwd(dy, x, act_id, form), key + "/exact")
        MARGINS[key + "/exact"] = 0.0
        return
    lo, hi, ov = bwd_reference(dy, x, act_id, form)
    _admissible(dx, lo, hi, key, skip=ov)
    return ov


@pytest.mark.parametrize("pair", PAIRS, ids=_pid)
def test_every_instance_forward_backward_and_bias_gradient(pair):
    """act_fwd, act_bwd, act_bwd with the fused bias gradient and act_bwd_segmented of one (id, form) at T = 77,
    F = 328 (41 column vectors: the bias kernel's last column tile is partial), every element against the rounding-aware
    fp64 bounds (bit exact for the piecewise-linear functors); dx with the bias gradient == dx without; dbias against the
    fp64 column sums of the kernel's own dx within the bound of its summation depth; segmented == dense per segment"""
    act_id, form = pair
    T, F = 77, 328
    x, dy = act_inputs(T, F, form, seed=1000 + 3 * act_id + form)
    xc, dyc = x.cuda(), dy.cuda()
    key = _pid(pair)
    y = K().act_fwd(xc, act_id, form)
    _check_fwd(x, y, act_id, form, "fwd/" + key)
    dx = K().act_bwd(dyc, xc, act_id, form)
    ov = _check_bwd(dy, x, dx, act_id, form, "bwd/" + key)
    if ov is not None and bool(ov.any()):
        MARGINS["bwd_overflow_elements/" + key] = float(ov.sum())
    _check_bias(dyc, xc, dx, act_id, form, key)
    _check_segmented(dyc, xc, dx, act_id, form, key)


def _colsum_bar(dxd, db0, T):
    """fp32 sums in the bias kernel: each thread adds ceil(rows_per_split / 8) rows, then 8 row lanes, then the 8 row
    splits of the cluster, then the buffer's prior contents: a chain of at most that many additions"""
    rps = -(-T // 8)
    depth = -(-rps // 8) + 8 + 8 + 1
    return depth * U * (dxd.abs().sum(0) + db0.abs()) + 1e-300


def _check_bias(dyc, xc, dx, act_id, form, key):
    W = xc.shape[1]
    db0 = torch.randn(W, generator=torch.Generator().manual_seed(3)).cuda()
    db = db0.clone()
    dxf = K().act_bwd(dyc, xc, act_id, form, bias_grad_accum=db)
    assert _same_bits(dxf, dx)
    dxd = dx.double().cpu()
    # columns with an inf / NaN dx, or whose fp32 partial sums can leave the fp32 range (huge inputs), are not compared
    fin = torch.isfinite(dxd).all(0) & (dxd.abs().sum(0) + db0.double().cpu().abs() < 2.0**120)
    want = db0.double().cpu() + dxd.sum(0)
    err = (db.double().cpu() - want).abs()
    bar = _colsum_bar(dxd, db0.double().cpu(), xc.shape[0])
    r = (err / bar)[fin]
    MARGINS["dbias/" + key] = max(MARGINS.get("dbias/" + key, 0.0), r.max().item() if r.numel() else 0.0)
    assert bool((err[fin] <= bar[fin]).all()), (key, r.max().item())
    db2 = db0.clone()
    assert _same_bits(K().act_bwd(dyc, xc, act_id, form, bias_grad_accum=db2), dx)
    assert _same_bits(db2, db)  # two runs: the same bits


def _check_segmented(dyc, xc, dx, act_id, form, key):
    """segments with empty ones among them (first, middle, last), each against the dense launch on its own rows"""
    T, W = xc.shape
    cuts = [0, 0, 5, 5, 40, T, T]
    seg = torch.tensor(cuts, dtype=torch.int32).cuda()
    S = len(cuts) - 1
    db0 = torch.randn(S, W, generator=torch.Generator().manual_seed(4)).cuda()
    db = db0.clone()
    dxs = K().act_bwd_segmented(dyc, xc, act_id, form, seg, db)
    assert _same_bits(dxs, dx)
    for s in range(S):
        a, b = cuts[s], cuts[s + 1]
        ref = db0[s].clone()
        if b > a:
            K().act_bwd(dyc[a:b].contiguous(), xc[a:b].contiguous(), act_id, form, bias_grad_accum=ref)
        assert _same_bits(db[s], ref), (key, s)


SHAPES = [(T, F) for T in (1, 7, 77, 2003) for F in (8, 328, 4104)]


@pytest.mark.parametrize("T,F", SHAPES)
@pytest.mark.parametrize("name,form", [("relu2", GLU), ("silu", GLU), ("gelu", PLAIN)])
def test_shapes_grid_stride_and_row_splits(name, form, T, F):
    """the shapes where the index arithmetic goes wrong: one row, row counts that do not divide over the 8 row splits,
    a partial 32-vector column tile (F = 328), a single vector (F = 8), and enough rows for the grid-stride loop to wrap"""
    act_id = ACT_IDS[name]
    x, dy = act_inputs(T, F, form, seed=T * 31 + F, special=0.05)
    xc, dyc = x.cuda(), dy.cuda()
    key = f"shapes/{name}"
    _check_fwd(x, K().act_fwd(xc, act_id, form), act_id, form, "fwd/" + key)
    dx = K().act_bwd(dyc, xc, act_id, form)
    _check_bwd(dy, x, dx, act_id, form, "bwd/" + key)
    _check_bias(dyc, xc, dx, act_id, form, key)


def test_sigma_sweep_normal_inputs():
    """N(0, s^2) inputs for s in (0.5, 3, 30) without special values: the bulk of a real MLP's pre-activations"""
    for act_id in range(len(ACT_NAMES)):
        for form in forms_of(act_id):
            x, dy = act_inputs(64, 256, form, seed=77 + act_id, special=0.0)
            _check_fwd(x, K().act_fwd(x.cuda(), act_id, form), act_id, form, "fwd/normal")
            _check_bwd(dy, x, K().act_bwd(dy.cuda(), x.cuda(), act_id, form), act_id, form, "bwd/normal")


NONFINITE = [math.nan, math.inf, -math.inf]


@pytest.mark.parametrize("form", [PLAIN, GLU, SIGMOID_GLU])
def test_nan_and_inf_forward_match_torch(form):
    """NaN in gives NaN out for every activation (plain and GLU, with u = 1.5), and the values at +-inf are torch's"""
    ids = range(len(ACT_NAMES)) if form != SIGMOID_GLU else [ACT_IDS["sigmoid"]]
    for act_id in ids:
        g = torch.tensor(NONFINITE * 8).bfloat16().reshape(1, 24)[:, :16].repeat(2, 1)
        x = g if form == PLAIN else torch.cat([torch.full_like(g, 1.5), g], 1)
        y = K().act_fwd(x.cuda(), act_id, form).cpu()
        if form == GLU:
            want = rn_bf16(1.5 * rn_bf16(act_oracle.base(g.double(), act_id)))
        else:
            want = _torch_ref_fwd(x, act_id, form)
        _eq_nan(y, want, f"nonfinite/{ACT_NAMES[act_id]}/{form}")
        assert bool(torch.isnan(y[:, 0::3]).all()), ACT_NAMES[act_id]


# dx at x = NaN, +inf, -inf with dy = 1 (plain form), as the kernels compute it; where torch autograd differs (DESIGN.md)
# the entry says so.  None: NaN.
BWD_NONFINITE = {
    "celu": (1.0, 1.0, 0.0), "elu": (1.0, 1.0, 0.0), "selu": (1.046875, 1.046875, 0.0), "gelu": (None, None, None),
    "gelu_tanh": (None, None, None), "hardshrink": (1.0, 1.0, 1.0), "hardsigmoid": (0.0, 0.0, 0.0),
    "hardswish": (1.0, 1.0, 0.0), "hardtanh": (0.0, 0.0, 0.0), "laplace": (None, 0.0, 0.0),
    "leaky_relu": (0.010009765625, 1.0, 0.010009765625), "log_sigmoid": (None, 0.0, 1.0), "mish": (None, None, None),
    "relu": (0.0, 1.0, 0.0), "relu2": (0.0, math.inf, 0.0), "relu6": (0.0, 0.0, 0.0), "sigmoid": (None, 0.0, 0.0),
    "silu": (None, None, None), "softplus": (None, 1.0, 0.0), "softshrink": (1.0, 1.0, 1.0),
    "softsign": (None, 0.0, 0.0), "tanh": (None, 0.0, 0.0), "tanhshrink": (None, 1.0, 1.0),
}


def test_backward_at_nan_and_inf_is_pinned():
    """the backward kernels' values at non-finite x (dy = 1), pinned so that a change is seen"""
    x = torch.tensor(NONFINITE * 8).bfloat16().reshape(3, 8)
    got = {}
    for act_id, name in enumerate(ACT_NAMES):
        dx = K().act_bwd(torch.ones(3, 8).bfloat16().cuda(), x.cuda(), act_id, PLAIN).cpu().double()
        got[name] = tuple(None if math.isnan(v) else v for v in dx[0, :3].tolist())
    assert got == BWD_NONFINITE, repr({k: v for k, v in got.items() if BWD_NONFINITE.get(k) != v})
