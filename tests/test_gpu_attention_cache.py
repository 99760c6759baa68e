"""GPU: every instance of the KV-cache attention kernel (csrc/attention_cache.cu) against a plain fp64 reference, element by
element, and its exact properties.

Per-element bars, with the terms of test_gpu_attention_elementwise.py.  For new token i of sequence b (past cached tokens),
the keys are cache positions 0 .. past + i, n_t = past + i + 1 of them, b_k the bf16 ALiBi bias of position k:

    S = scale * q K^T + b    P = softmax(S)    O = P V
    out:  (u + 2 e_t + 2 rho_t) sum_k P_tk |V_kd| + u |O_td|,   e_t = eps_t + sig_t,   rho_t = (n_t + 8) 2^-23

u is the bf16 rounding of P before P.V and of the output, eps_t the exp2 error, sig_t the fp32 tensor-core score and rho_t
the fp32 row sum and accumulator.  Cache positions past the new tokens hold NaN in every per-element case.
"""

import math

import pytest
import torch

import alibi_oracle as A
from attention_cache_instances import CASES
from dolomite_engine_b200.alibi import alibi_slopes

pytestmark = pytest.mark.gpu

U = 2.0**-8
ACC = 2.0**-23
EXP = 2.0**-22
LOG2E = 1.0 / math.log(2.0)
DEV = "cuda"


def K():
    from dolomite_engine_b200 import kernels

    return kernels


def _scale(c) -> float:
    return 1.0 / math.sqrt(c["hd"]) if c["scale"] == "rsqrt" else 1.0 / c["hd"]


def _inputs(c, fill=float("nan"), extra_rows: int = 0):
    """qkv [sum n + extra_rows, ...], cu_new, past, k / v caches [B, L_max, ng * hd] with `fill` past each sequence's
    new tokens; L_max is not a multiple of 64"""
    ng, g, hd, past, n = c["ng"], c["g"], c["hd"], c["past"], c["n"]
    gen = torch.Generator().manual_seed(c["seed"])
    B, T = len(past), sum(n)
    L_max = max(p + m for p, m in zip(past, n)) + 37
    x = torch.randn(T + extra_rows, ng, g + 2, hd, generator=gen, dtype=torch.float64)
    if c["dist"] == "peaked":
        x[:, :, :g] *= 4
    elif c["dist"] == "flat":
        x[:, :, :g] = 0
    kc = torch.randn(B, L_max, ng * hd, generator=gen).bfloat16()
    vc = torch.randn(B, L_max, ng * hd, generator=gen).bfloat16()
    for b in range(B):
        kc[b, past[b] + n[b]:] = fill
        vc[b, past[b] + n[b]:] = fill
    cu = torch.tensor([0] + list(torch.tensor(n).cumsum(0).tolist()), dtype=torch.int32)
    return (x.reshape(T + extra_rows, -1).bfloat16().to(DEV), cu.to(DEV), torch.tensor(past, dtype=torch.int32, device=DEV),
            kc.to(DEV), vc.to(DEV))


def _run(c, qkv, cu, past, kc, vc, slopes, out=None):
    return K().attn_cache(qkv, cu, past, kc, vc, c["ng"], c["g"], c["hd"], _scale(c), out=out, alibi_slopes=slopes)


def _slopes(c):
    return alibi_slopes(c["ng"] * c["g"]).to(DEV) if c["alibi"] else None


@pytest.mark.parametrize("name", sorted(CASES))
def test_attention_cache_per_element_vs_fp64(name):
    c = CASES[name]
    ng, g, hd, scale = c["ng"], c["g"], c["hd"], _scale(c)
    qkv, cu, past, kc, vc = _inputs(c)
    slopes = _slopes(c)
    out = _run(c, qkv, cu, past, kc, vc, slopes)
    T = qkv.shape[0]
    got = out.view(T, ng, g, hd)
    x = qkv.double().view(T, ng, g + 2, hd)
    L_max = kc.shape[1]
    bias = A.alibi_bias(slopes.cpu(), torch.arange(L_max).unsqueeze(0), True)[0].double().to(DEV) if slopes is not None else None
    worst = 0.0
    cu_h = cu.tolist()
    for b, (p, n) in enumerate(zip(c["past"], c["n"])):
        if n == 0:
            continue
        s, L = cu_h[b], p + n
        kk = kc[b, :L].double().view(L, ng, hd)
        vv = vc[b, :L].double().view(L, ng, hd)
        allowed = torch.arange(L, device=DEV)[None, :] <= (p + torch.arange(n, device=DEV))[:, None]  # [n, L]
        n_t = (p + torch.arange(n, device=DEV) + 1).double()
        for gi in range(ng):
            for j in range(g):
                h = gi * g + j
                Q = x[s:s + n, gi, j]
                raw = Q @ kk[:, gi].T
                bb = bias[h, :L] if bias is not None else torch.zeros(L, dtype=torch.float64, device=DEV)
                S = (scale * raw + bb).masked_fill(~allowed, -math.inf)
                P = torch.softmax(S, -1)
                Oref = P @ vv[:, gi]
                lam = LOG2E * (scale * raw.abs() + bb.abs()).masked_fill(~allowed, 0).amax(-1)
                sig = (scale * hd * ACC * (Q.abs() @ kk[:, gi].abs().T)).masked_fill(~allowed, 0).amax(-1)
                e_t = EXP * (1 + lam) + sig
                rho = (n_t + 8) * ACC
                bar = ((U + 2 * e_t + 2 * rho)[:, None] * P) @ vv[:, gi].abs() + U * Oref.abs()
                err = (got[s:s + n, gi, j].double() - Oref).abs()
                worst = max(worst, (err / bar.clamp_min(1e-300)).max().item())
    print(f"\nmax err/bar {name}: out={worst:.3g}")
    assert worst <= 1.0


# ------------------------------------------------------------------------------------------------
# exact properties (torch.equal)
# ------------------------------------------------------------------------------------------------
def _case(hd, alibi, ng=2, g=3, past=(0, 65, 700, 1, 128), n=(130, 17, 64, 0, 2), seed=11, dist="normal"):
    return dict(hd=hd, alibi=alibi, ng=ng, g=g, scale="rsqrt", dist=dist, past=list(past), n=list(n), seed=seed)


SPLIT_GRID = [(64, False, 2, 3), (80, True, 1, 7), (128, False, 8, 1), (256, True, 1, 16), (16, False, 3, 2), (160, True, 2, 5)]


@pytest.mark.parametrize("hd,alibi,ng,g", SPLIT_GRID)
def test_split_across_calls_gives_the_same_bits(hd, alibi, ng, g):
    """the new tokens of every sequence in one call, or over four calls of 17, 1, 64 and the rest (a call whose counts are
    all 1 runs attn_cache too); the cache holds the keys / values of every new token from the start"""
    c = _case(hd, alibi, ng, g, past=(0, 65, 700, 1), n=(130, 90, 83, 82))
    qkv, cu, past, kc, vc = _inputs(c, fill=0.0)
    slopes = _slopes(c)
    whole = _run(c, qkv, cu, past, kc, vc, slopes)
    cu_h = cu.tolist()
    done = [0] * len(c["n"])
    for chunk in (17, 1, 64, None):
        take = [m - d if chunk is None else min(chunk, m - d) for m, d in zip(c["n"], done)]
        rows = torch.cat([torch.arange(cu_h[b] + done[b], cu_h[b] + done[b] + t) for b, t in enumerate(take)]).to(DEV)
        cu_c = torch.tensor([0] + torch.tensor(take).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
        past_c = past + torch.tensor(done, dtype=torch.int32, device=DEV)
        part = _run(c, qkv[rows].contiguous(), cu_c, past_c, kc, vc, slopes)
        assert torch.equal(part, whole[rows]), chunk
        done = [d + t for d, t in zip(done, take)]


@pytest.mark.parametrize("hd,alibi", [(64, False), (96, True), (192, False), (256, True)])
def test_other_sequences_do_not_change_a_sequence(hd, alibi):
    """scaling the caches and queries of every other sequence by 64 leaves a sequence's output bits as they are"""
    c = _case(hd, alibi)
    qkv, cu, past, kc, vc = _inputs(c, fill=0.0)
    slopes = _slopes(c)
    ref = _run(c, qkv, cu, past, kc, vc, slopes)
    cu_h = cu.tolist()
    for b in range(len(c["n"])):
        q2, k2, v2 = qkv.clone() * 64, kc.clone() * 64, vc.clone() * 64
        q2[cu_h[b]:cu_h[b + 1]] = qkv[cu_h[b]:cu_h[b + 1]]
        k2[b], v2[b] = kc[b], vc[b]
        got = _run(c, q2, cu, past, k2, v2, slopes)
        assert torch.equal(got[cu_h[b]:cu_h[b + 1]], ref[cu_h[b]:cu_h[b + 1]]), b


@pytest.mark.parametrize("hd,alibi", [(32, True), (80, False), (128, True), (160, False), (256, False)])
def test_cache_positions_past_the_new_tokens_change_nothing(hd, alibi):
    c = _case(hd, alibi)
    slopes = _slopes(c)
    zero = _run(c, *_inputs(c, fill=0.0), slopes)
    nan = _run(c, *_inputs(c, fill=float("nan")), slopes)
    big = _run(c, *_inputs(c, fill=1e30), slopes)
    assert torch.equal(nan, zero) and torch.equal(big, zero)


@pytest.mark.parametrize("hd,alibi", [(16, False), (64, True), (192, True), (256, False)])
def test_every_real_row_is_written_and_nothing_else(hd, alibi):
    """a NaN-filled out is overwritten on the rows of the new tokens; rows past them (qkv rows of no sequence) and the
    sequences with n = 0 write nothing"""
    c = _case(hd, alibi, n=(130, 0, 64, 0, 3))
    qkv, cu, past, kc, vc = _inputs(c, extra_rows=5)
    out = torch.full((qkv.shape[0], c["ng"] * c["g"] * hd), float("nan"), dtype=torch.bfloat16, device=DEV)
    _run(c, qkv, cu, past, kc, vc, _slopes(c), out=out)
    T = sum(c["n"])
    assert not out[:T].isnan().any()
    assert out[T:].isnan().all()
