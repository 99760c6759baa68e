"""GPU: every wide-head attention kernel instance (head_dim 160, 192, 256; csrc/attention_wide.cu) against a plain fp64
reference, element by element, and exact properties.

The reference and the per-element running-error bars are those of test_gpu_attention_elementwise.py (its module docstring
derives them): the wide kernels have the same rounding points -- fp32 tensor-core scores, one ex2.approx per probability,
bf16 P before P.V and dV, fp32 P and dP in dS, bf16 dS before dK and dQ, fp32 accumulators, one bf16 rounding per output.
Each test prints max(err / bar) per output.
"""

import numpy as np
import pytest
import torch

from attention_wide_instances import DECODE_CASES, FWD_BWD_CASES, HEAD_DIMS
from dolomite_engine_b200.alibi import alibi_slopes
from test_gpu_attention_elementwise import (ACC, DEV, EXP, K, LOG2E, U, _bias, _inputs, _ratio, _reference, _run,
                                            _scale)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(FWD_BWD_CASES))
def test_wide_attention_fwd_bwd_per_element_vs_fp64(name):
    c = FWD_BWD_CASES[name]
    ng, g, hd = c["ng"], c["g"], c["hd"]
    qkv, dout, cu = _inputs(c)
    slopes = alibi_slopes(ng * g).to(DEV) if c["alibi"] else None
    out, lse, dqkv = _run(c, slopes, qkv, dout, cu)
    T = qkv.shape[0]
    r = _reference(c, qkv, dout, out, lse, cu, slopes, backward=True)
    d = dqkv.view(T, ng, g + 2, hd)
    ratios = {
        "lse": _ratio(lse, r["lse"], r["lse_bar"]),
        "out": _ratio(out.view(T, ng, g, hd), r["out"], r["out_bar"]),
        "dq": _ratio(d[:, :, :g], r["dq"], r["dq_bar"]),
        "dk": _ratio(d[:, :, g], r["dk"], r["dk_bar"]),
        "dv": _ratio(d[:, :, g + 1], r["dv"], r["dv_bar"]),
    }
    print(f"\nmax err/bar {name}: " + " ".join(f"{k}={v:.3g}" for k, v in ratios.items()))
    for k, v in ratios.items():
        assert v <= 1.0, (k, ratios)


@pytest.mark.parametrize("name", sorted(DECODE_CASES))
def test_wide_attention_decode_per_element_vs_fp64(name):
    c = DECODE_CASES[name]
    ng, g, hd, lens = c["ng"], c["g"], c["hd"], c["lens"]
    nh, B, L_max, scale = ng * g, len(lens), max(lens), _scale(c)
    gen = torch.Generator().manual_seed(c["seed"])
    kc = torch.randn(B, L_max, ng * hd, generator=gen).bfloat16().to(DEV)
    vc = torch.randn(B, L_max, ng * hd, generator=gen).bfloat16().to(DEV)
    qkv = torch.randn(B, ng * (g + 2) * hd, generator=gen).bfloat16().to(DEV)
    slopes = alibi_slopes(nh).to(DEV) if c["alibi"] else None
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV)
    out = K().attn_decode(qkv, kc, vc, lens_d, ng, g, hd, scale, alibi_slopes=slopes)
    assert torch.equal(out, K().attn_decode(qkv, kc, vc, lens_d, ng, g, hd, scale, alibi_slopes=slopes))
    out = out.view(B, ng, g, hd)
    bias = _bias(slopes, nh, L_max)
    q = qkv.double().view(B, ng, g + 2, hd)[:, :, :g]
    worst = 0.0
    for b, n in enumerate(lens):
        kk = kc[b, :n].double().view(n, ng, hd)
        vv = vc[b, :n].double().view(n, ng, hd)
        for gi in range(ng):
            raw = kk[:, gi] @ q[b, gi].T  # [n, g]
            bb = bias.view(ng, g, -1)[gi, :, :n].T if bias is not None else torch.zeros_like(raw)
            S = scale * raw + bb
            P = torch.softmax(S, 0)
            Oref = P.T @ vv[:, gi]  # [g, hd]
            lam = LOG2E * (scale * raw.abs() + bb.abs()).amax(0)
            sig = (scale * hd * ACC * (kk[:, gi].abs() @ q[b, gi].abs().T)).amax(0)
            e_t = EXP * (1 + lam) + sig
            rho = (n + 8) * ACC
            bar = ((2 * e_t + 2 * rho)[:, None] * P.T) @ vv[:, gi].abs() + U * Oref.abs()
            worst = max(worst, _ratio(out[b, gi], Oref, bar))
    print(f"\nmax err/bar {name}: out={worst:.3g}")
    assert worst <= 1.0


# ------------------------------------------------------------------------------------------------
# exact properties (torch.equal)
# ------------------------------------------------------------------------------------------------
def _case(hd, alibi, dropout, ng=2, g=2, lens=(130, 65, 0, 257, 63), seed=5):
    return dict(hd=hd, alibi=alibi, dropout=dropout, ng=ng, g=g, scale="rsqrt", dist="normal", lens=list(lens), seed=seed)


PACK_CASES = [(160, False, 0.15), (192, True, 0.0), (256, True, 0.15), (256, False, 0.0)]


@pytest.mark.parametrize("hd,alibi,dropout", PACK_CASES)
def test_wide_two_calls_give_the_same_bytes(hd, alibi, dropout):
    c = _case(hd, alibi, dropout, ng=1, g=5)
    qkv, dout, cu = _inputs(c)
    sl = alibi_slopes(5).to(DEV) if alibi else None
    first = _run(c, sl, qkv, dout, cu)
    second = _run(c, sl, qkv, dout, cu)
    for a, b in zip(first, second):
        assert torch.equal(a, b)


@pytest.mark.parametrize("hd,alibi,dropout", PACK_CASES)
def test_wide_packing_invariance_bit_exact(hd, alibi, dropout):
    """a document's out, lse and dqkv rows do not depend on its neighbours: random large values around it, and the
    document alone in a buffer of its own length (TMA zero-fill replaces the neighbour rows), give the same bits"""
    c = _case(hd, alibi, dropout)
    qkv, dout, cu = _inputs(c)
    sl = alibi_slopes(4).to(DEV) if alibi else None
    out, lse, dqkv = _run(c, sl, qkv, dout, cu)
    s, e = int(cu[1]), int(cu[2])  # the 65-token document: ends mid-tile, neighbours on both sides
    gen = torch.Generator().manual_seed(99)
    qkv2, dout2 = qkv.clone(), dout.clone()
    keep = torch.zeros(qkv.shape[0], dtype=torch.bool, device=DEV)
    keep[s:e] = True
    qkv2[~keep] = (64 * torch.randn(qkv.shape, generator=gen)).bfloat16().to(DEV)[~keep]
    dout2[~keep] = (64 * torch.randn(dout.shape, generator=gen)).bfloat16().to(DEV)[~keep]
    out2, lse2, dqkv2 = _run(c, sl, qkv2, dout2, cu)
    assert torch.isfinite(out2).all() and torch.isfinite(dqkv2).all()
    assert torch.equal(out2[s:e], out[s:e]) and torch.equal(lse2[:, s:e], lse[:, s:e]) and torch.equal(dqkv2[s:e], dqkv[s:e])
    for d in (0, len(cu) - 2):  # the first document keeps its global positions (its dropout masks); the last without dropout
        s, e = int(cu[d]), int(cu[d + 1])
        if d and dropout:
            continue
        ca = dict(c, lens=[e - s])
        oa, la, da = _run(ca, sl, qkv[s:e].contiguous(), dout[s:e].contiguous(), np.array([0, e - s], np.int32))
        assert torch.equal(oa, out[s:e]) and torch.equal(la, lse[:, s:e]) and torch.equal(da, dqkv[s:e]), d


@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_wide_every_output_element_is_written_and_cta_order_changes_no_bit(hd):
    """dqkv pre-filled with NaN holds no NaN afterwards, and attn_head_fastest in {0, 1, 8} gives identical results"""
    c = _case(hd, hd == 192, 0.15 if hd == 160 else 0.0, ng=3, g=2)
    qkv, dout, cu = _inputs(c)
    sl = alibi_slopes(6).to(DEV) if c["alibi"] else None
    default = K().get_option("attn_head_fastest")
    results = []
    try:
        for opt in (0, 1, 8):
            K().set_option("attn_head_fastest", opt)
            results.append(_run(c, sl, qkv, dout, cu))
    finally:
        K().set_option("attn_head_fastest", default)
    for res in results[1:]:
        for a, b in zip(res, results[0]):
            assert torch.equal(a, b)
    out, lse, _ = results[0]
    args = (torch.from_numpy(cu).to(DEV), max(c["lens"]), c["ng"], c["g"], hd, _scale(c))
    dqkv = K().attn_varlen_bwd(dout, qkv, out, lse, *args, dqkv=torch.full_like(qkv, float("nan")),
                               dropout_p=c["dropout"], dropout_keys=(12345, 678), alibi_slopes=sl)
    assert not dqkv.isnan().any() and torch.equal(dqkv, results[0][2])
