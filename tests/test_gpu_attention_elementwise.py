"""GPU: every attention kernel instance against a plain fp64 reference, element by element, and exact properties.

Per-element bars.  The reference is computed on the GPU with fp64 matmuls, one document and one q head at a time, from the
same bf16 tensors the kernels get (Z = the dropout keep scales, b = the bf16 ALiBi bias of the key's index in its document):

    S = scale * Q K^T + b (causal inside the document)    lse = logsumexp(S)    P = exp(S - lse)    Pd = P * Z    O = Pd V
    Delta = rowsum(dO * out)    dP = dO V^T    dS = P * (Z * dP - Delta)
    dV = Pd^T dO    dK = scale * dS^T Q    dQ = scale * dS K    (dK, dV summed over the q heads of the kv group)

`out` in Delta is the kernel's bf16 forward output, the backward's documented input, and the backward gets the kernel's
LSE.  Each bar is a running-error bound built from the kernels' rounding points (attention_fwd.cu, attention_bwd.cu,
attention_decode.cu), evaluated with the same fp64 matmuls on absolute values.  Per query row t:

    u      = 2^-8    bf16 unit roundoff: P before P.V and before dV, dS before dK and dQ, every output once
    eps_t  = 2^-22 (1 + Lam_t)    relative error of one exp2: the argument is formed in fp32 from terms up to
             Lam_t = log2(e) max_j (|scale q.k_j| + |b_j|) over the row's keys (fp32 keeps 2^-24 of each; three roundings
             and the product with the rounded scale * log2 e), plus ex2.approx's 2^-22
    sig_t  = scale hd 2^-23 max_j sum_d |q_d k_jd|    the fp32 tensor-core score (hd additions, each within 2^-23)
    e_t    = eps_t + sig_t    relative error of one unnormalised probability
    rho    = (n + 8) 2^-23    an fp32 sum of n terms (row sum l, the O / dV / dK / dQ accumulators) and a few roundings
    beta_t = e_t + (n_t + 8) 2^-24 + 4 2^-24 (|lse_t| + Lam_t)    LSE bar (natural log units): the exp errors, the fp32
             row sum of n_t keys, logf, m * scale and the final add, and the log2(e) product of the backward
    gam_t  = (hd + 8) 2^-24 sum_d |dO_td out_td|    fp32 Delta
    eta_tk = hd 2^-23 sum_d |dO_td V_kd|    fp32 tensor-core dP

    lse:  |lse - ref| <= beta_t
    out:  (u + 2 e_t + 2 rho_t) sum_j Pd_tj |V_jd| + u |O_td|        (decode: the same without the u of P)
    dV:   sum_t (u + e_t + beta_t + rho) Pd_tk |dO_td| + u |dV_kd|
    dK:   scale sum_t W_tk |Q_td| + u |dK_kd|,  dQ: scale sum_k W_tk |K_kd| + u |dQ_td|, with
          W_tk = P_tk [(u + e_t + beta_t + rho + 2^-22) |Z dP_tk - Delta_t| + Z_tk eta_tk + gam_t]

No bar is a fraction of a tensor-wide norm; the constants come from the arithmetic above, not from measured errors.
Each test prints max(err / bar) per output.
"""

import math

import numpy as np
import pytest
import torch

import alibi_oracle as A
import oracle.dolomite_oracle as O
from attention_instances import DECODE_CASES, FWD_BWD_CASES
from dolomite_engine_b200.alibi import alibi_slopes

pytestmark = pytest.mark.gpu

U = 2.0**-8  # bf16 unit roundoff
F32 = 2.0**-24  # fp32 unit roundoff (round to nearest)
ACC = 2.0**-23  # one fp32 addition of a tensor-core or fp32 accumulation, any rounding direction
EXP = 2.0**-22  # ex2.approx.f32 relative error
LOG2E = 1.0 / math.log(2.0)
KEYS = (12345, 678)  # dropout keys of every dropout case
DEV = "cuda"


def K():
    from dolomite_engine_b200 import kernels

    return kernels


class _FixedKeys(O.DropoutOracle):
    """the oracle's attention dropout masks with the kernels' keys"""

    def __init__(self, keys):
        self._k = keys

    def keys(self, site):
        return self._k


def _scale(c) -> float:
    return 1.0 / math.sqrt(c["hd"]) if c["scale"] == "rsqrt" else 1.0 / c["hd"]


def _inputs(c):
    """bf16 qkv [T, ng * (g + 2) * hd] and dout [T, nh * hd] of case c (on the GPU) and cu_seqlens (numpy)"""
    ng, g, hd, lens = c["ng"], c["g"], c["hd"], c["lens"]
    gen = torch.Generator().manual_seed(c["seed"])
    T = sum(lens)
    x = torch.randn(T, ng, g + 2, hd, generator=gen, dtype=torch.float64)
    dout = torch.randn(T, ng * g * hd, generator=gen)
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    dist = c.get("dist", "normal")
    if dist == "peaked":  # nearly one-hot softmax rows
        x[:, :, :g] *= 4
    elif dist == "flat":  # every logit is the bias: the LSE is a long fp32 sum
        x[:, :, :g] = 0
    elif dist == "late":
        # queries get a common direction mu; in documents of >= 256 tokens the keys of the last 128-key tile are shifted
        # along the mean query so that q_t . shift is ~6 / scale on average: the rows of the last tile find their maximum
        # logit in their last key tile, after the running max has settled on the earlier tiles
        mu = torch.randn(ng, 1, hd, generator=gen, dtype=torch.float64)
        mu /= mu.norm(dim=-1, keepdim=True)
        x[:, :, :g] += 2 * mu
        xb = x.to(torch.bfloat16).double()
        for d in range(len(lens)):
            s, e = int(cu[d]), int(cu[d + 1])
            if e - s < 256:
                continue
            qbar = xb[s:e, :, :g].mean(dim=(0, 2))  # [ng, hd]
            shift = 6.0 / _scale(c) * qbar / (qbar * qbar).sum(-1, keepdim=True)
            x[s + (e - s - 1) // 128 * 128:e, :, g] += shift
    qkv = x.reshape(T, -1).to(torch.bfloat16)
    return qkv.to(DEV), dout.to(torch.bfloat16).to(DEV), cu


def _bias(slopes, nh: int, L: int):
    """[nh, L] fp64 bias of key positions 0..L-1 (bf16 values), or None"""
    if slopes is None:
        return None
    return A.alibi_bias(slopes.cpu(), torch.arange(L).unsqueeze(0), True)[0].double().to(DEV)


def _reference(c, qkv, dout, out_k, lse_k, cu, slopes, backward: bool):
    """fp64 reference and per-element bars of every output of case c (see the module docstring)"""
    ng, g, hd, p = c["ng"], c["g"], c["hd"], c["dropout"]
    nh, T, scale = ng * g, qkv.shape[0], _scale(c)
    x = qkv.double().view(T, ng, g + 2, hd)
    do = dout.double().view(T, ng, g, hd)
    ok = out_k.double().view(T, ng, g, hd)
    r = {n: torch.zeros(T, ng, g, hd, dtype=torch.float64, device=DEV) for n in ("out", "out_bar", "dq", "dq_bar")}
    r.update({n: torch.zeros(T, ng, hd, dtype=torch.float64, device=DEV) for n in ("dk", "dk_bar", "dv", "dv_bar")})
    r["lse"] = torch.zeros(nh, T, dtype=torch.float64, device=DEV)
    r["lse_bar"] = torch.zeros(nh, T, dtype=torch.float64, device=DEV)
    drop = _FixedKeys(KEYS) if p else None
    bias_all = _bias(slopes, nh, max(c["lens"]))
    for d in range(len(cu) - 1):
        s, e = int(cu[d]), int(cu[d + 1])
        L = e - s
        if L == 0:
            continue
        causal = torch.ones(L, L, dtype=torch.bool, device=DEV).tril()
        n_t = torch.arange(1, L + 1, dtype=torch.float64, device=DEV)
        rho_f = (n_t + 8) * ACC
        rho_b = (g * L + 8) * ACC
        tok = np.arange(s, e)
        for gi in range(ng):
            Kd, Vd = x[s:e, gi, g], x[s:e, gi, g + 1]
            for j in range(g):
                h = gi * g + j
                Q = x[s:e, gi, j]
                raw = Q @ Kd.T
                b = bias_all[h, :L] if bias_all is not None else torch.zeros(L, dtype=torch.float64, device=DEV)
                S = (scale * raw + b).masked_fill(~causal, -math.inf)
                lse = torch.logsumexp(S, -1)
                P = torch.exp(S - lse[:, None])
                Z = drop.attn_scale(0, h, tok, tok, p).double().to(DEV) if drop else torch.ones_like(P)
                Pd = P * Z
                Oref = Pd @ Vd
                lam = LOG2E * (scale * raw.abs() + b.abs()).masked_fill(~causal, 0).amax(-1)
                sig = (scale * hd * ACC * (Q.abs() @ Kd.abs().T)).masked_fill(~causal, 0).amax(-1)
                e_t = EXP * (1 + lam) + sig
                beta = e_t + (n_t + 8) * F32 + 4 * F32 * (lse.abs() + lam)
                r["lse"][h, s:e], r["lse_bar"][h, s:e] = lse, beta
                r["out"][s:e, gi, j] = Oref
                r["out_bar"][s:e, gi, j] = ((U + 2 * e_t + 2 * rho_f)[:, None] * Pd) @ Vd.abs() + U * Oref.abs()
                if not backward:
                    continue
                dO, Ok = do[s:e, gi, j], ok[s:e, gi, j]
                delta = (dO * Ok).sum(-1)
                gam = (hd + 8) * F32 * (dO * Ok).abs().sum(-1)
                dP = dO @ Vd.T
                eta = hd * ACC * (dO.abs() @ Vd.abs().T)
                Adiff = Z * dP - delta[:, None]
                dS = P * Adiff
                cb = U + e_t + beta + rho_b
                W = P * ((cb + EXP)[:, None] * Adiff.abs() + Z * eta + gam[:, None])
                r["dv"][s:e, gi] += Pd.T @ dO
                r["dv_bar"][s:e, gi] += (cb[:, None] * Pd).T @ dO.abs()
                r["dk"][s:e, gi] += scale * (dS.T @ Q)
                r["dk_bar"][s:e, gi] += scale * (W.T @ Q.abs())
                dQ = scale * (dS @ Kd)
                r["dq"][s:e, gi, j] = dQ
                r["dq_bar"][s:e, gi, j] = scale * (W @ Kd.abs()) + U * dQ.abs()
    r["dk_bar"] += U * r["dk"].abs()
    r["dv_bar"] += U * r["dv"].abs()
    return r


def _ratio(got, ref, bar) -> float:
    """max |got - ref| / bar over all elements (bar 0 demands an exact 0 error); NaN in got gives NaN"""
    err = (got.double() - ref).abs()
    return (err / bar.clamp_min(1e-300)).max().item() if err.numel() else 0.0


def _run(c, slopes, qkv, dout, cu):
    """attn_varlen_fwd and attn_varlen_bwd of case c -> out, lse, dqkv"""
    ng, g, hd = c["ng"], c["g"], c["hd"]
    cu_d = torch.from_numpy(cu).to(DEV)
    args = (cu_d, max(c["lens"]), ng, g, hd, _scale(c))
    dk = dict(dropout_p=c["dropout"], dropout_keys=KEYS, alibi_slopes=slopes)
    out, lse = K().attn_varlen_fwd(qkv, *args, **dk)
    dqkv = K().attn_varlen_bwd(dout, qkv, out, lse, *args, **dk)
    return out, lse, dqkv


@pytest.mark.parametrize("name", sorted(FWD_BWD_CASES))
def test_attention_fwd_bwd_per_element_vs_fp64(name):
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
def test_attention_decode_per_element_vs_fp64(name):
    c = DECODE_CASES[name]
    ng, g, hd, lens = c["ng"], c["g"], c["hd"], c["lens"]
    nh, B, L_max, scale = ng * g, len(lens), max(lens), _scale(c)
    gen = torch.Generator().manual_seed(c["seed"])
    kc = torch.randn(B, L_max, ng * hd, generator=gen).bfloat16().to(DEV)
    vc = torch.randn(B, L_max, ng * hd, generator=gen).bfloat16().to(DEV)
    qkv = torch.randn(B, ng * (g + 2) * hd, generator=gen).bfloat16().to(DEV)
    slopes = alibi_slopes(nh).to(DEV) if c["alibi"] else None
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV)
    out = K().attn_decode(qkv, kc, vc, lens_d, ng, g, hd, scale, alibi_slopes=slopes).view(B, ng, g, hd)
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
def _case(hd, alibi, dropout, ng=2, g=2, lens=(130, 65, 0, 257, 63), seed=5, scale="rsqrt"):
    return dict(hd=hd, alibi=alibi, dropout=dropout, ng=ng, g=g, scale=scale, dist="normal", lens=list(lens), seed=seed)


def _slopes(c):
    return alibi_slopes(c["ng"] * c["g"]).to(DEV) if c["alibi"] else None


PACK_CASES = [(16, False, 0.15), (32, True, 0.0), (64, False, 0.0), (80, True, 0.15), (96, False, 0.15), (128, True, 0.0)]


@pytest.mark.parametrize("hd,alibi,dropout", PACK_CASES)
def test_packing_invariance_bit_exact(hd, alibi, dropout):
    """a document's out, lse and dqkv rows do not depend on its neighbours: masked keys contribute exactly 0 and each
    document's tiles start at its first token (dropout masks hash global positions, which stay where they are)"""
    c = _case(hd, alibi, dropout)
    qkv, dout, cu = _inputs(c)
    sl = _slopes(c)
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
    # alone in a buffer of its own length: TMA zero-fill replaces the neighbour rows.  The first document keeps its global
    # positions (and so its dropout masks); the last one is compared without dropout.
    for d in (0, len(cu) - 2):
        s, e = int(cu[d]), int(cu[d + 1])
        if d and dropout:
            continue
        ca = dict(c, lens=[e - s])
        oa, la, da = _run(ca, sl, qkv[s:e].contiguous(), dout[s:e].contiguous(), np.array([0, e - s], np.int32))
        assert torch.equal(oa, out[s:e]) and torch.equal(la, lse[:, s:e]) and torch.equal(da, dqkv[s:e]), d


@pytest.mark.parametrize("cfg", ["gqa-hd80-alibi-dropout", "mha-hd128-8heads-long"])
def test_cta_order_does_not_change_a_bit(cfg):
    """attn_head_fastest (the CTA order of all three kernels) in {0, 1, 8, n_heads + 3}: identical out, lse and dqkv.
    The 8-head hd-128 batch of 6500 tokens is past the forward's all-heads-in-one-chunk threshold (24 MB of K / V)."""
    if cfg.startswith("gqa"):
        c = _case(80, True, 0.15, ng=3, g=2)
    else:
        c = _case(128, False, 0.0, ng=8, g=1, lens=(3000, 1, 2500, 0, 1000), seed=6)
    qkv, dout, cu = _inputs(c)
    sl = _slopes(c)
    default = K().get_option("attn_head_fastest")
    results = []
    try:
        for opt in (0, 1, 8, c["ng"] * c["g"] + 3):
            K().set_option("attn_head_fastest", opt)
            results.append(_run(c, sl, qkv, dout, cu))
    finally:
        K().set_option("attn_head_fastest", default)
    for res in results[1:]:
        for a, b in zip(res, results[0]):
            assert torch.equal(a, b)


@pytest.mark.parametrize("hd,alibi,dropout", [(16, True, 0.0), (80, False, 0.15), (96, True, 0.15), (128, False, 0.0)])
def test_every_output_element_is_written(hd, alibi, dropout):
    """out, lse and every slot of dqkv pre-filled with NaN hold no NaN afterwards (lse through the C entry point, since the
    wrapper allocates it); a q head whose dO is all zeros gets dQ exactly 0 and leaves the other heads' dQ unchanged"""
    from dolomite_engine_b200 import _lib

    c = _case(hd, alibi, dropout, ng=2, g=3)
    qkv, dout, cu = _inputs(c)
    sl = _slopes(c)
    ng, g, T, nh = c["ng"], c["g"], qkv.shape[0], c["ng"] * c["g"]
    cu_d = torch.from_numpy(cu).to(DEV)
    out = torch.full((T, nh * hd), float("nan"), dtype=torch.bfloat16, device=DEV)
    lse = torch.full((nh, T), float("nan"), dtype=torch.float32, device=DEV)
    common = (qkv.data_ptr(), qkv.stride(0), out.data_ptr(), lse.data_ptr(), cu_d.data_ptr(), len(cu) - 1, T, max(c["lens"]),
              ng, g, hd, _scale(c), float(dropout), KEYS[0], KEYS[1])
    if alibi:
        _lib.call("dolomite_b200_attn_varlen_fwd_alibi", *common, sl.data_ptr(), K()._stream())
    else:
        _lib.call("dolomite_b200_attn_varlen_fwd_dropout", *common, K()._stream())
    assert not out.isnan().any() and not lse.isnan().any()
    args = (cu_d, max(c["lens"]), ng, g, hd, _scale(c))
    kw = dict(dropout_p=dropout, dropout_keys=KEYS, alibi_slopes=sl)
    dqkv = K().attn_varlen_bwd(dout, qkv, out, lse, *args, dqkv=torch.full_like(qkv, float("nan")), **kw)
    assert not dqkv.isnan().any()
    zero_head = 4  # group 1, slot 1
    dout0 = dout.clone()
    dout0[:, zero_head * hd:(zero_head + 1) * hd] = 0
    dq0 = K().attn_varlen_bwd(dout0, qkv, out, lse, *args, **kw).view(T, ng, g + 2, hd)
    d = dqkv.view(T, ng, g + 2, hd)
    assert torch.equal(dq0[:, 1, 1], torch.zeros_like(dq0[:, 1, 1]))
    for h in range(nh):
        if h != zero_head:
            assert torch.equal(dq0[:, h // g, h % g], d[:, h // g, h % g]), h


@pytest.mark.parametrize("hd,alibi,dropout", [(32, False, 0.15), (80, True, 0.0), (128, False, 0.0)])
def test_row_strided_qkv_and_dqkv(hd, alibi, dropout):
    """qkv and dqkv as views with a row stride past the slot layout (NaN in the padding columns): results identical to the
    contiguous run, and the padding columns of a given dqkv keep their sentinel"""
    c = _case(hd, alibi, dropout)
    qkv, dout, cu = _inputs(c)
    sl = _slopes(c)
    T, Wd = qkv.shape
    pad = 24
    big = torch.full((T, Wd + pad), float("nan"), dtype=torch.bfloat16, device=DEV)
    big[:, :Wd] = qkv
    qv = big[:, :Wd]
    ref = _run(c, sl, qkv, dout, cu)
    cu_d = torch.from_numpy(cu).to(DEV)
    args = (cu_d, max(c["lens"]), c["ng"], c["g"], hd, _scale(c))
    kw = dict(dropout_p=dropout, dropout_keys=KEYS, alibi_slopes=sl)
    out, lse = K().attn_varlen_fwd(qv, *args, **kw)
    assert torch.equal(out, ref[0]) and torch.equal(lse, ref[1])
    dbig = torch.full((T, Wd + pad), float("nan"), dtype=torch.bfloat16, device=DEV)
    d = K().attn_varlen_bwd(dout, qv, out, lse, *args, dqkv=dbig[:, :Wd], **kw)
    assert torch.equal(d, ref[2]) and dbig[:, Wd:].isnan().all()
    d2 = K().attn_varlen_bwd(dout, qv, out, lse, *args, **kw)  # allocated with qkv's strides
    assert d2.stride() == qv.stride() and torch.equal(d2, ref[2])


@pytest.mark.parametrize("hd,alibi", [(16, False), (80, True), (128, False)])
def test_decode_ignores_cache_positions_past_the_length(hd, alibi):
    ng, g = 2, 3
    lens = [1, 127, 128, 129, 300]
    B, L_max = len(lens), 384
    gen = torch.Generator().manual_seed(11)
    kc = torch.randn(B, L_max, ng * hd, generator=gen).bfloat16().to(DEV)
    vc = torch.randn(B, L_max, ng * hd, generator=gen).bfloat16().to(DEV)
    qkv = torch.randn(B, ng * (g + 2) * hd, generator=gen).bfloat16().to(DEV)
    sl = alibi_slopes(ng * g).to(DEV) if alibi else None
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV)
    out = K().attn_decode(qkv, kc, vc, lens_d, ng, g, hd, hd**-0.5, alibi_slopes=sl)
    kn, vn = kc.clone(), vc.clone()
    for b, n in enumerate(lens):
        kn[b, n:] = float("nan")
        vn[b, n:] = float("nan")
    out2 = K().attn_decode(qkv, kn, vn, lens_d, ng, g, hd, hd**-0.5, alibi_slopes=sl)
    assert torch.equal(out2, out)
