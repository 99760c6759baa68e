"""MoE MLP of MoEDolomite on the B200 kernels (reference: moe_dolomite/moe/base.py:53-181 SparseMoE, moe/scatter.py:18-138
ScatterMoE, moe_dolomite/layer.py:51-95 SparseMoEBlock).

    router logits = x gate^T -> top-k on raw logits -> fp32 softmax over the k selected -> bf16 weights
    tokens grouped by expert (segments padded to 128 rows)  -> grouped wgmma GEMM c_fc -> activation (any name
    activations.resolve accepts) -> grouped GEMM c_proj -> gate-weighted combine (+ m_residual scale + residual add fused)

Padding rows of a segment are zeros in the gathered input (or a copy of token 0's row with the fused gather), so their
`act` rows are finite but not zero for functions with f(0) != 0 (sigmoid, softplus, hard_sigmoid, laplace, log_sigmoid),
and with expert biases their `fc` rows are the bias (plus the copied row's product).  They never reach a result: the
combine reads only the rows of `row_of_slot`, and the combine backward writes zero `dyg` rows for them, so they add exact
zeros to the c_proj weight gradient and give zero `d_fc` rows to the c_fc one.

Expert biases (ParameterizedExperts with add_bias, moe/base.py:12-50; the reference's `eager` experts -- ScatterMoE
forbids them, moe/scatter.py:22): bias[e] is added in the grouped GEMMs' fp32 epilogue on expert e's rows, one rounding to
bf16 as in the dense biased linear.  Their gradients are per-segment column sums over the padded expert segments
`plan.offsets` (whose padding rows add exact zeros): d c_proj.bias[e] of `dyg` (which carries the gate weight and
m_residual), d c_fc.bias[e] of `d_fc`, fused into the activation backward.  Both reduce in a fixed order with no float
atomics, and an expert without tokens adds exact zeros.  Activations stay grouped between the two expert GEMMs exactly
like `parallel_linear(grouped_out=True)` -> `parallel_linear(grouped_in=True, gates=...)`.

Shapes: any E in [1, 256] and any n_embd / n_inner that are multiples of 8.  The grouped GEMMs zero-fill each expert's
K and N tails from its own extent, so no product ever reads another expert's weights.  The router kernels index
contiguous [T, E] buffers while the gate GEMMs need 16-byte rows: kernels.router_logits / router_grad convert between
the two, copies only when E % 8 != 0.
"""

from __future__ import annotations

import os

from . import kernels as K

# DOLO_MOE_FUSED_GATHER=1: the expert c_fc GEMM gathers its token rows itself (the producer warp copies them into the
# operand ring).  Exact; off by default: one warp's loads do not keep the ring as full as TMA loads of a gathered copy.
FUSED_GATHER = os.environ.get("DOLO_MOE_FUSED_GATHER", "0") == "1"


def forward(engine, unit, p: str, x, residual, m_res: float, layer: int = 0):
    cfg = engine.cfg
    k = cfg.num_experts_per_tok
    b_fc, b_proj = unit.views.get(p + "mlp.c_fc.bias"), unit.views.get(p + "mlp.c_proj.bias")
    # [T, E] bf16 (tiny N: direct-store epilogue), contiguous for the router kernels (a copy when E % 8 != 0)
    logits = K.router_logits(engine._linear(unit, p + "mlp.gate.weight", x, flags=0))
    plan = K.moe_route(logits, k)
    if engine._aux_fwd is not None:  # load-balancing statistics of this layer (once per forward: not in recomputed blocks)
        acc, T_real, router_logits = engine._aux_fwd
        K.moe_aux_stats(logits, plan, T_real, acc)
        router_logits.append(logits)
    if FUSED_GATHER:
        # scattermoe `parallel_linear(grouped_in=False, grouped_out=True)`: the expert GEMM reads the token rows straight
        # out of x (copied by its producer warp); no grouped copy of x is written in forward
        fc = K.gemm_grouped_m_gather(x, unit.views[p + "mlp.c_fc.weight"], plan, bias=b_fc)
    else:
        fc = K.gemm_grouped_m(K.moe_gather(x, plan), unit.views[p + "mlp.c_fc.weight"], plan, b_mn=False, bias=b_fc)
    act = K.act_fwd(fc, *engine.act)
    yg = K.gemm_grouped_m(act, unit.views[p + "mlp.c_proj.weight"], plan, b_mn=False, bias=b_proj)
    p_res = engine._drop_p("resid_pdrop")
    if p_res > 0:  # moe/base.py:106-120: dropout on the combined expert output, then layer.py's `* m_residual` / `+ residual`
        y = K.moe_combine(yg, plan)
        out = K.dropout_fwd(y, p_res, engine._drop_keys(4 * layer + 2), residual=residual, post_mul=m_res, out=y)
    else:
        out = K.moe_combine(yg, plan, c=residual, alpha=m_res)
    return out, (plan, logits, fc, act, yg)


def backward(engine, unit, p: str, x, dh, m_res: float, saved, layer: int = 0):
    """returns d(x) (gradient wrt the MoE input, i.e. the ln_2 output); accumulates expert / gate weight grads"""
    plan, logits, fc, act, yg = saved
    p_res = engine._drop_p("resid_pdrop")
    if p_res > 0:
        dyg, dw = K.moe_combine_bwd(K.dropout_bwd(dh, p_res, engine._drop_keys(4 * layer + 2), pre_mul=m_res), yg, plan)
    else:
        dyg, dw = K.moe_combine_bwd(dh, yg, plan, alpha=m_res)
    w_proj, w_fc = unit.views[p + "mlp.c_proj.weight"], unit.views[p + "mlp.c_fc.weight"]
    # the first expert weight gradient of an accumulation window OVERWRITES its buffer (engine.zero_grad is lazy); an expert
    # without tokens is written as zeros by the K-grouped GEMM itself
    beta_proj = 0.0 if engine.take_fresh(p + "mlp.c_proj.weight") else 1.0
    beta_fc = 0.0 if engine.take_fresh(p + "mlp.c_fc.weight") else 1.0
    K.gemm_grouped_k(dyg, act, plan, unit.gviews[p + "mlp.c_proj.weight"], beta=beta_proj)  # dWproj[e] (+)= dY_e^T act_e
    # expert biases: their gradient buffers are cleared by zero_grad (not lazily), so the segment sums accumulate; dyg
    # already holds m_residual (the dense c_proj's colsum alpha)
    gb_fc, gb_proj = unit.gviews.get(p + "mlp.c_fc.bias"), unit.gviews.get(p + "mlp.c_proj.bias")
    if gb_proj is not None:
        K.colsum_accum_segmented(dyg, plan.offsets, gb_proj)                          # dbproj[e] += sum of dY_e rows
    d_act = K.gemm_grouped_m(dyg, w_proj, plan, b_mn=True)                            # [rows, F]
    if gb_fc is not None:  # dbfc[e] += sum of d_fc_e rows, fused into the activation backward
        d_fc = K.act_bwd_segmented(d_act, fc, *engine.act, plan.offsets, gb_fc)
    else:
        d_fc = K.act_bwd(d_act, fc, *engine.act)
    xg = K.moe_gather(x, plan)  # grouped (zero-padded) copy of the block input: the contraction operand of the c_fc wgrad
    K.gemm_grouped_k(d_fc, xg, plan, unit.gviews[p + "mlp.c_fc.weight"], beta=beta_fc)  # dWfc[e] (+)= dfc_e^T x_e
    del xg
    dxg = K.gemm_grouped_m(d_fc, w_fc, plan, b_mn=True)                               # [rows, H]
    dx = K.moe_token_sum(dxg, plan)
    # router path: softmax-over-k backward (+ the load-balancing term) -> dense dlogits -> gate wgrad and dx contribution;
    # an FP8 router casts (and takes the amax of) dlogits with the term in it, as te.Linear would see it
    if engine._aux_bwd is not None:
        c, s, T_real = engine._aux_bwd
        dlogits = K.moe_router_bwd_aux(logits, plan, dw, c, s, T_real)
    else:
        dlogits = K.moe_router_bwd(plan, dw)
    dlogits = K.router_grad(dlogits)  # 16-byte rows for the GEMMs below (a copy when E % 8 != 0)
    if engine._is_fp8(p + "mlp.gate.weight"):  # the router as te.Linear (num_experts % 16 == 0)
        return engine._linear_bwd_fp8(unit, p + "mlp.gate.weight", None, x, dlogits, dx_add=dx)
    gate = unit.views[p + "mlp.gate.weight"]
    ggate = unit.gviews[p + "mlp.gate.weight"]
    # dGate[E, H] += dlogits^T x: E rows are one row of output tiles with the whole token stream as contraction.  Not split
    # over K: the fp32 atomics of a split-K launch sum in arrival order, and the training step is bit-identical run to run.
    K.gemm(dlogits, x, a_mn=True, b_mn=True, out=ggate, c=ggate, beta=1.0, flags=0)
    dx = K.gemm(dlogits, gate, b_mn=True, out=dx, c=dx, beta=1.0, flags=0)          # dx += dlogits gate
    return dx
