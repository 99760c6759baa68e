"""Thin torch-tensor wrappers over the C ABI (include/dolomite_b200.h).

torch is used only for device memory and streams; every computation below is a hand-written sm_90a kernel.
All functions launch on torch's current CUDA stream and never synchronise.
"""

from __future__ import annotations

import torch

from . import _lib

_BF16 = torch.bfloat16


def set_option(key: str, value: int) -> None:
    """process-wide tuning knobs of the CUDA library (include/dolomite_b200.h: dolomite_b200_set_option)"""
    _lib.call("dolomite_b200_set_option", key.encode(), int(value))


def get_option(key: str) -> int:
    import ctypes

    v = ctypes.c_int(0)
    _lib.call("dolomite_b200_get_option", key.encode(), ctypes.addressof(v))
    return int(v.value)


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: torch.Tensor | None) -> int | None:
    return None if t is None else t.data_ptr()


def _req(t: torch.Tensor, dtype, name: str) -> None:
    if not t.is_cuda:
        raise _lib.DolomiteB200Error(f"{name} must be a CUDA tensor (no CPU fallback on the hot path)")
    if t.dtype != dtype:
        raise _lib.DolomiteB200Error(f"{name} must be {dtype}, got {t.dtype}")


# ------------------------------------------------------------------------------------------------
# Row layout of [rows, cols] outputs.  TMA and the 16-byte vector kernels need 16-byte row strides, so a width that is
# not a multiple of 16 bytes (the logits of an odd vocabulary) is allocated [rows, round_up(cols, 16 B)] and used as a
# [rows, cols] view of that buffer.  The extra columns are never part of a result (the GEMM's TMA stores and the
# cross-entropy kernel may write zeros there).  Widths that are already multiples give a plain contiguous tensor.
# ------------------------------------------------------------------------------------------------
def rows_empty(rows: int, cols: int, dtype=_BF16, device=None) -> torch.Tensor:
    """uninitialised [rows, cols] tensor whose row stride is a multiple of 16 bytes"""
    per = 16 // torch.empty((), dtype=dtype).element_size()
    ld = -(-cols // per) * per
    if ld == cols:
        return torch.empty(rows, cols, dtype=dtype, device=device)
    return torch.empty(rows, ld, dtype=dtype, device=device)[:, :cols]


def rows_aligned(t: torch.Tensor) -> torch.Tensor:
    """`t` ([rows, cols], unit column stride) if its row stride keeps 16 bytes, else a copy into rows_empty"""
    per = 16 // t.element_size()
    if t.stride(1) == 1 and t.stride(0) % per == 0 and t.data_ptr() % 16 == 0:
        return t
    out = rows_empty(t.shape[0], t.shape[1], t.dtype, t.device)
    out.copy_(t)
    return out


# ------------------------------------------------------------------------------------------------
# RMSNorm (normalization/rmsnorm/base.py:18-25)
# ------------------------------------------------------------------------------------------------
def rmsnorm_fwd(x: torch.Tensor, w: torch.Tensor, eps: float, out: torch.Tensor | None = None):
    _req(x, _BF16, "x"), _req(w, _BF16, "w")
    assert x.is_contiguous() and x.dim() == 2
    T, H = x.shape
    y = torch.empty_like(x) if out is None else out
    rstd = torch.empty(T, dtype=torch.float32, device=x.device)
    _lib.call("dolomite_b200_rmsnorm_fwd", x.data_ptr(), w.data_ptr(), y.data_ptr(), rstd.data_ptr(), T, H, eps, _stream())
    return y, rstd


_ws_cache: dict = {}


def _workspace(nbytes: int, device) -> torch.Tensor:
    key = (device, "ws")
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    return buf


def rmsnorm_bwd(dy, x, w, rstd, dw_accum: torch.Tensor | None, dx_add: torch.Tensor | None = None, out=None):
    _req(dy, _BF16, "dy"), _req(x, _BF16, "x")
    T, H = x.shape
    dx = torch.empty_like(x) if out is None else out
    ws = _workspace(_lib.load().dolomite_b200_rmsnorm_bwd_workspace_bytes(H), x.device)
    if dw_accum is not None:
        _req(dw_accum, torch.float32, "dw_accum")
    _lib.call(
        "dolomite_b200_rmsnorm_bwd", dy.data_ptr(), x.data_ptr(), w.data_ptr(), rstd.data_ptr(), _ptr(dx_add),
        dx.data_ptr(), _ptr(dw_accum), ws.data_ptr(), T, H, _stream(),
    )
    return dx


# ------------------------------------------------------------------------------------------------
# RoPE (position_embedding/rope.py:104-114) in place on packed qkv
# ------------------------------------------------------------------------------------------------
def rope_qk_inplace(qkv, n_groups: int, q_per_group: int, head_dim: int, cos, sin, position_ids, inverse=False):
    _req(qkv, _BF16, "qkv"), _req(cos, _BF16, "cos"), _req(sin, _BF16, "sin")
    assert qkv.dim() == 2 and qkv.stride(1) == 1
    assert position_ids.dtype in (torch.int32, torch.int64) and position_ids.is_contiguous()
    T = qkv.shape[0]
    _lib.call(
        "dolomite_b200_rope_qk_inplace", qkv.data_ptr(), qkv.stride(0), T, n_groups, q_per_group, head_dim,
        cos.data_ptr(), sin.data_ptr(), position_ids.data_ptr(), int(position_ids.dtype == torch.int64),
        cos.shape[0], int(inverse), _stream(),
    )
    return qkv


# ------------------------------------------------------------------------------------------------
# LayerNorm and the MLP activations (activations/{base,glu}.py)
# ------------------------------------------------------------------------------------------------
def layernorm_fwd(x, w, b, eps: float, out=None):
    """y = bf16((x - mean) * rstd * w + b) -> (y, mean, rstd)"""
    _req(x, _BF16, "x"), _req(w, _BF16, "w")
    T, H = x.shape
    y = torch.empty_like(x) if out is None else out
    mean = torch.empty(T, dtype=torch.float32, device=x.device)
    rstd = torch.empty(T, dtype=torch.float32, device=x.device)
    _lib.call("dolomite_b200_layernorm_fwd", x.data_ptr(), w.data_ptr(), _ptr(b), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
              T, H, eps, _stream())
    return y, mean, rstd


def layernorm_bwd(dy, x, w, mean, rstd, dw_accum, db_accum, dx_add=None, out=None):
    _req(dy, _BF16, "dy"), _req(x, _BF16, "x")
    T, H = x.shape
    dx = torch.empty_like(x) if out is None else out
    ws = _workspace(_lib.load().dolomite_b200_layernorm_bwd_workspace_bytes(H), x.device)
    _lib.call("dolomite_b200_layernorm_bwd", dy.data_ptr(), x.data_ptr(), w.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
              _ptr(dx_add), dx.data_ptr(), _ptr(dw_accum), _ptr(db_accum), ws.data_ptr(), T, H, _stream())
    return dx


def act_fwd(x, act_id: int, form: int, out=None):
    """MLP activation (activations.resolve gives `act_id`, `form`): plain [T, F] -> [T, F]; GLU forms [T, 2F] -> [T, F]"""
    _req(x, _BF16, "x")
    T, W = x.shape
    F = W if form == 0 else W // 2
    y = torch.empty(T, F, dtype=_BF16, device=x.device) if out is None else out
    _lib.call("dolomite_b200_act_fwd", act_id, form, x.data_ptr(), y.data_ptr(), T, F, _stream())
    return y


def act_bwd(dy, x, act_id: int, form: int, out=None, bias_grad_accum=None):
    """dx of act_fwd; with `bias_grad_accum` (fp32, one per column of x) also += column sums of dx (bias gradient of c_fc)"""
    _req(dy, _BF16, "dy"), _req(x, _BF16, "x")
    T, W = x.shape
    dx = torch.empty_like(x) if out is None else out
    if bias_grad_accum is not None:
        _req(bias_grad_accum, torch.float32, "bias_grad_accum")
        assert bias_grad_accum.numel() == W
    _lib.call("dolomite_b200_act_bwd", act_id, form, dy.data_ptr(), x.data_ptr(), dx.data_ptr(), _ptr(bias_grad_accum), T,
              W if form == 0 else W // 2, _stream())
    return dx


def gelu_fwd(x, out=None):
    _req(x, _BF16, "x")
    y = torch.empty_like(x) if out is None else out
    _lib.call("dolomite_b200_gelu_fwd", x.data_ptr(), y.data_ptr(), x.numel(), _stream())
    return y


def gelu_bwd(dy, x, out=None, bias_grad_accum=None):
    _req(dy, _BF16, "dy"), _req(x, _BF16, "x")
    T, F = x.shape
    dx = torch.empty_like(x) if out is None else out
    _lib.call("dolomite_b200_gelu_bwd", dy.data_ptr(), x.data_ptr(), dx.data_ptr(), _ptr(bias_grad_accum), T, F, _stream())
    return dx


def swiglu_fwd(x, out=None):
    _req(x, _BF16, "x")
    T, F2 = x.shape
    y = torch.empty(T, F2 // 2, dtype=_BF16, device=x.device) if out is None else out
    _lib.call("dolomite_b200_swiglu_fwd", x.data_ptr(), y.data_ptr(), T, F2 // 2, _stream())
    return y


def swiglu_bwd(dy, x, out=None, bias_grad_accum=None):
    """dx of y = up * silu(gate); with `bias_grad_accum` (fp32 [2F]) also += column sums of dx (bias gradient of c_fc)"""
    _req(dy, _BF16, "dy"), _req(x, _BF16, "x")
    T, F2 = x.shape
    dx = torch.empty_like(x) if out is None else out
    if bias_grad_accum is not None:
        _req(bias_grad_accum, torch.float32, "bias_grad_accum")
        assert bias_grad_accum.numel() == F2
        _lib.call("dolomite_b200_swiglu_bwd_bias", dy.data_ptr(), x.data_ptr(), dx.data_ptr(), bias_grad_accum.data_ptr(),
                  T, F2 // 2, _stream())
    else:
        _lib.call("dolomite_b200_swiglu_bwd", dy.data_ptr(), x.data_ptr(), dx.data_ptr(), T, F2 // 2, _stream())
    return dx


# ------------------------------------------------------------------------------------------------
# Embedding (gpt_dolomite/base.py:351-372)
# ------------------------------------------------------------------------------------------------
def embedding_fwd(ids, wte, scale: float = 1.0, out=None):
    _req(ids, torch.int64, "ids"), _req(wte, _BF16, "wte")
    T = ids.numel()
    V, H = wte.shape
    y = torch.empty(T, H, dtype=_BF16, device=wte.device) if out is None else out
    _lib.call("dolomite_b200_embedding_fwd", ids.data_ptr(), wte.data_ptr(), y.data_ptr(), T, H, V, scale, _stream())
    return y


def embedding_bwd(ids, dout, dwte_accum, scale: float = 1.0):
    _req(ids, torch.int64, "ids"), _req(dout, _BF16, "dout"), _req(dwte_accum, torch.float32, "dwte")
    T = ids.numel()
    V, H = dwte_accum.shape
    _lib.call("dolomite_b200_embedding_bwd", ids.data_ptr(), dout.data_ptr(), dwte_accum.data_ptr(), T, H, V, scale, _stream())


# ------------------------------------------------------------------------------------------------
# Cross entropy fwd+bwd (model_wrapper/pretraining.py:124-125)
# ------------------------------------------------------------------------------------------------
def cross_entropy_fwd_bwd(logits, labels, ignore_index=-100, logit_scale=1.0, grad_scale=1.0, dlogits=None):
    _req(logits, _BF16, "logits"), _req(labels, torch.int64, "labels")
    T, V = logits.shape
    assert logits.stride(1) == 1
    dl = logits if dlogits is None else dlogits
    loss_tok = torch.empty(T, dtype=torch.float32, device=logits.device)
    loss = torch.empty(1, dtype=torch.float32, device=logits.device)
    scratch = torch.empty(2, dtype=torch.float32, device=logits.device)
    _lib.call(
        "dolomite_b200_cross_entropy_fwd_bwd", logits.data_ptr(), logits.stride(0), labels.data_ptr(), dl.data_ptr(),
        loss_tok.data_ptr(), loss.data_ptr(), scratch.data_ptr(), T, V, ignore_index, logit_scale, grad_scale, _stream(),
    )
    return loss, loss_tok, dl


def cross_entropy_count(labels, ignore_index=-100):
    """-> scratch (fp32 [2]); scratch[0] = number of labels != ignore_index (the divisor of the mean loss and its gradient)"""
    _req(labels, torch.int64, "labels")
    scratch = torch.empty(2, dtype=torch.float32, device=labels.device)
    _lib.call("dolomite_b200_cross_entropy_count", labels.data_ptr(), labels.numel(), ignore_index, scratch.data_ptr(), _stream())
    return scratch


def cross_entropy_rows(logits, labels, loss_tok, scratch, ignore_index=-100, logit_scale=1.0, grad_scale=1.0):
    """one chunk of rows: logits [t, V] are overwritten by their gradient, loss_tok [t] receives the per-token losses"""
    _req(logits, _BF16, "logits"), _req(labels, torch.int64, "labels"), _req(loss_tok, torch.float32, "loss_tok")
    t, V = logits.shape
    assert logits.stride(1) == 1 and labels.numel() == t and loss_tok.numel() == t
    _lib.call("dolomite_b200_cross_entropy_rows", logits.data_ptr(), logits.stride(0), labels.data_ptr(), logits.data_ptr(),
              loss_tok.data_ptr(), scratch.data_ptr(), t, V, ignore_index, logit_scale, grad_scale, _stream())
    return logits


def cross_entropy_mean(loss_tok, scratch):
    loss = torch.empty(1, dtype=torch.float32, device=loss_tok.device)
    _lib.call("dolomite_b200_cross_entropy_mean", loss_tok.data_ptr(), loss_tok.numel(), scratch.data_ptr(), loss.data_ptr(), _stream())
    return loss


def colsum_accum(x, out, scale: float = 1.0):
    _req(x, _BF16, "x"), _req(out, torch.float32, "out")
    T, N = x.shape
    _lib.call("dolomite_b200_colsum_accum", x.data_ptr(), x.stride(0), out.data_ptr(), T, N, scale, _stream())


def scale_by_device_scalar(x, scale):
    """x *= scale in place; x contiguous, or [rows, cols] rows of a rows_empty buffer (whole rows of the buffer are
    scaled, its spare columns included)"""
    _req(x, _BF16, "x"), _req(scale, torch.float32, "scale")
    n = x.numel()
    if not x.is_contiguous():
        assert x.dim() == 2 and x.stride(1) == 1 and x.stride(0) >= x.shape[1]
        n = x.shape[0] * x.stride(0)
        assert x.storage_offset() + n <= x.untyped_storage().nbytes() // x.element_size()
    _lib.call("dolomite_b200_scale_bf16_by_device_scalar", x.data_ptr(), n, scale.data_ptr(), _stream())


def add_scaled(a, b, alpha: float, out=None):
    _req(a, _BF16, "a"), _req(b, _BF16, "b")
    o = torch.empty_like(a) if out is None else out
    _lib.call("dolomite_b200_add_scaled", a.data_ptr(), b.data_ptr(), o.data_ptr(), alpha, a.numel(), _stream())
    return o


# ------------------------------------------------------------------------------------------------
# dropout (nn.Dropout after the embeddings / attention c_proj / MLP c_proj; attention-probability dropout lives in the
# attention kernels).  Masks are counter-based: (seed, site) -> two 32-bit keys on the host, element index on the device.
# ------------------------------------------------------------------------------------------------
_M64 = (1 << 64) - 1


def dropout_keys(seed: int, site: int) -> tuple[int, int]:
    """two 32-bit keys of one dropout call site of one forward pass: splitmix64 of (seed, site)"""
    z = (int(seed) * 0x9E3779B97F4A7C15 + (int(site) + 1) * 0xD1B54A32D192ED03) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    z ^= z >> 31
    return int(z & 0xFFFFFFFF), int(z >> 32)


def dropout_fwd(x, p: float, keys: tuple[int, int], residual=None, post_mul: float = 1.0, out=None):
    """[residual +] bf16(bf16(x * mask / (1 - p)) * post_mul)"""
    _req(x, _BF16, "x")
    assert x.is_contiguous() and (residual is None or (residual.is_contiguous() and residual.shape == x.shape))
    o = torch.empty_like(x) if out is None else out
    _lib.call("dolomite_b200_dropout_fwd", x.data_ptr(), _ptr(residual), o.data_ptr(), x.numel(), float(p), float(post_mul),
              keys[0], keys[1], _stream())
    return o


def dropout_bwd(dy, p: float, keys: tuple[int, int], pre_mul: float = 1.0, out=None):
    """bf16(bf16(dy * pre_mul) * mask / (1 - p))"""
    _req(dy, _BF16, "dy")
    assert dy.is_contiguous()
    o = torch.empty_like(dy) if out is None else out
    _lib.call("dolomite_b200_dropout_bwd", dy.data_ptr(), o.data_ptr(), dy.numel(), float(p), float(pre_mul), keys[0], keys[1],
              _stream())
    return o


# ------------------------------------------------------------------------------------------------
# optimizer kernels (train_utils.py:99-106)
# ------------------------------------------------------------------------------------------------
def sumsq_accum(g, out):
    _req(g, torch.float32, "g")
    ws = _workspace(_lib.load().dolomite_b200_sumsq_workspace_bytes(), g.device)
    _lib.call("dolomite_b200_sumsq_accum", g.data_ptr(), g.numel(), out.data_ptr(), ws.data_ptr(), _stream())


def clip_coef(sumsq, max_norm: float, coef_out, norm_out=None):
    _lib.call("dolomite_b200_clip_coef", sumsq.data_ptr(), float(max_norm), coef_out.data_ptr(), _ptr(norm_out), _stream())


def adamw_step(p, g, m, v, p_bf16, lr, beta1, beta2, eps, weight_decay, step, clip=None):
    _req(p, torch.float32, "p"), _req(g, torch.float32, "g")
    _lib.call(
        "dolomite_b200_adamw_step", p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), _ptr(p_bf16), p.numel(),
        lr, beta1, beta2, eps, weight_decay, step, _ptr(clip), _stream(),
    )


def cast_f32_to_bf16(src, dst):
    _lib.call("dolomite_b200_cast_f32_to_bf16", src.data_ptr(), dst.data_ptr(), src.numel(), _stream())


def accum_bf16_into_f32(src, dst, scale=1.0):
    _lib.call("dolomite_b200_accum_bf16_into_f32", src.data_ptr(), dst.data_ptr(), scale, src.numel(), _stream())


# ------------------------------------------------------------------------------------------------
# GEMM (nn.Linear fwd / dgrad / wgrad; linear.py:5-25)
# ------------------------------------------------------------------------------------------------
GEMM_TMA_STORE = 1
GEMM_SPLITK_ACCUMULATE = 2
GEMM_DIRECT_EPILOGUE = 16  # epilogue selection flags of the ABI: accepted, no effect on sm_90 (see include/dolomite_b200.h)
GEMM_F32_TMA_EPILOGUE = 32
# Split-K + fp32-atomic accumulation of weight gradients is off for the block weight gradients (many output tiles, the
# fp32 atomics cost L2 throughput); the entry point stays for shapes with very few output tiles.
wgrad_splitk = False
_default_gemm_flags = GEMM_TMA_STORE
gemm_timer = None  # bench.py: list collecting (flops, start_event, end_event) per GEMM launch


def set_default_gemm_flags(flags: int) -> None:
    global _default_gemm_flags
    _default_gemm_flags = flags


def gemm(a, b, *, a_mn=False, b_mn=False, out=None, out_dtype=_BF16, c=None, alpha=1.0, beta=0.0, bias=None, flags=None):
    """D[M,N] = alpha * A·Bᵀ + bias + beta*C.  A logical [M,K] (stored [K,M] if a_mn), B logical [N,K] (stored [K,N] if b_mn)."""
    _req(a, _BF16, "a"), _req(b, _BF16, "b")
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1
    if a_mn:
        K, M = a.shape
    else:
        M, K = a.shape
    if b_mn:
        Kb, N = b.shape
    else:
        N, Kb = b.shape
    if K != Kb:
        raise _lib.DolomiteB200Error(f"gemm: contraction mismatch {K} vs {Kb}")
    if out is None:
        out = rows_empty(M, N, out_dtype, a.device)
    d_is_f32 = int(out.dtype == torch.float32)
    assert out.stride(1) == 1 and out.shape == (M, N)
    if c is not None:
        assert c.dtype == out.dtype and c.stride(1) == 1
    if flags is None:
        flags = _default_gemm_flags
        if d_is_f32 or c is not None:
            flags &= ~GEMM_TMA_STORE
        if d_is_f32 and c is out and beta == 1.0 and bias is None and wgrad_splitk:
            flags |= GEMM_SPLITK_ACCUMULATE  # weight-gradient accumulation: split-K + fp32 atomics
    if gemm_timer is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    _lib.call(
        "dolomite_b200_gemm_bf16", a.data_ptr(), a.stride(0), int(a_mn), b.data_ptr(), b.stride(0), int(b_mn),
        out.data_ptr(), out.stride(0), d_is_f32, _ptr(c), 0 if c is None else c.stride(0), alpha, beta, _ptr(bias),
        M, N, K, flags, _stream(),
    )
    if gemm_timer is not None:
        e1.record()
        gemm_timer.append((2.0 * M * N * K, e0, e1))
    return out


def gemm_wgrad_multi(problems: list[tuple], n_rows: int | None = None) -> None:
    """problems: up to 4 tuples (dy [K, M] bf16, x [K, N] bf16, dw [M, N] fp32, alpha, accumulate) -> ONE persistent launch
    computing dw (+)= alpha * dy^T x for all of them (the weight gradients of a transformer block; 21.6 waves of tiles
    instead of four launches that each end in a partly filled wave)."""
    import ctypes

    n = len(problems)
    assert 1 <= n <= 4
    K = problems[0][0].shape[0] if n_rows is None else n_rows
    P, L, F, I = ctypes.c_void_p * n, ctypes.c_int64 * n, ctypes.c_float * n, ctypes.c_int * n
    for dy, x, dw, _, _ in problems:
        _req(dy, _BF16, "dy"), _req(x, _BF16, "x"), _req(dw, torch.float32, "dw")
        assert dy.shape[0] == K and x.shape[0] == K and dy.stride(1) == 1 and x.stride(1) == 1 and dw.stride(1) == 1
        assert dw.shape == (dy.shape[1], x.shape[1])
    if gemm_timer is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    _lib.call(
        "dolomite_b200_gemm_bf16_wgrad_multi", n, P(*[q[0].data_ptr() for q in problems]), L(*[q[0].stride(0) for q in problems]),
        P(*[q[1].data_ptr() for q in problems]), L(*[q[1].stride(0) for q in problems]), P(*[q[2].data_ptr() for q in problems]),
        L(*[q[2].stride(0) for q in problems]), L(*[q[0].shape[1] for q in problems]), L(*[q[1].shape[1] for q in problems]),
        K, F(*[float(q[3]) for q in problems]), I(*[int(bool(q[4])) for q in problems]), _stream(),
    )
    if gemm_timer is not None:
        e1.record()
        gemm_timer.append((sum(2.0 * K * q[0].shape[1] * q[1].shape[1] for q in problems), e0, e1))


def gemm_tile_n(shapes: list[tuple[int, int]]) -> tuple[int, float]:
    """output tile width (128 | 256) of a dense gemm / gemm_wgrad_multi launch over these (M, N) outputs on the current
    device, and the per-tile cost ratio c_256 / c_128 of the automatic choice"""
    import ctypes

    n = len(shapes)
    tile_n, cost = ctypes.c_int(0), ctypes.c_float(0.0)
    _lib.call("dolomite_b200_gemm_bf16_tile_n", n, (ctypes.c_int64 * n)(*[s[0] for s in shapes]),
              (ctypes.c_int64 * n)(*[s[1] for s in shapes]), ctypes.addressof(tile_n), ctypes.addressof(cost))
    return int(tile_n.value), float(cost.value)


# ------------------------------------------------------------------------------------------------
# FP8 (te.Linear under te.fp8_autocast with DelayedScaling, HYBRID: e4m3 forward, e5m2 output gradients)
# ------------------------------------------------------------------------------------------------
E4M3, E5M2 = 0, 1
FP8_MAX = {E4M3: 448.0, E5M2: 57344.0}
_U8 = torch.uint8


def fp8_cast(x, fmt: int, scale, *, plain: bool = True, transpose: bool = False, amax=None, out=None, out_t=None):
    """x bf16 [rows, cols] -> (q [rows, cols] or None, q_t [cols, rows] or None), uint8 storage of fp8 `fmt`;
    q = satfinite_rne(fp32(x) * scale).  `scale`: fp32 device scalar (a 1-element view); `amax`: 1-element fp32 view that
    receives max(amax, max|x|)."""
    _req(x, _BF16, "x"), _req(scale, torch.float32, "scale")
    assert x.dim() == 2 and x.stride(1) == 1 and (plain or transpose)
    rows, cols = x.shape
    if plain and out is None:
        out = torch.empty(rows, cols, dtype=_U8, device=x.device)
    if transpose and out_t is None:
        out_t = torch.empty(cols, rows, dtype=_U8, device=x.device)
    if amax is not None:
        _req(amax, torch.float32, "amax")
    _lib.call("dolomite_b200_fp8_cast", x.data_ptr(), x.stride(0), rows, cols, fmt, scale.data_ptr(),
              _ptr(out) if plain else None, _ptr(out_t) if transpose else None, _ptr(amax), _stream())
    return (out if plain else None), (out_t if transpose else None)


def fp8_scaling_update(amax_history, scale, scale_inv, fmt: int) -> None:
    """DelayedScaling update of every slot of one format: amax_history fp32 [len, n], scale / scale_inv fp32 [n]"""
    _req(amax_history, torch.float32, "amax_history"), _req(scale, torch.float32, "scale")
    _req(scale_inv, torch.float32, "scale_inv")
    L, n = amax_history.shape
    assert amax_history.is_contiguous() and scale.numel() == n and scale_inv.numel() == n
    _lib.call("dolomite_b200_fp8_scaling_update", amax_history.data_ptr(), L, n, scale.data_ptr(), scale_inv.data_ptr(),
              FP8_MAX[fmt], _stream())


def gemm_fp8(a, a_fmt: int, a_scale_inv, b, b_fmt: int, b_scale_inv, *, out=None, out_dtype=_BF16, c=None, alpha=1.0,
             beta=0.0, bias=None, split_accumulate: bool = False):
    """D[M,N] = alpha * (a_scale_inv * b_scale_inv * A·Bᵀ + bias) + beta*C with A fp8 [M,K], B fp8 [N,K] (uint8 storage)"""
    _req(a, _U8, "a"), _req(b, _U8, "b"), _req(a_scale_inv, torch.float32, "a_scale_inv")
    _req(b_scale_inv, torch.float32, "b_scale_inv")
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1
    M, K = a.shape
    N, Kb = b.shape
    if K != Kb:
        raise _lib.DolomiteB200Error(f"gemm_fp8: contraction mismatch {K} vs {Kb}")
    if out is None:
        out = torch.empty(M, N, dtype=out_dtype, device=a.device)
    assert out.stride(1) == 1 and out.shape == (M, N)
    if c is not None:
        assert c.dtype == out.dtype and c.stride(1) == 1
    if gemm_timer is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    _lib.call(
        "dolomite_b200_gemm_fp8", a.data_ptr(), a.stride(0), a_fmt, b.data_ptr(), b.stride(0), b_fmt, a_scale_inv.data_ptr(),
        b_scale_inv.data_ptr(), out.data_ptr(), out.stride(0), int(out.dtype == torch.float32), _ptr(c),
        0 if c is None else c.stride(0), alpha, beta, _ptr(bias), M, N, K, int(split_accumulate), _stream(),
    )
    if gemm_timer is not None:
        e1.record()
        gemm_timer.append((2.0 * M * N * K, e0, e1))
    return out


def gemm_fp8_wgrad_multi(problems: list[tuple], dy_fmt: int = E5M2, x_fmt: int = E4M3, split_accumulate: bool = True):
    """problems: up to 4 tuples (dyt fp8 [M, K], dy_scale_inv, xt fp8 [N, K], x_scale_inv, dw fp32 [M, N], alpha,
    accumulate) -> ONE launch computing dw (+)= alpha * s_dy * s_x * dyt · xtᵀ for all of them"""
    import ctypes

    n = len(problems)
    assert 1 <= n <= 4
    K = problems[0][0].shape[1]
    P, L, F, I = ctypes.c_void_p * n, ctypes.c_int64 * n, ctypes.c_float * n, ctypes.c_int * n
    for dyt, sdy, xt, sx, dw, _, _ in problems:
        _req(dyt, _U8, "dyt"), _req(xt, _U8, "xt"), _req(dw, torch.float32, "dw")
        assert dyt.shape[1] == K and xt.shape[1] == K and dyt.stride(1) == 1 and xt.stride(1) == 1 and dw.stride(1) == 1
        assert dw.shape == (dyt.shape[0], xt.shape[0])
    if gemm_timer is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    _lib.call(
        "dolomite_b200_gemm_fp8_wgrad_multi", n, P(*[q[0].data_ptr() for q in problems]), L(*[q[0].stride(0) for q in problems]),
        P(*[q[2].data_ptr() for q in problems]), L(*[q[2].stride(0) for q in problems]),
        P(*[q[1].data_ptr() for q in problems]), P(*[q[3].data_ptr() for q in problems]),
        P(*[q[4].data_ptr() for q in problems]), L(*[q[4].stride(0) for q in problems]),
        L(*[q[0].shape[0] for q in problems]), L(*[q[2].shape[0] for q in problems]), K,
        F(*[float(q[5]) for q in problems]), I(*[int(bool(q[6])) for q in problems]), dy_fmt, x_fmt, int(split_accumulate),
        _stream(),
    )
    if gemm_timer is not None:
        e1.record()
        gemm_timer.append((sum(2.0 * K * q[0].shape[0] * q[2].shape[0] for q in problems), e0, e1))


# ------------------------------------------------------------------------------------------------
# packed var-len causal attention (attention/padding_free.py:51-62)
# ------------------------------------------------------------------------------------------------
def _req_slopes(alibi_slopes, n_heads: int) -> None:
    _req(alibi_slopes, torch.float32, "alibi_slopes")
    if alibi_slopes.numel() != n_heads or not alibi_slopes.is_contiguous():
        raise ValueError(f"alibi_slopes must be a contiguous fp32 [{n_heads}] tensor, got {tuple(alibi_slopes.shape)}")


def _attn_layout(qkv, n_heads: int, head_dim: int, **rows) -> None:
    """the layouts the attention kernels address without looking at strides: qkv rows of unit column stride (any row
    stride), every `rows` tensor (out, dout) a contiguous [T, n_heads * head_dim] tensor; checked before any launch"""
    if qkv.dim() != 2 or qkv.stride(1) != 1:
        raise ValueError(f"qkv must be a 2-D tensor with unit column stride, got strides {tuple(qkv.stride())}")
    T = qkv.shape[0]
    for name, t in rows.items():
        if tuple(t.shape) != (T, n_heads * head_dim) or not t.is_contiguous():
            raise ValueError(f"{name} must be a contiguous [{T}, {n_heads * head_dim}] tensor, got shape "
                             f"{tuple(t.shape)} strides {tuple(t.stride())}")


def _attn_lse_layout(lse, n_heads: int, T: int) -> None:
    if lse.dtype != torch.float32 or tuple(lse.shape) != (n_heads, T) or not lse.is_contiguous():
        raise ValueError(f"lse must be a contiguous fp32 [{n_heads}, {T}] tensor, got {lse.dtype} shape "
                         f"{tuple(lse.shape)} strides {tuple(lse.stride())}")


def _attn_dqkv(qkv, dqkv=None):
    """the dQKV buffer of the backward: the kernels write it with qkv's row stride, so a new one gets qkv's strides and a
    given one must have them"""
    if dqkv is None:
        return torch.empty_strided(qkv.shape, qkv.stride(), dtype=qkv.dtype, device=qkv.device)
    if dqkv.shape != qkv.shape or dqkv.stride() != qkv.stride():
        raise ValueError(f"dqkv must have qkv's shape {tuple(qkv.shape)} and strides {tuple(qkv.stride())}, got "
                         f"{tuple(dqkv.shape)} / {tuple(dqkv.stride())}")
    return dqkv


def attn_varlen_fwd(qkv, cu_seqlens, max_seqlen: int, n_groups: int, q_per_group: int, head_dim: int, scale: float, out=None,
                    dropout_p: float = 0.0, dropout_keys: tuple[int, int] = (0, 0), alibi_slopes=None):
    """`dropout_p` > 0: attention-probability dropout (training mode; attention/padding_free.py:49-59), masks from
    `dropout_keys` (kernels.dropout_keys); the backward call must be given the same p and keys.
    `alibi_slopes` (fp32 [n_heads], alibi.alibi_slopes): ALiBi key bias bf16(slope * index of the key in its document);
    the backward call must be given the same slopes"""
    nh = n_groups * q_per_group
    _attn_layout(qkv, nh, head_dim, **({} if out is None else {"out": out}))
    _req(qkv, _BF16, "qkv"), _req(cu_seqlens, torch.int32, "cu_seqlens")
    if out is not None:
        _req(out, _BF16, "out")
    T = qkv.shape[0]
    o = torch.empty(T, nh * head_dim, dtype=_BF16, device=qkv.device) if out is None else out
    lse = torch.empty(nh, T, dtype=torch.float32, device=qkv.device)
    if alibi_slopes is not None:
        _req_slopes(alibi_slopes, nh)
        _lib.call(
            "dolomite_b200_attn_varlen_fwd_alibi", qkv.data_ptr(), qkv.stride(0), o.data_ptr(), lse.data_ptr(),
            cu_seqlens.data_ptr(), cu_seqlens.numel() - 1, T, int(max_seqlen), n_groups, q_per_group, head_dim, scale,
            float(dropout_p), dropout_keys[0], dropout_keys[1], alibi_slopes.data_ptr(), _stream(),
        )
        return o, lse
    if dropout_p:
        _lib.call(
            "dolomite_b200_attn_varlen_fwd_dropout", qkv.data_ptr(), qkv.stride(0), o.data_ptr(), lse.data_ptr(),
            cu_seqlens.data_ptr(), cu_seqlens.numel() - 1, T, int(max_seqlen), n_groups, q_per_group, head_dim, scale,
            float(dropout_p), dropout_keys[0], dropout_keys[1], _stream(),
        )
        return o, lse
    _lib.call(
        "dolomite_b200_attn_varlen_fwd", qkv.data_ptr(), qkv.stride(0), o.data_ptr(), lse.data_ptr(),
        cu_seqlens.data_ptr(), cu_seqlens.numel() - 1, T, int(max_seqlen), n_groups, q_per_group, head_dim, scale, _stream(),
    )
    return o, lse


def attn_varlen_bwd(dout, qkv, out, lse, cu_seqlens, max_seqlen, n_groups, q_per_group, head_dim, scale, dqkv=None,
                    dropout_p: float = 0.0, dropout_keys: tuple[int, int] = (0, 0), alibi_slopes=None):
    T = qkv.shape[0]
    _attn_layout(qkv, n_groups * q_per_group, head_dim, dout=dout, out=out)
    _attn_lse_layout(lse, n_groups * q_per_group, T)
    dqkv = _attn_dqkv(qkv, dqkv)
    _req(dout, _BF16, "dout"), _req(qkv, _BF16, "qkv"), _req(out, _BF16, "out"), _req(dqkv, _BF16, "dqkv")
    ws_bytes = _lib.load().dolomite_b200_attn_varlen_bwd_workspace_bytes(T, n_groups, q_per_group, head_dim)
    ws = _workspace(ws_bytes, qkv.device)
    if alibi_slopes is not None:
        _req_slopes(alibi_slopes, n_groups * q_per_group)
        _lib.call(
            "dolomite_b200_attn_varlen_bwd_alibi", dout.data_ptr(), qkv.data_ptr(), qkv.stride(0), out.data_ptr(),
            lse.data_ptr(), dqkv.data_ptr(), cu_seqlens.data_ptr(), cu_seqlens.numel() - 1, T, int(max_seqlen), n_groups,
            q_per_group, head_dim, scale, float(dropout_p), dropout_keys[0], dropout_keys[1], alibi_slopes.data_ptr(),
            ws.data_ptr(), _stream(),
        )
        return dqkv
    if dropout_p:
        _lib.call(
            "dolomite_b200_attn_varlen_bwd_dropout", dout.data_ptr(), qkv.data_ptr(), qkv.stride(0), out.data_ptr(),
            lse.data_ptr(), dqkv.data_ptr(), cu_seqlens.data_ptr(), cu_seqlens.numel() - 1, T, int(max_seqlen), n_groups,
            q_per_group, head_dim, scale, float(dropout_p), dropout_keys[0], dropout_keys[1], ws.data_ptr(), _stream(),
        )
        return dqkv
    _lib.call(
        "dolomite_b200_attn_varlen_bwd", dout.data_ptr(), qkv.data_ptr(), qkv.stride(0), out.data_ptr(), lse.data_ptr(),
        dqkv.data_ptr(), cu_seqlens.data_ptr(), cu_seqlens.numel() - 1, T, int(max_seqlen), n_groups, q_per_group,
        head_dim, scale, ws.data_ptr(), _stream(),
    )
    return dqkv


def attn_decode(qkv, k_cache, v_cache, lens, n_groups: int, q_per_group: int, head_dim: int, scale: float,
                alibi_slopes=None):
    """one new token per sequence against its KV cache: qkv [B, qkv_dim] (roped), caches [B, L_max, n_groups * head_dim], lens
    int32 [B] (valid positions including the new token) -> [B, n_heads * head_dim].  `alibi_slopes`: ALiBi bias of each
    cache position (see attn_varlen_fwd)"""
    _req(qkv, _BF16, "qkv"), _req(k_cache, _BF16, "k_cache"), _req(v_cache, _BF16, "v_cache"), _req(lens, torch.int32, "lens")
    B = qkv.shape[0]
    assert k_cache.shape == v_cache.shape and k_cache.shape[0] == B and k_cache.shape[2] == n_groups * head_dim
    assert k_cache.is_contiguous() and v_cache.is_contiguous() and qkv.stride(1) == 1
    out = torch.empty(B, n_groups * q_per_group * head_dim, dtype=_BF16, device=qkv.device)
    if alibi_slopes is not None:
        _req_slopes(alibi_slopes, n_groups * q_per_group)
        _lib.call("dolomite_b200_attn_decode_alibi", qkv.data_ptr(), qkv.stride(0), k_cache.data_ptr(), v_cache.data_ptr(),
                  lens.data_ptr(), out.data_ptr(), B, k_cache.shape[1], n_groups, q_per_group, head_dim, scale,
                  alibi_slopes.data_ptr(), _stream())
        return out
    _lib.call("dolomite_b200_attn_decode", qkv.data_ptr(), qkv.stride(0), k_cache.data_ptr(), v_cache.data_ptr(), lens.data_ptr(),
              out.data_ptr(), B, k_cache.shape[1], n_groups, q_per_group, head_dim, scale, _stream())
    return out


# ------------------------------------------------------------------------------------------------
# MoE: routing plan, grouped expert GEMMs (moe_dolomite/moe/scatter.py:18-138)
# ------------------------------------------------------------------------------------------------
class MoEPlan:
    """device-side routing state of one MoE layer invocation (no host sync anywhere)"""

    __slots__ = ("T", "E", "k", "max_rows", "sel_idx", "sel_w", "counts", "offsets", "tile_group", "cursors",
                 "row_of_slot", "slot_of_row", "token_of_row")


def moe_route(router_logits, k: int) -> MoEPlan:
    _req(router_logits, _BF16, "router_logits")
    T, E = router_logits.shape
    dev = router_logits.device
    p = MoEPlan()
    p.T, p.E, p.k = T, E, k
    p.max_rows = _lib.load().dolomite_b200_moe_max_rows(T, E, k)
    i32 = dict(dtype=torch.int32, device=dev)
    p.sel_idx = torch.empty(T, k, **i32)
    p.sel_w = torch.empty(T, k, dtype=torch.float32, device=dev)
    p.counts = torch.empty(E, **i32)
    p.offsets = torch.empty(E + 1, **i32)
    p.tile_group = torch.empty(p.max_rows // 128, **i32)
    p.cursors = torch.empty(E, **i32)
    p.row_of_slot = torch.empty(T * k, **i32)
    p.slot_of_row = torch.empty(p.max_rows, **i32)
    p.token_of_row = torch.empty(p.max_rows, **i32)
    _lib.call("dolomite_b200_moe_route", router_logits.data_ptr(), T, E, k, p.sel_idx.data_ptr(), p.sel_w.data_ptr(),
              p.counts.data_ptr(), p.offsets.data_ptr(), p.tile_group.data_ptr(), p.cursors.data_ptr(),
              p.row_of_slot.data_ptr(), p.slot_of_row.data_ptr(), p.token_of_row.data_ptr(), _stream())
    return p


def moe_gather(x, plan: MoEPlan):
    T, H = x.shape
    xg = torch.empty(plan.max_rows, H, dtype=_BF16, device=x.device)
    _lib.call("dolomite_b200_moe_gather", x.data_ptr(), xg.data_ptr(), plan.slot_of_row.data_ptr(), plan.offsets.data_ptr(),
              T, plan.E, plan.k, H, _stream())
    return xg


def moe_combine(yg, plan: MoEPlan, c=None, alpha: float = 1.0):
    H = yg.shape[1]
    out = torch.empty(plan.T, H, dtype=_BF16, device=yg.device)
    _lib.call("dolomite_b200_moe_combine", yg.data_ptr(), plan.row_of_slot.data_ptr(), plan.sel_w.data_ptr(), _ptr(c),
              out.data_ptr(), plan.T, plan.k, H, alpha, _stream())
    return out


def moe_combine_bwd(dy, yg, plan: MoEPlan, alpha: float = 1.0):
    H = yg.shape[1]
    dyg = torch.empty_like(yg)
    dw = torch.zeros(plan.T, plan.k, dtype=torch.float32, device=yg.device)
    _lib.call("dolomite_b200_moe_combine_bwd", dy.data_ptr(), yg.data_ptr(), plan.slot_of_row.data_ptr(),
              plan.offsets.data_ptr(), plan.sel_w.data_ptr(), dyg.data_ptr(), dw.data_ptr(), plan.T, plan.E, plan.k, H,
              alpha, _stream())
    return dyg, dw


def moe_token_sum(dxg, plan: MoEPlan):
    H = dxg.shape[1]
    dx = torch.empty(plan.T, H, dtype=_BF16, device=dxg.device)
    _lib.call("dolomite_b200_moe_token_sum", dxg.data_ptr(), plan.row_of_slot.data_ptr(), dx.data_ptr(), plan.T, plan.k, H, _stream())
    return dx


def moe_router_bwd(plan: MoEPlan, dw):
    dl = torch.empty(plan.T, plan.E, dtype=_BF16, device=dw.device)
    _lib.call("dolomite_b200_moe_router_bwd", plan.sel_idx.data_ptr(), plan.sel_w.data_ptr(), dw.data_ptr(), dl.data_ptr(),
              plan.T, plan.E, plan.k, _stream())
    return dl


# MoE load-balancing loss (moe_dolomite/base.py:24-43, transformers' Mixtral load_balancing_loss_func)
def moe_aux_acc(E: int, device) -> torch.Tensor:
    """cleared [2, E] fp32 accumulator of the load-balancing statistics of one forward: [sum of probabilities | counts]"""
    return torch.zeros(2, E, dtype=torch.float32, device=device)


def moe_aux_stats(router_logits, plan: MoEPlan, T_real: int, acc) -> None:
    """acc += this layer's statistics over its first T_real token rows (fixed summation order: bit-identical run to run)"""
    _req(router_logits, _BF16, "router_logits"), _req(acc, torch.float32, "acc")
    T, E = router_logits.shape
    assert router_logits.is_contiguous() and acc.is_contiguous() and acc.numel() == 2 * E and T == plan.T and E == plan.E
    n = _lib.load().dolomite_b200_moe_aux_partial_floats(T_real, E)
    partial = torch.empty(max(n, 1), dtype=torch.float32, device=acc.device)
    _lib.call("dolomite_b200_moe_aux_stats", router_logits.data_ptr(), plan.sel_idx.data_ptr(), T, T_real, E, plan.k,
              partial.data_ptr(), acc.data_ptr(), _stream())


def moe_aux_finalize(acc, n_tokens: int, coef: float = 0.0, loss=None):
    """-> (aux [1] fp32, backward coefficients c [E] fp32) of the statistics in `acc` over n_tokens = layers * real tokens;
    adds coef * aux into the fp32 device scalar `loss` when it is given.  No host sync."""
    _req(acc, torch.float32, "acc")
    E = acc.shape[-1]
    if loss is not None:
        _req(loss, torch.float32, "loss")
        assert loss.numel() == 1
    aux = torch.empty(1, dtype=torch.float32, device=acc.device)
    c = torch.empty(E, dtype=torch.float32, device=acc.device)
    _lib.call("dolomite_b200_moe_aux_finalize", acc.data_ptr(), E, int(n_tokens), float(coef), aux.data_ptr(), c.data_ptr(),
              _ptr(loss), _stream())
    return aux, c


def moe_router_bwd_aux(router_logits, plan: MoEPlan, dw, c, s, T_real: int):
    """moe_router_bwd + the load-balancing term s * p * (c - <p, c>) on the first T_real rows; s: fp32 device scalar"""
    _req(router_logits, _BF16, "router_logits"), _req(c, torch.float32, "c"), _req(s, torch.float32, "s")
    assert router_logits.is_contiguous() and tuple(router_logits.shape) == (plan.T, plan.E) and c.numel() == plan.E
    dl = torch.empty(plan.T, plan.E, dtype=_BF16, device=dw.device)
    _lib.call("dolomite_b200_moe_router_bwd_aux", router_logits.data_ptr(), plan.sel_idx.data_ptr(), plan.sel_w.data_ptr(),
              dw.data_ptr(), c.data_ptr(), s.data_ptr(), dl.data_ptr(), plan.T, T_real, plan.E, plan.k, _stream())
    return dl


def gemm_grouped_m(a, w3, plan: MoEPlan, *, b_mn: bool, alpha: float = 1.0, flags=None):
    """rows of `a` grouped by expert.  b_mn=False: w3 [E, N, K] -> D = A W[e]^T;  b_mn=True: w3 [E, K, N] -> D = A W[e]"""
    _req(a, _BF16, "a"), _req(w3, _BF16, "w3")
    rows, K = a.shape
    E = w3.shape[0]
    N = w3.shape[2] if b_mn else w3.shape[1]
    assert (w3.shape[1] if b_mn else w3.shape[2]) == K and rows == plan.max_rows and w3.is_contiguous()
    out = torch.empty(rows, N, dtype=_BF16, device=a.device)
    if flags is None:
        flags = _default_gemm_flags
    _lib.call("dolomite_b200_gemm_bf16_grouped_m", a.data_ptr(), a.stride(0), w3.data_ptr(), w3.shape[2], int(b_mn),
              out.data_ptr(), N, alpha, rows, N, K, plan.tile_group.data_ptr(), E, flags, _stream())
    return out


def gemm_grouped_m_gather(x, w3, plan: MoEPlan, alpha: float = 1.0, flags=None):
    """expert forward with the gather fused into the operand load (rows copied by the producer warp): x [T, K] UNGROUPED, w3 [E, N, K] ->
    D[row] = x[token_of_row[row]] W[expert(row)]^T for every grouped row (moe/scatter.py:38-49 `parallel_linear`)"""
    _req(x, _BF16, "x"), _req(w3, _BF16, "w3")
    T, K = x.shape
    E, N = w3.shape[0], w3.shape[1]
    assert w3.shape[2] == K and w3.is_contiguous() and x.stride(1) == 1 and T == plan.T
    out = torch.empty(plan.max_rows, N, dtype=_BF16, device=x.device)
    if flags is None:
        flags = _default_gemm_flags
    if gemm_timer is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    _lib.call("dolomite_b200_gemm_bf16_grouped_m_gather", x.data_ptr(), x.stride(0), T, plan.token_of_row.data_ptr(),
              w3.data_ptr(), w3.shape[2], out.data_ptr(), N, alpha, plan.max_rows, N, K, plan.tile_group.data_ptr(), E, flags,
              _stream())
    if gemm_timer is not None:
        e1.record()
        gemm_timer.append((2.0 * T * plan.k * N * K, e0, e1))
    return out


def gemm_grouped_k(a, b, plan: MoEPlan, out3, alpha: float = 1.0, beta: float = 1.0):
    """expert wgrad: out3[e] (+)= a[rows_e]^T b[rows_e]; a [rows, M], b [rows, N], out3 fp32 [E, M, N]"""
    _req(a, _BF16, "a"), _req(b, _BF16, "b"), _req(out3, torch.float32, "out3")
    rows, M = a.shape
    N = b.shape[1]
    assert out3.shape == (plan.E, M, N) and out3.is_contiguous()
    _lib.call("dolomite_b200_gemm_bf16_grouped_k", a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), out3.data_ptr(), N,
              alpha, beta, M, N, rows, plan.offsets.data_ptr(), plan.E, _stream())
    return out3
