"""NEFTune noise restated in numpy, bit for bit with csrc/elementwise.cu `embedding_fwd_neft_kernel`, and the oracle's
forward with that noise on wte(ids) (model_wrapper/base.py:246-267: `x + zeros_like(x).uniform_(-mag, mag)` in training mode).

The reference draws u from torch's Philox stream, which no independent kernel reproduces; what is restated is the
distribution (u uniform on (0, 1], 2^24 equally likely values) and torch's rounding points for a bf16 tensor
(ATen/native/cuda/DistributionTemplates.h `uniform_kernel`): from = bf16(-mag), to = bf16(mag), range = bf16(to - from),
v = bf16(fp32(fp32(u * range) + from)), v == to -> from, out = bf16(x + v).

Keys: `oracle.dolomite_oracle.DropoutOracle(pass seed).keys(NEFT_SITE)`.  Dropout sites are 0 and 4 i + 1 .. 4 i + 3; the
noise uses site -1 (DolomiteEngine.NEFT_SITE), which no dropout site uses."""

from __future__ import annotations

import numpy as np
import torch

import oracle.dolomite_oracle as O

NEFT_SITE = -1
_U32 = np.uint32


def _bf16(x: np.ndarray) -> np.ndarray:
    """round fp32 to bf16 (nearest even) and back"""
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).float().numpy()


def bounds(mag: float) -> tuple[np.float32, np.float32, np.float32]:
    frm = _bf16(np.array([-mag], dtype=np.float32))[0]
    to = _bf16(np.array([mag], dtype=np.float32))[0]
    rng = _bf16(np.array([to - frm], dtype=np.float32))[0]
    return np.float32(frm), np.float32(to), np.float32(rng)


def uniform_u(keys: tuple[int, int], n: int, start: int = 0) -> np.ndarray:
    """u of flat elements start .. start + n - 1: ((h >> 8) + 1) * 2^-24, h = dropout_hash_flat(e, key0, key1)"""
    k0, k1 = keys
    with np.errstate(over="ignore"):
        e = np.arange(start, start + n, dtype=np.uint64)
        h = O._lowbias32(O._lowbias32((e & np.uint64(0xFFFFFFFF)).astype(_U32) ^ _U32(k0))
                         + (e >> np.uint64(32)).astype(_U32) + _U32(k1))
    return ((h >> _U32(8)) + _U32(1)).astype(np.float32) * np.float32(2.0 ** -24)


def noise(keys: tuple[int, int], n: int, mag: float, start: int = 0) -> np.ndarray:
    """the bf16-valued noise v (as fp32) of n flat elements"""
    frm, to, rng = bounds(mag)
    u = uniform_u(keys, n, start)
    v = _bf16((u * rng).astype(np.float32) + frm)
    return np.where(v == to, frm, v).astype(np.float32)


def embed(wte_bf16: torch.Tensor, ids: torch.Tensor, keys: tuple[int, int], mag: float) -> torch.Tensor:
    """bf16 [T, H] = bf16(wte[ids] + v)"""
    x = wte_bf16[ids.long().cpu()].float()
    v = torch.from_numpy(noise(keys, x.numel(), mag)).view_as(x)
    return (x + v).to(torch.bfloat16)


def forward_logits(p: dict, cfg: O.OracleConfig, input_ids, position_ids, cu_seqlens, v: torch.Tensor | None,
                   bf16: bool = True) -> torch.Tensor:
    """O.forward_logits with the noise v [T, H] added to wte(ids) (one bf16 rounding), before `+ wpe`, dropout and m_emb"""
    if bf16:
        p = {k: O._r(t, True) for k, t in p.items()}
    ids = torch.as_tensor(np.asarray(input_ids), dtype=torch.long)
    pos = torch.as_tensor(np.asarray(position_ids), dtype=torch.long)
    h = p["transformer.wte.weight"][ids]
    if v is not None:
        h = O._r(h + v, bf16)
    if cfg.position_embedding_type == "learned_absolute":
        h = O._r(h + p["transformer.wpe.weight"][pos], bf16)
    h = O._drop(h, 0, cfg.embd_pdrop, bf16)
    if cfg.m_emb is not None:
        h = O._r(h * cfg.m_emb, bf16)
    cos = sin = None
    if cfg.position_embedding_type == "rope":
        ct, st = O.rope_tables(cfg.head_dim, cfg.n_positions, cfg.rope_theta, bf16, cfg.rope_scaling)
        cos, sin = ct[pos].unsqueeze(1), st[pos].unsqueeze(1)
    for i in range(cfg.n_layer):
        h = O.block(h, p, i, cfg, cos, sin, cu_seqlens, bf16)
    h = O.norm(h, p, "transformer.ln_f.", cfg, bf16)
    head = p["transformer.wte.weight"] if cfg.tie_word_embeddings else p["lm_head.weight"]
    logits = O.linear(h, head, None, bf16)
    if cfg.m_width is not None:
        logits = O._r(logits / cfg.m_width, bf16)
    return logits
