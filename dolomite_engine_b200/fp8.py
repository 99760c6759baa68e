"""FP8 training of the linear layers with delayed scaling (`mixed_precision_args: {dtype: fp8, fp8_backend: nvte}`).

Restates what the reference gets from TransformerEngine (distributed/fp8/nv_te.py:15-42 swaps nn.Linear for te.Linear;
pretrain.py:126-134 / finetune.py:90-98 wrap the training forward in te.fp8_autocast with
DelayedScaling(fp8_format=Format.HYBRID, amax_history_len=16, amax_compute_algo="max")).  TransformerEngine itself is not a
dependency: the arithmetic below follows TE 1.x and is not pinned by a test against TE.

Every FP8 linear owns three tensor slots -- its input and weight (e4m3, forward) and its output gradient (e5m2, backward).
Each slot has an amax history [16] (row 0 = current step), a scale and a scale_inv, kept as flat fp32 device tensors:
    fwd_history [16, 2 n] (slot 2 i = input of linear i, 2 i + 1 = its weight), fwd_scale / fwd_scale_inv [2 n]
    bwd_history [16, n], bwd_scale / bwd_scale_inv [n]
The casts fold max|x| into row 0 of their slot; `update()` turns the history into new scales on the device (one launch per
format, kernels.fp8_scaling_update) -- no host synchronisation anywhere.
"""

from __future__ import annotations

from contextlib import contextmanager, nullcontext

import torch

from . import kernels as K

AMAX_HISTORY_LEN = 16


def fp8_weight_names(cfg) -> list[str]:
    """Reference parameter names of the linears that run in FP8: the nn.Linear / ParameterizedLinear modules whose weight
    dimensions are all multiples of 16 (nv_te.py:15-42).  MoE experts (ParameterizedExperts) are not nn.Linear, and a tied
    LM head is F.linear on wte: both stay BF16.  The MoE router gate is included when its shape allows."""
    H, F = cfg.n_embd, cfg.n_inner
    hd = cfg.n_embd // cfg.n_head
    qkv = H + 2 * cfg.num_key_value_heads * hd
    glu = cfg.activation_function.endswith("glu")
    E = getattr(cfg, "num_experts", 0) if cfg.model_type == "moe_dolomite" else 0
    names = []
    for i in range(cfg.n_layer):
        p = f"transformer.h.{i}."
        shapes = [("attn.c_attn.weight", (qkv, H)), ("attn.c_proj.weight", (H, H))]
        if E:
            shapes.append(("mlp.gate.weight", (E, H)))
        else:
            shapes += [("mlp.c_fc.weight", (2 * F if glu else F, H)), ("mlp.c_proj.weight", (H, F))]
        names += [p + n for n, shape in shapes if all(d % 16 == 0 for d in shape)]
    if not cfg.tie_word_embeddings and cfg.vocab_size % 16 == 0 and H % 16 == 0:
        names.append("lm_head.weight")
    return names


class Fp8Recipe:
    """DelayedScaling state of every FP8 linear of a model (see the module docstring for the layout)."""

    def __init__(self, weight_names: list[str], device, history_len: int = AMAX_HISTORY_LEN):
        self.names = list(weight_names)
        self.index = {n: i for i, n in enumerate(self.names)}
        n = len(self.names)
        f32 = dict(dtype=torch.float32, device=device)
        self.fwd_history = torch.zeros(history_len, 2 * n, **f32)
        self.fwd_scale = torch.ones(2 * n, **f32)
        self.fwd_scale_inv = torch.ones(2 * n, **f32)
        self.bwd_history = torch.zeros(history_len, n, **f32)
        self.bwd_scale = torch.ones(n, **f32)
        self.bwd_scale_inv = torch.ones(n, **f32)

    def __contains__(self, name: str) -> bool:
        return name in self.index

    def input_slot(self, name: str):
        """(scale, scale_inv, amax) 1-element views of the input slot of linear `name`"""
        j = 2 * self.index[name]
        return self.fwd_scale[j : j + 1], self.fwd_scale_inv[j : j + 1], self.fwd_history[0, j : j + 1]

    def weight_slot(self, name: str):
        j = 2 * self.index[name] + 1
        return self.fwd_scale[j : j + 1], self.fwd_scale_inv[j : j + 1], self.fwd_history[0, j : j + 1]

    def grad_slot(self, name: str):
        j = self.index[name]
        return self.bwd_scale[j : j + 1], self.bwd_scale_inv[j : j + 1], self.bwd_history[0, j : j + 1]

    def update(self, all_reduce: bool = False) -> None:
        """End of a micro-step: new scales of every slot from its amax history.  `all_reduce`: the current amaxes are first
        all-reduced (MAX) over the default group, as TE does, so that every rank holds identical scales (every rank of the
        default group must call update)."""
        if all_reduce:
            row0 = torch.cat([self.fwd_history[0], self.bwd_history[0]])
            torch.distributed.all_reduce(row0, op=torch.distributed.ReduceOp.MAX)
            n2 = self.fwd_history.shape[1]
            self.fwd_history[0].copy_(row0[:n2])
            self.bwd_history[0].copy_(row0[n2:])
        if self.names:
            K.fp8_scaling_update(self.fwd_history, self.fwd_scale, self.fwd_scale_inv, K.E4M3)
            K.fp8_scaling_update(self.bwd_history, self.bwd_scale, self.bwd_scale_inv, K.E5M2)

    _KEYS = ("fwd_history", "fwd_scale", "fwd_scale_inv", "bwd_history", "bwd_scale", "bwd_scale_inv")

    def state_dict(self) -> dict:
        out = {k: getattr(self, k).detach().cpu().clone() for k in self._KEYS}
        out["names"] = list(self.names)
        return out

    def load_state_dict(self, sd: dict) -> None:
        if list(sd["names"]) != self.names:
            raise ValueError("FP8 recipe state was saved for a different set of FP8 linears")
        for k in self._KEYS:
            dst = getattr(self, k)
            if tuple(sd[k].shape) != tuple(dst.shape):
                raise ValueError(f"FP8 recipe state {k}: shape {tuple(sd[k].shape)} vs {tuple(dst.shape)}")
            dst.copy_(sd[k])


@contextmanager
def fp8_autocast(engine):
    """te.fp8_autocast around a training forward: the FP8 linears of `engine` run in FP8 inside"""
    prev = engine.fp8_autocast
    engine.fp8_autocast = True
    try:
        yield
    finally:
        engine.fp8_autocast = prev


def setup_training(args, model):
    """mixed_precision_args dtype fp8 (backend nvte): enables the FP8 linears of the model's engine and returns the
    forward context of train_step (pretrain.py:126-134 / finetune.py:90-98); otherwise returns nullcontext"""
    if args.mixed_precision_args.dtype != "fp8":
        return nullcontext
    engine = model.engine if hasattr(model, "engine") else model.model.engine
    engine.enable_fp8()
    return lambda: fp8_autocast(engine)
