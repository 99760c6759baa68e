"""Training engine of the B200 path: flat parameter units + explicit forward/backward over the C-ABI kernels.

Replaces, for the padding-free GPTDolomite / MoEDolomite step, what the reference gets from autograd over
`GPTDolomiteModel.forward` (gpt_dolomite/base.py:170-244), `GPTDolomiteBlock.forward` (layer.py:49-87),
`PaddingFreeAttention.forward` (attention/padding_free.py:15-77), `MLP.forward` (mlp.py:45-50) and the tied LM head
(main.py:172-177), and what torch FSDP does around it (distributed/__init__.py:126-230).

Data layout in HBM
  * one FlatUnit per FSDP unit (root = wte [+wpe] + ln_f [+lm_head]; one per transformer block), mirroring
    `_no_split_modules` wrapping.  Per unit: fp32 master shard (the nn.Parameter the optimizer sees), fp32 gradient
    shard, a full bf16 compute buffer (what the all-gather fills and the kernels read) and a full fp32 gradient
    accumulation buffer that the wgrad GEMM epilogues add into (what the reduce-scatter consumes).
  * activations are [T, features] bf16 row-major; attention reads q/k/v straight out of the packed c_attn output.
No op here has a PyTorch fallback: without the CUDA library every call raises.
"""

from __future__ import annotations

import math
import os
from dataclasses import dataclass
from typing import TYPE_CHECKING

import torch

from . import kernels as K
from .activations import resolve as resolve_activation

if TYPE_CHECKING:  # the config module lives in hf_models, which imports this module
    from .hf_models.config import CommonConfig

_ALIGN = 64  # elements; keeps every parameter 128-byte aligned inside a flat unit (TMA needs 16 B)


@dataclass
class ParamSpec:
    name: str  # reference state-dict name
    shape: tuple
    offset: int
    numel: int
    init: str  # "normal:<std>" | "ones" | "zeros"


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class FlatUnit:
    """One FSDP unit: contiguous flat buffers + named views (reference parameter names)."""

    def __init__(self, name: str, specs: list[tuple[str, tuple, str]], world_size: int = 1, rank: int = 0):
        self.name = name
        self.specs: list[ParamSpec] = []
        off = 0
        for pname, shape, init in specs:
            n = math.prod(shape)
            self.specs.append(ParamSpec(pname, tuple(shape), off, n, init))
            off += _round_up(n, _ALIGN)
        self.numel = off
        self.world_size = world_size
        self.rank = rank
        self.padded = _round_up(max(off, 1), world_size * _ALIGN)
        self.shard_numel = self.padded // world_size
        self.master: torch.nn.Parameter | None = None  # fp32 [shard_numel]
        self.compute: torch.Tensor | None = None  # bf16 [padded]
        self.grad_full: torch.Tensor | None = None  # fp32 [padded]
        self.views: dict[str, torch.Tensor] = {}
        self.gviews: dict[str, torch.Tensor] = {}
        self.gathered = False  # compute buffer holds current parameters
        self.pooled = False  # compute / grad_full are shared with other units (stage-3 resharding)
        self.exp_avg = None
        self.exp_avg_sq = None

    # ---- allocation / init ----
    def allocate(self, device) -> None:
        self.master = torch.nn.Parameter(torch.zeros(self.shard_numel, dtype=torch.float32, device=device))
        self.master.grad = torch.zeros(self.shard_numel, dtype=torch.float32, device=device)
        self.compute = torch.zeros(self.padded, dtype=torch.bfloat16, device=device)
        if self.world_size == 1:
            self.grad_full = self.master.grad  # no reduce-scatter: wgrad accumulates straight into the shard grad
        else:
            self.grad_full = torch.zeros(self.padded, dtype=torch.float32, device=device)
        for s in self.specs:
            self.views[s.name] = self.compute[s.offset : s.offset + s.numel].view(s.shape)
            self.gviews[s.name] = self.grad_full[s.offset : s.offset + s.numel].view(s.shape)

    def bind_pooled(self, compute: torch.Tensor, grad_full: torch.Tensor) -> None:
        """stage-3 resharding: the gathered bf16 parameters and the full fp32 gradients of this unit live in a buffer that
        several units take turns using (distributed._Comm decides who owns it when); only the shards stay per unit"""
        assert compute.numel() == self.padded and grad_full.numel() == self.padded
        self.compute, self.grad_full = compute, grad_full
        self.pooled = True
        self.gathered = False
        for s in self.specs:
            self.views[s.name] = compute[s.offset : s.offset + s.numel].view(s.shape)
            self.gviews[s.name] = grad_full[s.offset : s.offset + s.numel].view(s.shape)

    def full_master_from(self, full_fp32: torch.Tensor) -> None:
        """install parameters from a full flat fp32 tensor (host or device)"""
        lo = self.rank * self.shard_numel
        with torch.no_grad():
            self.master.copy_(full_fp32[lo : lo + self.shard_numel])
            if not self.pooled:
                self.compute.copy_(full_fp32.to(self.compute.device))
        self.gathered = not self.pooled

    def init_full(self, generator: torch.Generator) -> torch.Tensor:
        """reference init rules (SURVEY section 8 a19) in fp32; every rank draws the same values (same seed, same
        generator device).  CPU generator = reproducible against the oracle; CUDA generator = fast for big models."""
        full = torch.zeros(self.padded, dtype=torch.float32, device=generator.device)
        for s in self.specs:
            v = full[s.offset : s.offset + s.numel].view(s.shape)
            if s.init == "ones":
                v.fill_(1.0)
            elif s.init == "zeros":
                v.zero_()
            else:
                std = float(s.init.split(":")[1])
                v.copy_(torch.randn(s.shape, generator=generator, device=generator.device) * std)
        return full


class KVCache:
    """keys / values of every layer by position: k[l], v[l] bf16 [batch, max_len, n_kv_groups * head_dim]; lens int32 [batch]"""

    def __init__(self, engine: "DolomiteEngine", batch: int, max_len: int):
        dim = engine.n_groups * engine.hd
        mk = lambda: torch.zeros(batch, max_len, dim, dtype=torch.bfloat16, device=engine.device)  # noqa: E731
        self.k = [mk() for _ in range(engine.cfg.n_layer)]
        self.v = [mk() for _ in range(engine.cfg.n_layer)]
        self.lens = torch.zeros(batch, dtype=torch.int32, device=engine.device)
        self.max_len = max_len


def _block_specs(cfg: CommonConfig, i: int) -> list[tuple[str, tuple, str]]:
    """parameters of GPTDolomiteBlock i in registration order (layer.py:33-47, attention/base.py:73-86, mlp.py:26-41)"""
    H, F = cfg.n_embd, cfg.n_inner
    hd = cfg.n_embd // cfg.n_head
    qkv = H + 2 * cfg.num_key_value_heads * hd
    std = cfg.initializer_range
    if cfg.init_method == "mup":
        std /= math.sqrt(cfg.m_width)
    std_proj = cfg.initializer_range / math.sqrt(2 * cfg.n_layer)
    if cfg.init_method == "mup":
        std_proj /= math.sqrt(cfg.m_width)
    glu = cfg.activation_function.endswith("glu")
    fc_out = 2 * F if glu else F
    p = f"transformer.h.{i}."
    specs = [(p + "ln_1.weight", (H,), "ones"), (p + "attn.c_attn.weight", (qkv, H), f"normal:{std}")]
    if cfg.add_bias:
        specs.append((p + "attn.c_attn.bias", (qkv,), "zeros"))
    specs.append((p + "attn.c_proj.weight", (H, H), f"normal:{std_proj}"))
    if cfg.add_bias:
        specs.append((p + "attn.c_proj.bias", (H,), "zeros"))
    specs.append((p + "ln_2.weight", (H,), "ones"))
    E = getattr(cfg, "num_experts", 0) if cfg.model_type == "moe_dolomite" else 0
    if E:
        specs.append((p + "mlp.gate.weight", (E, H), f"normal:{std}"))
        specs.append((p + "mlp.c_fc.weight", (E, fc_out, H), f"normal:{std}"))
        if cfg.add_bias:
            specs.append((p + "mlp.c_fc.bias", (E, fc_out), "zeros"))
        specs.append((p + "mlp.c_proj.weight", (E, H, F), f"normal:{std_proj}"))
        if cfg.add_bias:
            specs.append((p + "mlp.c_proj.bias", (E, H), "zeros"))
    else:
        specs.append((p + "mlp.c_fc.weight", (fc_out, H), f"normal:{std}"))
        if cfg.add_bias:
            specs.append((p + "mlp.c_fc.bias", (fc_out,), "zeros"))
        specs.append((p + "mlp.c_proj.weight", (H, F), f"normal:{std_proj}"))
        if cfg.add_bias:
            specs.append((p + "mlp.c_proj.bias", (H,), "zeros"))
    if cfg.normalization_function == "layernorm":  # torch.nn.LayerNorm always carries a bias
        specs.append((p + "ln_1.bias", (H,), "zeros"))
        specs.append((p + "ln_2.bias", (H,), "zeros"))
    return specs


def _root_specs(cfg: CommonConfig) -> list[tuple[str, tuple, str]]:
    H, V = cfg.n_embd, cfg.vocab_size
    specs = [("transformer.wte.weight", (V, H), f"normal:{cfg.initializer_range}")]
    specs.append(("transformer.ln_f.weight", (H,), "ones"))
    if not cfg.tie_word_embeddings:
        # gpt_dolomite/main.py:19-21: ParameterizedLinear(..., std=initializer_range) -- no muP width scaling on the head
        specs.append(("lm_head.weight", (V, H), f"normal:{cfg.initializer_range}"))
    # appended last: the random stream (and flat layout) of every rope / rmsnorm configuration stays what it was
    if cfg.normalization_function == "layernorm":
        specs.append(("transformer.ln_f.bias", (H,), "zeros"))
    if cfg.position_embedding_type == "learned_absolute":  # ParameterizedEmbedding(n_positions, n_embd), base.py:127-134
        specs.append(("transformer.wpe.weight", (cfg.n_positions, H), f"normal:{cfg.initializer_range}"))
    return specs


def check_supported(cfg: CommonConfig, *, attention_implementation: str = "flash_attention_2",
                    use_padding_free_transformer: bool = True) -> None:
    """The B200 hot path implements the configurations SURVEY.md section 8 puts in scope; everything else raises
    (mirrors the reference's NotImplementedError / ValueError conventions, SURVEY section 8b).  The keyword arguments are
    the model's `attn_implementation` / `use_padding_free_transformer`; only alibi depends on them."""
    if cfg.position_embedding_type not in ("rope", "nope", "learned_absolute", "alibi"):
        raise NotImplementedError(
            f"position_embedding_type={cfg.position_embedding_type!r}: the B200 path implements rope, nope, "
            "learned_absolute and alibi"
        )
    if cfg.position_embedding_type == "alibi" and (
        attention_implementation == "flash_attention_2" or use_padding_free_transformer
    ):
        # gpt_dolomite/base.py:529-530 asserts the same for flash attention; the padding-free transformer needs flash
        raise NotImplementedError(
            "position_embedding_type='alibi' runs with attn_implementation 'eager' or 'sdpa' and "
            "use_padding_free_transformer=False (the reference: alibi is not implemented with flash attention, "
            "gpt_dolomite/base.py:530)"
        )
    if cfg.rope_scaling is not None:
        rs = cfg.rope_scaling
        if not isinstance(rs, dict) or "factor" not in rs or "original_max_position_embeddings" not in rs:
            raise ValueError("rope_scaling needs `factor` and `original_max_position_embeddings` (YaRN, gpt_dolomite/base.py:541-547)")
        if rs.get("type", "yarn") not in ("yarn",):
            raise NotImplementedError(f"rope_scaling type {rs.get('type')!r}: the reference implements YaRN only")
    if cfg.normalization_function not in ("rmsnorm", "layernorm"):
        raise NotImplementedError(
            f"normalization_function={cfg.normalization_function!r}: rmsnorm and layernorm are implemented in CUDA")
    resolve_activation(cfg.activation_function)  # ValueError / NotImplementedError as the reference's lookup
    if cfg.model_type == "moe_dolomite" and cfg.normalization_function != "rmsnorm":
        raise NotImplementedError("MoE blocks are implemented with rmsnorm (the MoEDolomite / Granite-MoE shape)")
    # dropout > 0: identity in eval mode; in training mode the residual / embedding dropouts are elementwise kernels
    # (csrc/dropout.cu) and the attention-probability dropout lives inside the attention kernels
    hd = cfg.n_embd // cfg.n_head
    if hd not in (16, 32, 64, 80, 96, 128):
        raise NotImplementedError(f"head_dim={hd}: supported head dims are 16, 32, 64, 80, 96, 128")
    if cfg.model_type == "moe_dolomite":
        if cfg.num_experts % 8 or not (1 <= cfg.num_experts_per_tok <= min(8, cfg.num_experts)):
            raise NotImplementedError("MoE: num_experts must be a multiple of 8 (<= 256) and 1 <= top-k <= 8")
        if cfg.add_bias:
            raise NotImplementedError("MoE experts with bias are not supported (ScatterMoE asserts the same, moe/scatter.py:22)")
        if cfg.n_inner % 64 or cfg.n_embd % 64:
            raise NotImplementedError("MoE: n_embd and n_inner must be multiples of 64 (grouped GEMM K tiles)")
    # vocab_size may be any value: [T, V] logits live in buffers with 16-byte row strides (kernels.rows_empty)
    if cfg.n_embd % 8 or cfg.n_inner % 8:
        raise NotImplementedError("n_embd and n_inner must be multiples of 8 (16-byte vector kernels / TMA)")


class DolomiteEngine:
    """Owns the flat units of one model replica/shard and runs the explicit forward / backward."""

    def __init__(self, cfg: CommonConfig, device, world_size: int = 1, rank: int = 0, seed: int | None = 42,
                 init_on_device: bool = False, attention_implementation: str = "flash_attention_2",
                 use_padding_free_transformer: bool = True):
        check_supported(cfg, attention_implementation=attention_implementation,
                        use_padding_free_transformer=use_padding_free_transformer)
        self.cfg = cfg
        self.device = torch.device(device)
        self.world_size, self.rank = world_size, rank
        self.hd = cfg.n_embd // cfg.n_head
        self.n_groups = cfg.num_key_value_heads
        self.q_per_group = cfg.n_head // cfg.num_key_value_heads
        self.qkv_dim = cfg.n_embd + 2 * cfg.num_key_value_heads * self.hd
        self.is_moe = cfg.model_type == "moe_dolomite"
        self.is_glu = cfg.activation_function.endswith("glu")
        self.act = resolve_activation(cfg.activation_function)  # (CUDA function id, form) of the MLP activation
        self.is_layernorm = cfg.normalization_function == "layernorm"
        self.learned_positions = cfg.position_embedding_type == "learned_absolute"
        self.has_dropout = bool(cfg.resid_pdrop or cfg.embd_pdrop or cfg.attn_pdrop)
        self.training = True  # mirrors nn.Module.training of the owning model (DolomitePreTrainedModel.train)
        # Dropout masks are counter-based (kernels.dropout_keys): seed of the pass = dropout_seed + passes so far; backward
        # and re-computed (checkpointed) blocks regenerate the masks of their forward from the seed kept in `_saved`.
        self.dropout_seed: int | None = None  # None: torch.initial_seed() mixed with the rank on first use
        self._dropout_passes = 0
        self._dropout_now: int | None = None  # seed of the pass being run / backpropagated; None = no dropout (eval)
        self.units: list[FlatUnit] = [FlatUnit("root", _root_specs(cfg), world_size, rank)]
        for i in range(cfg.n_layer):
            self.units.append(FlatUnit(f"h.{i}", _block_specs(cfg, i), world_size, rank))
        for u in self.units:
            u.allocate(self.device)
        if seed is not None:
            g = torch.Generator(device=self.device if init_on_device else "cpu").manual_seed(seed)
            for u in self.units:
                u.full_master_from(u.init_full(g))
        self._setup_rope()
        # ALiBi: the slopes stay on the device (a non-persistent buffer in the reference: not part of the state dict).
        # Whether a pass applies the bias is decided per forward (`alibi=`), as the reference decides per call
        # (gpt_dolomite/base.py:559-598); backward and recomputed blocks reuse the decision of their forward.
        self.alibi_slopes = None
        if cfg.position_embedding_type == "alibi":
            from .alibi import alibi_slopes

            self.alibi_slopes = alibi_slopes(cfg.n_head).to(self.device)
        self._alibi_now = None  # slopes of the pass being run / backpropagated; None = no bias
        self.comm = None  # set by distributed.ShardedDataParallel
        self._saved = None
        self.requires_gradient_sync = True
        self.checkpoint_every: int | None = None  # block activation checkpointing: re-run blocks 0, k, 2k, ... in backward
        self.head_chunk_bytes = 1 << 30  # bf16 logits of one LM-head chunk (forward(fuse_head_loss=True))
        self.batch_block_wgrads = True  # the four weight gradients of a dense block in one persistent launch
        self._deferred_wgrads: list | None = None  # list while a block's backward collects its weight gradients
        # Weight gradients on a second stream: nothing in a block's backward chain waits for them, so the launch of block i
        # runs next to block i - 1's chain -- whose HBM-bound kernels (SwiGLU / norm / RoPE backward, column sums) fit on the SMs
        # NEXT TO a GEMM CTA (it leaves 1.5 KB of shared memory, 39 K registers and 1800 thread slots free) and hide behind it.
        self.overlap_wgrads = os.environ.get("DOLO_OVERLAP_WGRADS", "0") == "1"
        self._wgrad_stream = None  # created on first use
        self._kv_sink = None  # callable(layer, packed qkv) while a forward fills a KV cache (prefill)
        self._fresh_grads: set[str] = set()  # weights whose gradient buffer will be overwritten by the next wgrad GEMM
        # DOLO_EAGER_GRAD_ZERO=1: zero_grad() clears every gradient buffer (A/B switch for the lazy clearing, `_lazy_zero`)
        self.lazy_grad_zero = os.environ.get("DOLO_EAGER_GRAD_ZERO", "0") != "1"
        # FP8 linears (fp8.py): `fp8` holds the delayed-scaling state once enable_fp8() ran; `fp8_autocast` is switched on
        # around the training forward (te.fp8_autocast); `_fp8_now` is the mode of the pass being run or backpropagated
        self.fp8 = None
        self.fp8_autocast = False
        self._fp8_now = False
        # fp8 copies of the weights named in `_fp8_keep` ((name, transposed) -> uint8 tensor), kept for the current pass: the
        # scale is fixed for the step, so the LM head's chunk loop casts its [V, H] weight once, not once per chunk (other
        # weights are cast once per pass anyway and are not kept, which would hold an fp8 copy of the whole model)
        self._fp8_wcache: dict = {}
        self._fp8_keep: set = set()
        # MoE load-balancing loss (forward(router_aux=True)): `_aux_fwd` = (accumulator [2, E], T_real, router logits list)
        # while a forward collects the statistics -- never while backward re-runs a checkpointed block; `_aux_bwd` =
        # (c [E], s [1], T_real) while its backward runs
        self._aux_fwd = None
        self._aux_bwd = None
        if cfg.attention_multiplier is not None:
            self.softmax_scale = float(cfg.attention_multiplier)
        elif cfg.scale_attn_weights:
            self.softmax_scale = 1.0 / math.sqrt(self.hd)
        else:
            self.softmax_scale = 1.0

    def enable_fp8(self) -> None:
        """FP8 training of the linears fp8.fp8_weight_names(cfg) selects (mixed_precision_args dtype fp8, backend nvte)"""
        from .fp8 import Fp8Recipe, fp8_weight_names

        self.fp8 = Fp8Recipe(fp8_weight_names(self.cfg), self.device)

    def _is_fp8(self, wname: str) -> bool:
        return self._fp8_now and wname in self.fp8

    # ------------------------------------------------------------------------------------------
    def _ensure_rope(self, max_seqlen: int) -> None:
        """RoPE.forward regrows its cache when seq_len > max_seq_len_cached (position_embedding/rope.py:26-27, called with
        key_length = max_seqlen, gpt_dolomite/base.py:536-557); the kernel indexes the tables by position id, so they must
        cover the longest document of the batch (host-side check on a python int: no device sync)."""
        if self.rope_cos is not None and max_seqlen > self.rope_cos.shape[0]:
            self._setup_rope(n_positions=int(max_seqlen))

    def _setup_rope(self, n_positions: int | None = None) -> None:
        """cos/sin cache exactly as RoPE._set_cos_sin_cache (position_embedding/rope.py:36-55) then .to(bf16) (:29-30)"""
        self.rope_cos = self.rope_sin = None
        if self.cfg.position_embedding_type != "rope":
            return
        hd = self.hd
        base = float(self.cfg.rope_theta)
        mscale = 1.0
        rs = self.cfg.rope_scaling
        if rs is None:
            inv_freq = 1.0 / (base ** (torch.arange(0, hd, 2, dtype=torch.float32) / hd))
        else:
            # YaRNScaledRoPE (rope.py:56-101, :118-145; constructed in gpt_dolomite/base.py:534-547 with the class
            # defaults extrapolation_factor = attn_factor = 1, beta_fast = 32, beta_slow = 1): only the tables change
            scale, orig = float(rs["factor"]), int(rs["original_max_position_embeddings"])

            def correction_dim(num_rotations: float) -> float:
                return (hd * math.log(orig / (num_rotations * 2 * math.pi))) / (2 * math.log(base))

            pos_freqs = base ** (torch.arange(0, hd, 2).float() / hd)
            low = max(math.floor(correction_dim(32)), 0)
            high = min(math.ceil(correction_dim(1)), hd - 1)
            hi = high + 0.001 if low == high else high
            ramp = torch.clamp((torch.arange(hd // 2, dtype=torch.float32) - low) / (hi - low), 0, 1)
            mask = 1 - ramp
            inv_freq = (1.0 / (scale * pos_freqs)) * (1 - mask) + (1.0 / pos_freqs) * mask
            mscale = 1.0 if scale <= 1 else 0.1 * math.log(scale) + 1.0
        t = torch.arange(self.cfg.n_positions if n_positions is None else n_positions, dtype=torch.float32)
        freqs = torch.outer(t, inv_freq)
        emb = torch.cat((freqs, freqs), dim=-1)
        self.rope_cos = (emb.cos() * mscale).to(torch.bfloat16).to(self.device)
        self.rope_sin = (emb.sin() * mscale).to(torch.bfloat16).to(self.device)

    def named_views(self):
        for u in self.units:
            for s in u.specs:
                yield s.name, u, s

    def num_parameters(self) -> int:
        return sum(s.numel for u in self.units for s in u.specs)

    def convert_to_pooled(self, n_slots: int = 2) -> None:
        """Stage-3 memory layout (reference: FSDP FULL_SHARD, distributed/__init__.py:161-176 and :205-213): the block units
        stop owning a full bf16 parameter buffer and a full fp32 gradient buffer each; `n_slots` buffers of each kind are
        shared round-robin (block i uses slot i mod n_slots), so gathered parameters / unreduced gradients of at most
        `n_slots` blocks exist at any time.  The root unit (embeddings, final norm, head) keeps its own buffers, like the
        FSDP root.  All blocks have the same flat layout, which is what makes the slots interchangeable."""
        blocks = self.units[1:]
        if self.world_size == 1 or not blocks or blocks[0].pooled:
            return
        padded = blocks[0].padded
        assert all(u.padded == padded for u in blocks), "block units must share one flat layout"
        self.pool_slots = n_slots
        self.pool_compute = [torch.zeros(padded, dtype=torch.bfloat16, device=self.device) for _ in range(n_slots)]
        self.pool_grad = [torch.zeros(padded, dtype=torch.float32, device=self.device) for _ in range(n_slots)]
        for i, u in enumerate(blocks):
            u.bind_pooled(self.pool_compute[i % n_slots], self.pool_grad[i % n_slots])
        torch.cuda.empty_cache() if self.device.type == "cuda" else None

    def prepare_unit_grads(self, i: int) -> None:
        """pooled gradients: unit i's backward starts on a buffer that held another block's gradients.  Large GEMM weights
        are overwritten by their first weight-gradient GEMM (beta = 0, `_lazy_zero`); the tensors accumulated by reduction
        kernels or atomics (norm weights, biases, the MoE router) are cleared here."""
        u = self.units[i]
        if not u.pooled:
            return
        for s in u.specs:
            if self._lazy_zero(s):
                self._fresh_grads.add(s.name)
            else:
                u.gviews[s.name].zero_()

    def finish_unit_grads(self, i: int) -> None:
        """pooled gradients: a large weight that received no gradient must read as zero before the reduce-scatter"""
        u = self.units[i]
        if not u.pooled or not self._fresh_grads:
            return
        for s in u.specs:
            if s.name in self._fresh_grads:
                u.gviews[s.name].zero_()
                self._fresh_grads.discard(s.name)

    # parameters at least this large only ever receive their gradient from a weight-gradient GEMM first
    _LAZY_ZERO_MIN_NUMEL = 1 << 16

    def _lazy_zero(self, s: ParamSpec) -> bool:
        """True when the first gradient of `s` in a window comes from a weight-gradient GEMM that can OVERWRITE its buffer
        (beta = 0): the dense linears, and the 3-D expert weights (the K-grouped GEMM writes zeros for an expert without
        tokens).  Not the MoE router (split-K partial sums are atomically ADDED into a cleared buffer), not embedding tables
        that only receive scattered atomics (untied wte, wpe)."""
        if not self.lazy_grad_zero:
            return False
        if s.numel < self._LAZY_ZERO_MIN_NUMEL or not s.name.endswith(".weight") or s.name.endswith("mlp.gate.weight"):
            return False
        if s.name == "transformer.wpe.weight" or (s.name == "transformer.wte.weight" and not self.cfg.tie_word_embeddings):
            return False
        return True

    def take_fresh(self, wname: str) -> bool:
        """True exactly once per accumulation window and weight: its first weight-gradient GEMM must overwrite"""
        fresh = wname in self._fresh_grads
        self._fresh_grads.discard(wname)
        return fresh

    def zero_grad(self) -> None:
        """Clears the fp32 gradient buffers, lazily for the GEMM weights: the first weight-gradient GEMM of the next backward
        OVERWRITES its buffer (beta = 0) instead of read-modify-writing a freshly zeroed one, which saves one write and one
        read of every weight gradient per step (8 B / parameter); only the tensors that are accumulated by reduction kernels
        or atomics (norm weights, biases, the MoE router, scatter-only embedding tables) are cleared here."""
        self._fresh_grads = set()
        if self.comm is not None:
            self.comm.window_reset()
        for u in self.units:
            if u.pooled:  # cleared per unit at the start of its backward (prepare_unit_grads)
                continue
            for s in u.specs:
                if self._lazy_zero(s):
                    self._fresh_grads.add(s.name)
                else:
                    u.gviews[s.name].zero_()
            # sharded: the shard gradient is (over)written by the reduce-scatter, no need to clear it here
            if u.master.grad is not u.grad_full and self.comm is None:
                u.master.grad.zero_()

    # ------------------------------------------------------------------------------------------
    # forward
    # ------------------------------------------------------------------------------------------
    def _w(self, unit: FlatUnit, name: str):
        return unit.views.get(name)

    def _linear(self, unit: FlatUnit, wname: str, x, bname: str | None = None, *, c=None, alpha: float = 1.0,
                beta: float = 0.0, out=None, flags=None):
        """y = alpha * (x W^T + b) + beta * c, in FP8 (te.Linear under fp8_autocast) when `wname` is an FP8 linear and the
        pass runs under fp8_autocast, else in bf16"""
        w = unit.views[wname]
        bias = unit.views.get(bname) if bname is not None else None
        if not self._is_fp8(wname):
            return K.gemm(x, w, bias=bias, c=c, alpha=alpha, beta=beta, out=out, flags=flags)
        xs, xsi, xam = self.fp8.input_slot(wname)
        _, wsi, _ = self.fp8.weight_slot(wname)
        xq, _ = K.fp8_cast(x, K.E4M3, xs, amax=xam)
        wq = self._fp8_weight(wname, w, transposed=False)
        # fprop: one accumulator over the whole contraction (TE's fast accumulation for the forward GEMM)
        return K.gemm_fp8(xq, K.E4M3, xsi, wq, K.E4M3, wsi, bias=bias, c=c, alpha=alpha, beta=beta, out=out)

    def _fp8_weight(self, wname: str, w, transposed: bool):
        """e4m3 copy of weight `wname` (transposed: [in, out], the dgrad operand); kept for the pass if `_fp8_keep` names it"""
        key = (wname, transposed)
        q = self._fp8_wcache.get(key)
        if q is None:
            ws, _, wam = self.fp8.weight_slot(wname)
            if transposed:  # backward: the forward already recorded this weight's amax
                _, q = K.fp8_cast(w, K.E4M3, ws, plain=False, transpose=True)
            else:
                q, _ = K.fp8_cast(w, K.E4M3, ws, amax=wam)
            if wname in self._fp8_keep:
                self._fp8_wcache[key] = q
        return q

    def _norm_fwd(self, x, unit: FlatUnit, prefix: str):
        """RMSNorm or LayerNorm (get_normalization_function, normalization/__init__.py:13-30) -> (y, saved statistics)"""
        eps = self.cfg.layer_norm_epsilon
        if self.is_layernorm:
            y, mean, rstd = K.layernorm_fwd(x, unit.views[prefix + "weight"], unit.views.get(prefix + "bias"), eps)
            return y, (mean, rstd)
        return K.rmsnorm_fwd(x, unit.views[prefix + "weight"], eps)

    def _norm_bwd(self, dy, x, unit: FlatUnit, prefix: str, stats, dx_add=None):
        if self.is_layernorm:
            mean, rstd = stats
            return K.layernorm_bwd(dy, x, unit.views[prefix + "weight"], mean, rstd, unit.gviews[prefix + "weight"],
                                   unit.gviews.get(prefix + "bias"), dx_add=dx_add)
        return K.rmsnorm_bwd(dy, x, unit.views[prefix + "weight"], stats, unit.gviews[prefix + "weight"], dx_add=dx_add)

    # dropout call sites of one pass: 0 = embeddings, 4 i + 1 / + 2 / + 3 = block i attention residual / MLP residual /
    # attention probabilities
    def _drop_p(self, kind: str) -> float:
        if self._dropout_now is None:
            return 0.0
        return float(getattr(self.cfg, kind) or 0.0)

    def _drop_keys(self, site: int) -> tuple[int, int]:
        return K.dropout_keys(self._dropout_now, site)

    def _begin_dropout_pass(self) -> None:
        if not (self.has_dropout and self.training):
            self._dropout_now = None
            return
        if self.dropout_seed is None:
            self.dropout_seed = (int(torch.initial_seed()) + 0x632BE59BD9B4E019 * (self.rank + 1)) & ((1 << 63) - 1)
        self._dropout_now = (self.dropout_seed + self._dropout_passes) & ((1 << 63) - 1)
        self._dropout_passes += 1

    def _is_checkpointed(self, i: int) -> bool:
        k = self.checkpoint_every
        return k is not None and k > 0 and i % k == 0

    def _block_forward(self, i: int, x_in, position_ids, cu_seqlens, max_seqlen: int):
        """One GPTDolomiteBlock / SparseMoEBlock (gpt_dolomite/layer.py:49-87): returns (h_out, activations kept for backward)"""
        cfg = self.cfg
        u = self.units[i + 1]
        p = f"transformer.h.{i}."
        m_res = 1.0 if cfg.m_residual is None else float(cfg.m_residual)
        ln1, rstd1 = self._norm_fwd(x_in, u, p + "ln_1.")
        qkv = self._linear(u, p + "attn.c_attn.weight", ln1, p + "attn.c_attn.bias")
        if self.rope_cos is not None:
            K.rope_qk_inplace(qkv, self.n_groups, self.q_per_group, self.hd, self.rope_cos, self.rope_sin, position_ids)
        if self._kv_sink is not None:  # prefill of a KV cache: keys (rotated) and values of every prompt token
            self._kv_sink(i, qkv)
        p_att = self._drop_p("attn_pdrop")
        attn, lse = K.attn_varlen_fwd(qkv, cu_seqlens, max_seqlen, self.n_groups, self.q_per_group, self.hd, self.softmax_scale,
                                      dropout_p=p_att, dropout_keys=self._drop_keys(4 * i + 3) if p_att > 0 else (0, 0),
                                      alibi_slopes=self._alibi_now)
        p_res = self._drop_p("resid_pdrop")
        if p_res > 0:  # resid_dropout sits between c_proj and `* m_residual` / `+ residual` (padding_free.py:75, layer.py:73-77)
            y = self._linear(u, p + "attn.c_proj.weight", attn, p + "attn.c_proj.bias")
            h_mid = K.dropout_fwd(y, p_res, self._drop_keys(4 * i + 1), residual=x_in, post_mul=m_res, out=y)
        else:
            h_mid = self._linear(u, p + "attn.c_proj.weight", attn, p + "attn.c_proj.bias", c=x_in, alpha=m_res, beta=1.0)
        ln2, rstd2 = self._norm_fwd(h_mid, u, p + "ln_2.")
        if self.is_moe:
            from . import moe

            h, moe_saved = moe.forward(self, u, p, ln2, h_mid, m_res, layer=i)
            return h, (x_in, rstd1, ln1, qkv, attn, lse, h_mid, rstd2, ln2, moe_saved)
        fc = self._linear(u, p + "mlp.c_fc.weight", ln2, p + "mlp.c_fc.bias")
        act = K.act_fwd(fc, *self.act)
        if p_res > 0:  # gpt_dolomite/mlp.py:45-50 then layer.py:82-86
            y = self._linear(u, p + "mlp.c_proj.weight", act, p + "mlp.c_proj.bias")
            h = K.dropout_fwd(y, p_res, self._drop_keys(4 * i + 2), residual=h_mid, post_mul=m_res, out=y)
        else:
            h = self._linear(u, p + "mlp.c_proj.weight", act, p + "mlp.c_proj.bias", c=h_mid, alpha=m_res, beta=1.0)
        return h, (x_in, rstd1, ln1, qkv, attn, lse, h_mid, rstd2, ln2, fc, act)

    def forward(self, input_ids, position_ids, cu_seqlens, max_seqlen: int, labels=None, ignore_index: int = -100,
                save_for_backward: bool = True, fuse_head_loss: bool = False, alibi: bool = False,
                router_aux: bool = False, T_real: int | None = None, coef: float = 0.0):
        """Returns (logits_or_None, loss_or_None).  input_ids int64 [T]; cu_seqlens int32 [B+1].
        `fuse_head_loss`: the caller will backpropagate d(loss) = 1 (what train_step does), so the LM head's backward can run
        chunk-wise inside the loss computation and the [T, V] logits are never materialised.
        `alibi`: add the ALiBi bias of an alibi model to the attention logits (the key's index inside its document);
        False runs an alibi model as NoPE, which is what the reference's SDPA attention does without an attention mask.
        `router_aux` (MoE): also compute the load-balancing loss aux over the first `T_real` token rows (default: all) of
        every layer, add `coef * aux` to the loss, and return (logits_or_None, loss_or_None, aux [1] fp32, router logits:
        one bf16 [T, E] tensor per layer).  backward(aux_grad_dev=...) then takes s = coef * dL/dloss + dL/daux."""
        cfg = self.cfg
        self._aux_fwd = None
        if router_aux:
            if not self.is_moe:
                raise ValueError("router_aux needs an MoE model (model_type moe_dolomite)")
            T_real = input_ids.numel() if T_real is None else int(T_real)
            if not 0 < T_real <= input_ids.numel():
                raise ValueError(f"T_real={T_real} must be in [1, {input_ids.numel()}]")
            self._aux_fwd = (K.moe_aux_acc(cfg.num_experts, self.device), T_real, [])
        self._begin_dropout_pass()
        self._alibi_now = self._alibi_slopes_for(alibi)
        self._fp8_now = self.fp8 is not None and self.fp8_autocast and self.training and save_for_backward
        self._fp8_wcache.clear()
        T = input_ids.numel()
        root = self.units[0]
        comm = self.comm
        self._ensure_rope(int(max_seqlen))
        if comm is not None:
            comm.pre_forward_unit(0)
        m_emb = 1.0 if cfg.m_emb is None else float(cfg.m_emb)
        p_emb = self._drop_p("embd_pdrop")
        # gpt_dolomite/base.py:351-372: drop(wte(ids) [+ wpe(position_ids)]) * m_emb.  Without dropout and learned positions the
        # scale rides on the gather; otherwise it is a separate bf16 multiply after the sum / the mask (p = 0: all kept).
        post_scale = p_emb > 0 or (self.learned_positions and m_emb != 1.0)
        h = K.embedding_fwd(input_ids, root.views["transformer.wte.weight"], 1.0 if post_scale else m_emb)
        if self.learned_positions:  # wte(ids) + wpe(position_ids), one bf16 rounding
            if position_ids.dtype != torch.int64:
                position_ids = position_ids.long()
            h = K.add_scaled(h, K.embedding_fwd(position_ids, root.views["transformer.wpe.weight"], 1.0), 1.0)
        if post_scale:
            h = K.dropout_fwd(h, p_emb, self._drop_keys(0) if p_emb > 0 else (0, 0), post_mul=m_emb, out=h)
        saved_layers = []
        for i in range(cfg.n_layer):
            if comm is not None:
                comm.pre_forward_unit(i + 1)
            x_in = h
            h, layer = self._block_forward(i, x_in, position_ids, cu_seqlens, max_seqlen)
            if save_for_backward:
                # block activation checkpointing (gradient_checkpointing/block.py:13-37): every `checkpoint_every`-th
                # block keeps only its input and is re-run in backward
                saved_layers.append((x_in,) if self._is_checkpointed(i) else layer)
            del layer
            if comm is not None:
                comm.post_forward_unit(i + 1)
        hf, rstd_f = self._norm_fwd(h, root, "transformer.ln_f.")
        head_name = "transformer.wte.weight" if cfg.tie_word_embeddings else "lm_head.weight"
        head = root.views[head_name]
        inv_width = 1.0 if cfg.m_width is None else 1.0 / float(cfg.m_width)
        loss = None
        d_hf = dlogits = logits_out = None
        if labels is not None and save_for_backward and fuse_head_loss:
            # LM head + cross entropy + the head's own backward, chunk by chunk over the token rows
            # (gpt_dolomite/main.py:172-177, model_wrapper/pretraining.py:107-127): [T, V] logits never exist -- a chunk of
            # rows is projected, turned into its gradient in place by the row-resident CE kernel and consumed at once by
            # the head's dgrad / wgrad GEMMs.  Valid because the caller backpropagates d(loss) = 1 (train_step).
            scratch = K.cross_entropy_count(labels, ignore_index)
            loss_tok = torch.empty(T, dtype=torch.float32, device=hf.device)
            d_hf = torch.empty_like(hf)
            # FP8 head: the chunk rows are the contraction of its weight-gradient GEMM, a multiple of 16
            rows = self._head_chunk_rows(T, head.shape[0], self.head_chunk_bytes, 16 if self._is_fp8(head_name) else 8)
            buf = K.rows_empty(min(rows, T), head.shape[0], device=hf.device)
            self._fp8_keep = {head_name}
            for r0 in range(0, T, rows):
                r1 = min(T, r0 + rows)
                lg = self._linear(root, head_name, hf[r0:r1], alpha=inv_width, out=buf[: r1 - r0])
                K.cross_entropy_rows(lg, labels[r0:r1], loss_tok[r0:r1], scratch, ignore_index=ignore_index)
                self._linear_bwd(root, head_name, None, hf[r0:r1], lg, alpha=inv_width, dx_out=d_hf[r0:r1])
            loss = K.cross_entropy_mean(loss_tok, scratch)
            self._fp8_keep = set()
            self._fp8_wcache.clear()
            del buf
        else:
            logits = self._linear(root, head_name, hf, alpha=inv_width)
            if labels is not None:
                # fused CE fwd+bwd: dlogits overwrites the logits
                loss, _, dlogits = K.cross_entropy_fwd_bwd(logits, labels, ignore_index=ignore_index, dlogits=None)
            else:
                logits_out = logits.contiguous()  # [T, V] as the reference returns it: a copy when V % 8 != 0
        router_aux_saved = None
        if self._aux_fwd is not None:
            acc, T_real, router_logits = self._aux_fwd
            self._aux_fwd = None
            aux, c = K.moe_aux_finalize(acc, cfg.n_layer * T_real, coef, loss)  # loss += coef * aux on the device
            router_aux_saved = (c, T_real, float(coef))
        if save_for_backward:
            self._saved = dict(input_ids=input_ids, position_ids=position_ids, cu_seqlens=cu_seqlens, max_seqlen=max_seqlen,
                               layers=saved_layers, h_last=h, rstd_f=rstd_f, hf=hf, dlogits=dlogits, d_hf=d_hf, T=T,
                               dropout_seed=self._dropout_now, fp8=self._fp8_now, alibi=self._alibi_now,
                               router_aux=router_aux_saved)
        self._fp8_now = False
        self._fp8_wcache.clear()
        if router_aux_saved is not None:
            return logits_out, loss, aux, tuple(router_logits)
        return logits_out, loss

    def _alibi_slopes_for(self, alibi: bool):
        if not alibi:
            return None
        if self.alibi_slopes is None:
            raise ValueError("alibi=True needs a model with position_embedding_type='alibi'")
        return self.alibi_slopes

    @staticmethod
    def _head_chunk_rows(T: int, V: int, budget_bytes: int = 1 << 30, multiple: int = 8) -> int:
        """token rows per LM-head chunk: equal chunks of at most `budget_bytes` of bf16 logits, multiples of `multiple`
        rows (the rows of a chunk are the contraction length of its weight-gradient GEMM)"""
        max_rows = max(multiple, budget_bytes // (2 * V) // multiple * multiple)
        n_chunks = -(-T // max_rows)
        per = -(-T // n_chunks)
        return min(T, -(-per // multiple) * multiple)

    # ------------------------------------------------------------------------------------------
    # decoding with a KV cache (attention/sdpa.py:11-83, attention/flash.py:16-140 `past_key_values`)
    # ------------------------------------------------------------------------------------------
    def kv_slices(self, qkv):
        """(k, v) views [T, n_groups, head_dim] of a packed c_attn output (slot layout of attention/padding_free.py:79-116)"""
        T = qkv.shape[0]
        slots = qkv.view(T, self.n_groups, self.q_per_group + 2, self.hd)
        return slots[:, :, self.q_per_group], slots[:, :, self.q_per_group + 1]

    @torch.no_grad()
    def prefill(self, input_ids, position_ids, cu_seqlens, max_seqlen: int, cache: "KVCache", n_sequences: int | None = None,
                alibi: bool = False):
        """packed forward over the prompts (document b = sequence b for b < n_sequences; later documents, e.g. the alignment
        dummy of `_pad_packed_stream`, are run but not cached) that also fills `cache`; -> logits [T, V]"""
        cu = cu_seqlens.tolist()
        if n_sequences is not None:
            cu = cu[: n_sequences + 1]

        def sink(layer: int, qkv) -> None:
            k, v = self.kv_slices(qkv)
            for b in range(len(cu) - 1):
                n = cu[b + 1] - cu[b]
                cache.k[layer][b, :n].copy_(k[cu[b] : cu[b + 1]].reshape(n, -1))
                cache.v[layer][b, :n].copy_(v[cu[b] : cu[b + 1]].reshape(n, -1))

        self._kv_sink = sink
        try:
            logits, _ = self.forward(input_ids, position_ids, cu_seqlens, max_seqlen, save_for_backward=False, alibi=alibi)
        finally:
            self._kv_sink = None
        cache.lens.copy_(torch.tensor([cu[b + 1] - cu[b] for b in range(len(cu) - 1)], dtype=torch.int32))
        return logits

    @torch.no_grad()
    def decode_step(self, input_ids, cache: "KVCache", active=None, alibi: bool = False):
        """one new token per sequence: input_ids int64 [B]; appends its keys / values at position cache.lens[b] (sequences
        with active[b] == False are computed but their cache does not advance) -> logits [B, V].  Every op is the training
        kernel at T = B rows, except attention, which is the single-query cache kernel (csrc/attention_decode.cu).
        `alibi`: ALiBi bias of each cache position (the cache holds the real tokens of a sequence from position 0)."""
        cfg = self.cfg
        slopes = self._alibi_slopes_for(alibi)
        if self.comm is not None:
            raise NotImplementedError("decoding runs on an unsharded engine (world_size 1)")
        B = input_ids.numel()
        root = self.units[0]
        pos = cache.lens.long()  # position of the new token = tokens already cached
        rows = torch.arange(B, device=self.device)
        h = K.embedding_fwd(input_ids, root.views["transformer.wte.weight"], 1.0 if cfg.m_emb is None else float(cfg.m_emb))
        if self.learned_positions:
            h = K.add_scaled(h, K.embedding_fwd(pos, root.views["transformer.wpe.weight"], 1.0), 1.0)
        self._ensure_rope(int(cache.k[0].shape[1]))
        m_res = 1.0 if cfg.m_residual is None else float(cfg.m_residual)
        lens_incl = (cache.lens + 1).contiguous()
        for i in range(cfg.n_layer):
            u = self.units[i + 1]
            p = f"transformer.h.{i}."
            ln1, _ = self._norm_fwd(h, u, p + "ln_1.")
            qkv = K.gemm(ln1, u.views[p + "attn.c_attn.weight"], bias=u.views.get(p + "attn.c_attn.bias"))
            if self.rope_cos is not None:
                K.rope_qk_inplace(qkv, self.n_groups, self.q_per_group, self.hd, self.rope_cos, self.rope_sin, pos)
            k_new, v_new = self.kv_slices(qkv)
            cache.k[i][rows, pos] = k_new.reshape(B, -1)
            cache.v[i][rows, pos] = v_new.reshape(B, -1)
            attn = K.attn_decode(qkv, cache.k[i], cache.v[i], lens_incl, self.n_groups, self.q_per_group, self.hd, self.softmax_scale,
                                 alibi_slopes=slopes)
            h_mid = K.gemm(attn, u.views[p + "attn.c_proj.weight"], bias=u.views.get(p + "attn.c_proj.bias"), c=h, alpha=m_res,
                           beta=1.0)
            ln2, _ = self._norm_fwd(h_mid, u, p + "ln_2.")
            if self.is_moe:
                from . import moe

                h, _ = moe.forward(self, u, p, ln2, h_mid, m_res)
            else:
                fc = K.gemm(ln2, u.views[p + "mlp.c_fc.weight"], bias=u.views.get(p + "mlp.c_fc.bias"))
                act = K.act_fwd(fc, *self.act)
                h = K.gemm(act, u.views[p + "mlp.c_proj.weight"], bias=u.views.get(p + "mlp.c_proj.bias"), c=h_mid, alpha=m_res,
                           beta=1.0)
        hf, _ = self._norm_fwd(h, root, "transformer.ln_f.")
        head = root.views["transformer.wte.weight"] if cfg.tie_word_embeddings else root.views["lm_head.weight"]
        logits = K.gemm(hf, head, alpha=1.0 if cfg.m_width is None else 1.0 / float(cfg.m_width))
        cache.lens.add_(1 if active is None else active.to(torch.int32))
        return logits.contiguous()

    # ------------------------------------------------------------------------------------------
    # backward
    # ------------------------------------------------------------------------------------------
    def _linear_bwd(self, unit: FlatUnit, wname: str, bname: str | None, x, dy, alpha: float = 1.0, need_dx: bool = True,
                    dx_out=None):
        """autograd of y = alpha * (x W^T + b):  dx = alpha * dy W ; dW += alpha * dy^T x ; db += alpha * colsum(dy)"""
        if self._is_fp8(wname):
            return self._linear_bwd_fp8(unit, wname, bname, x, dy, alpha, need_dx, dx_out)
        w = unit.views[wname]
        gw = unit.gviews[wname]
        dx = K.gemm(dy, w, b_mn=True, alpha=alpha, out=dx_out) if need_dx else None
        fresh = self.take_fresh(wname)  # first gradient since zero_grad(): overwrite, the buffer was not cleared
        if self._deferred_wgrads is not None:
            # weight gradients of a block are launched together at the end of the block's backward (one persistent grid
            # over all their tiles instead of four launches with a partly filled last wave each)
            self._deferred_wgrads.append((dy, x, gw, alpha, not fresh))
            if len(self._deferred_wgrads) == 4:
                self._flush_wgrads()
        elif fresh:
            K.gemm(dy, x, a_mn=True, b_mn=True, out=gw, alpha=alpha)
        else:
            K.gemm(dy, x, a_mn=True, b_mn=True, out=gw, c=gw, alpha=alpha, beta=1.0)
        if bname is not None and bname in unit.gviews:
            K.colsum_accum(dy, unit.gviews[bname], alpha)
        return dx

    def _linear_bwd_fp8(self, unit: FlatUnit, wname: str, bname: str | None, x, dy, alpha: float = 1.0,
                        need_dx: bool = True, dx_out=None, dx_add=None):
        """te.Linear backward: dy is cast to e5m2 (plain for dgrad, transposed for wgrad); the weight and the input are
        re-cast, transposed, from their bf16 copies with the scales of their forward (the update runs after the backward),
        which gives the bits TE's saved fp8 copies hold.  dgrad / wgrad use the split accumulator, as TE does.
        `dx_add`: dx += ... (fp8 form of the bf16 GEMM's c / beta accumulation)"""
        if alpha != 1.0:
            # te.Linear's output gradient is that of its own output, i.e. bf16(alpha * dy) for the `* m_residual` /
            # `/ m_width` that follow it: cast (and record the amax of) that tensor, as TE does
            dy = K.dropout_bwd(dy, 0.0, (0, 0), pre_mul=alpha)
            alpha = 1.0
        w = unit.views[wname] if need_dx else None
        gw = unit.gviews[wname]
        xs, xsi, _ = self.fp8.input_slot(wname)
        _, wsi, _ = self.fp8.weight_slot(wname)
        gs, gsi, gam = self.fp8.grad_slot(wname)
        dyq, dyt = K.fp8_cast(dy, K.E5M2, gs, transpose=True, amax=gam)
        dx = None
        if need_dx:
            wt = self._fp8_weight(wname, w, transposed=True)
            if dx_add is not None:
                dx = K.gemm_fp8(dyq, K.E5M2, gsi, wt, K.E4M3, wsi, alpha=alpha, out=dx_add, c=dx_add, beta=1.0,
                                split_accumulate=True)
            else:
                dx = K.gemm_fp8(dyq, K.E5M2, gsi, wt, K.E4M3, wsi, alpha=alpha, out=dx_out, split_accumulate=True)
            del wt
        del dyq
        _, xt = K.fp8_cast(x, K.E4M3, xs, plain=False, transpose=True)
        fresh = self.take_fresh(wname)
        wg = (dyt, gsi, xt, xsi, gw, alpha, not fresh)
        if self._deferred_wgrads is not None:
            self._deferred_wgrads.append(("fp8", wg))
            if len(self._deferred_wgrads) == 4:
                self._flush_wgrads()
        else:
            K.gemm_fp8_wgrad_multi([wg])
        if bname is not None and bname in unit.gviews:
            K.colsum_accum(dy, unit.gviews[bname], alpha)
        return dx

    def _flush_wgrads(self) -> None:
        if not self._deferred_wgrads:
            return
        # FP8 entries are ("fp8", (dyt, s_dy, xt, s_x, dw, alpha, accumulate)); a block mixing FP8 and bf16 linears (a width
        # that is not a multiple of 16) gets one launch per kind
        fp8 = [q[1] for q in self._deferred_wgrads if isinstance(q[0], str)]
        bf16 = [q for q in self._deferred_wgrads if not isinstance(q[0], str)]

        def launch():
            if fp8:
                K.gemm_fp8_wgrad_multi(fp8)
            if bf16:
                K.gemm_wgrad_multi(bf16)

        if self.overlap_wgrads and self.device.type == "cuda":
            if self._wgrad_stream is None:
                self._wgrad_stream = torch.cuda.Stream(device=self.device)
            side, main = self._wgrad_stream, torch.cuda.current_stream()
            side.wait_stream(main)  # every operand of the list has been produced on the main stream
            with torch.cuda.stream(side):
                launch()
            # the allocator must not hand these blocks out before the launch has read them
            for t in [q[0] for q in bf16] + [q[1] for q in bf16] + [q[0] for q in fp8] + [q[2] for q in fp8]:
                t.record_stream(side)
        else:
            launch()
        self._deferred_wgrads.clear()

    def join_wgrad_stream(self, stream=None) -> None:
        """orders `stream` (default: the current one) after every weight-gradient launch issued so far"""
        if self._wgrad_stream is not None:
            (torch.cuda.current_stream() if stream is None else stream).wait_stream(self._wgrad_stream)

    def backward(self, dlogits=None, grad_scale_dev=None, aux_grad_dev=None) -> None:
        """Backward of the last forward.  `dlogits` overrides the CE gradient (logits-mode autograd).
        After forward(router_aux=True), `aux_grad_dev` (fp32 device scalar) is the factor s = coef * dL/dloss + dL/daux of
        the load-balancing term's router gradient; by default that of backpropagating the returned loss,
        coef * (grad_scale_dev or 1)."""
        s = self._saved
        if s is None:
            raise RuntimeError("backward called without a saved forward")
        self._aux_bwd = None
        if s.get("router_aux") is not None:
            c, T_real, coef = s["router_aux"]
            if aux_grad_dev is None:
                aux_grad_dev = torch.full((1,), coef, dtype=torch.float32, device=c.device)
                if grad_scale_dev is not None:
                    aux_grad_dev = aux_grad_dev * grad_scale_dev.reshape(1).float()
            self._aux_bwd = (c, aux_grad_dev.reshape(1).float().contiguous(), T_real)
        cfg = self.cfg
        root = self.units[0]
        comm = self.comm
        inv_width = 1.0 if cfg.m_width is None else 1.0 / float(cfg.m_width)
        m_res = 1.0 if cfg.m_residual is None else float(cfg.m_residual)
        head_name = "transformer.wte.weight" if cfg.tie_word_embeddings else "lm_head.weight"
        self._dropout_now = s.get("dropout_seed")  # the masks of the forward being backpropagated
        self._alibi_now = s.get("alibi")  # and its ALiBi decision (recomputed blocks too)
        self._fp8_now = s.get("fp8", False)  # and its FP8 mode (recomputed blocks too)
        self._fp8_wcache.clear()
        p_res = self._drop_p("resid_pdrop")
        if comm is not None:
            comm.pre_backward_unit(0)
        if dlogits is None and s.get("d_hf") is not None:
            # the head's backward already ran chunk-wise inside the loss computation (forward(fuse_head_loss=True))
            if grad_scale_dev is not None:
                raise RuntimeError("forward(fuse_head_loss=True) assumed d(loss) = 1; an upstream gradient cannot be applied")
            d_hf = s["d_hf"]
        else:
            # a caller's [T, V] gradient is staged into 16-byte rows when V % 8 != 0 (the dgrad / wgrad operand)
            dl = K.rows_aligned(dlogits) if dlogits is not None else s["dlogits"]
            if dl is None:
                raise RuntimeError("no loss gradient available: forward was run without labels and no dlogits was given")
            if grad_scale_dev is not None:
                K.scale_by_device_scalar(dl, grad_scale_dev)
            d_hf = self._linear_bwd(root, head_name, None, s["hf"], dl, alpha=inv_width)
        dh = self._norm_bwd(d_hf, s["h_last"], root, "transformer.ln_f.", s["rstd_f"])
        del d_hf
        for i in reversed(range(cfg.n_layer)):
            u = self.units[i + 1]
            if comm is not None:
                comm.pre_backward_unit(i + 1)
            p = f"transformer.h.{i}."
            layer = s["layers"][i]
            if len(layer) == 1:  # checkpointed block: re-run its forward from the saved input (MoE routing is deterministic)
                _, layer = self._block_forward(i, layer[0], s["position_ids"], s["cu_seqlens"], s["max_seqlen"])
            if self.is_moe:
                from . import moe

                x_in, rstd1, ln1, qkv, attn, lse, h_mid, rstd2, ln2, moe_saved = layer
                d_ln2 = moe.backward(self, u, p, ln2, dh, m_res, moe_saved, layer=i)
            else:
                x_in, rstd1, ln1, qkv, attn, lse, h_mid, rstd2, ln2, fc, act = layer
                if self.batch_block_wgrads:
                    self._deferred_wgrads = []
                if p_res > 0:
                    d_y = K.dropout_bwd(dh, p_res, self._drop_keys(4 * i + 2), pre_mul=m_res)
                    d_act = self._linear_bwd(u, p + "mlp.c_proj.weight", p + "mlp.c_proj.bias", act, d_y)
                    del d_y
                else:
                    d_act = self._linear_bwd(u, p + "mlp.c_proj.weight", p + "mlp.c_proj.bias", act, dh, alpha=m_res)
                # the c_fc bias gradient (column sums of d_fc) is accumulated by the activation backward while it writes d_fc
                d_fc = K.act_bwd(d_act, fc, *self.act, bias_grad_accum=u.gviews.get(p + "mlp.c_fc.bias"))
                del d_act
                d_ln2 = self._linear_bwd(u, p + "mlp.c_fc.weight", None, ln2, d_fc)
                del d_fc
            dh_mid = self._norm_bwd(d_ln2, h_mid, u, p + "ln_2.", rstd2, dx_add=dh)
            del d_ln2
            if p_res > 0:
                d_y = K.dropout_bwd(dh_mid, p_res, self._drop_keys(4 * i + 1), pre_mul=m_res)
                d_attn = self._linear_bwd(u, p + "attn.c_proj.weight", p + "attn.c_proj.bias", attn, d_y)
                del d_y
            else:
                d_attn = self._linear_bwd(u, p + "attn.c_proj.weight", p + "attn.c_proj.bias", attn, dh_mid, alpha=m_res)
            p_att = self._drop_p("attn_pdrop")
            dqkv = K.attn_varlen_bwd(d_attn, qkv, attn, lse, s["cu_seqlens"], s["max_seqlen"], self.n_groups,
                                     self.q_per_group, self.hd, self.softmax_scale, dropout_p=p_att,
                                     dropout_keys=self._drop_keys(4 * i + 3) if p_att > 0 else (0, 0),
                                     alibi_slopes=self._alibi_now)
            del d_attn
            if self.rope_cos is not None:
                K.rope_qk_inplace(dqkv, self.n_groups, self.q_per_group, self.hd, self.rope_cos, self.rope_sin,
                                  s["position_ids"], inverse=True)
            d_ln1 = self._linear_bwd(u, p + "attn.c_attn.weight", p + "attn.c_attn.bias", ln1, dqkv)
            del dqkv
            dh = self._norm_bwd(d_ln1, x_in, u, p + "ln_1.", rstd1, dx_add=dh_mid)
            del d_ln1, dh_mid
            if self._deferred_wgrads is not None:
                self._flush_wgrads()
                self._deferred_wgrads = None
            s["layers"][i] = None  # free this layer's activations
            if comm is not None:
                comm.post_backward_unit(i + 1)
        m_emb = 1.0 if cfg.m_emb is None else float(cfg.m_emb)
        p_emb = self._drop_p("embd_pdrop")
        if p_emb > 0 or (self.learned_positions and m_emb != 1.0):
            dh = K.dropout_bwd(dh, p_emb, self._drop_keys(0) if p_emb > 0 else (0, 0), pre_mul=m_emb, out=dh)
            m_emb = 1.0
        K.embedding_bwd(s["input_ids"], dh, root.gviews["transformer.wte.weight"], m_emb)
        if self.learned_positions:
            K.embedding_bwd(s["position_ids"], dh, root.gviews["transformer.wpe.weight"], 1.0)
        if self._fresh_grads:  # a weight that received no gradient in this backward still has to read as zero
            for name, unit, _ in self.named_views():
                if name in self._fresh_grads:
                    unit.gviews[name].zero_()
            self._fresh_grads.clear()
        if comm is not None:
            comm.post_backward_unit(0)
        self.join_wgrad_stream()  # optimizer / gradient norm / the next zero_grad run on the main stream
        if self._fp8_now:
            # DelayedScaling update of every slot.  TE updates the forward slots when the forward ends; nothing reads them
            # between that point and here except this backward, which must see the forward's scales, so running both
            # updates now gives the same scales to the next micro-step
            # a sharded model's ranks run the same linears in lock step: their amaxes are reduced so the scales agree
            self.fp8.update(all_reduce=self.comm is not None and self.world_size > 1)
            self._fp8_now = False
            self._fp8_wcache.clear()
        self._aux_bwd = None
        self._saved = None

    # ------------------------------------------------------------------------------------------
    # state dict (reference names; SURVEY section 8a)
    # ------------------------------------------------------------------------------------------
    def full_master(self, unit: FlatUnit) -> torch.Tensor:
        if self.world_size == 1:
            return unit.master.detach()
        return self.comm.gather_master(unit)

    def state_dict(self) -> dict:
        out = {}
        for u in self.units:
            full = self.full_master(u)
            for s in u.specs:
                out[s.name] = full[s.offset : s.offset + s.numel].view(s.shape).clone()
        if self.cfg.tie_word_embeddings:
            pass  # lm_head.weight is tied: _tied_weights_keys (gpt_dolomite/main.py:12) -> not serialised
        return out

    def load_state_dict(self, sd: dict, strict: bool = True) -> None:
        seen = set()
        for u in self.units:
            full = torch.zeros(u.padded, dtype=torch.float32)
            for s in u.specs:
                if s.name in sd:
                    t = sd[s.name]
                    if tuple(t.shape) != s.shape:
                        raise ValueError(f"shape mismatch for {s.name}: {tuple(t.shape)} vs {s.shape}")
                    full[s.offset : s.offset + s.numel].view(s.shape).copy_(t.detach().float().cpu())
                    seen.add(s.name)
                elif strict:
                    raise KeyError(f"missing key {s.name} in state_dict")
            u.full_master_from(full)
        if strict:
            extra = set(sd) - seen - ({"lm_head.weight"} if self.cfg.tie_word_embeddings else set())
            if extra:
                raise KeyError(f"unexpected keys in state_dict: {sorted(extra)[:5]}")

    def refresh_compute_from_master(self) -> None:
        """bf16 compute copy <- fp32 masters (world_size == 1; the sharded path all-gathers instead)"""
        assert self.world_size == 1
        for u in self.units:
            K.cast_f32_to_bf16(u.master.data, u.compute)
            u.gathered = True
