"""CPU: FP8 reference arithmetic (TransformerEngine DelayedScaling / te.Linear, restated), the FP8-linear selection rule and
the FP8 tensor-core instructions in the built library.

The reference functions at the top are what the GPU tests (test_gpu_fp8.py) compare the kernels against."""

import os
import shutil
import subprocess

import pytest
import torch

E4M3, E5M2 = 0, 1
FP8_MAX = {E4M3: 448.0, E5M2: 57344.0}
_DTYPE = {E4M3: torch.float8_e4m3fn, E5M2: torch.float8_e5m2}


def quantize_ref(x: torch.Tensor, scale: float, fmt: int) -> torch.Tensor:
    """q = satfinite_rne(fp32(x) * scale) as uint8 bits.  The product is rounded to fp32 once; torch's fp8 cast rounds to
    nearest-even but does not saturate, hence the clamp first."""
    mx = FP8_MAX[fmt]
    y = x.float() * torch.tensor(scale, dtype=torch.float32)
    return y.clamp(-mx, mx).to(_DTYPE[fmt]).view(torch.uint8)


def dequantize_ref(q: torch.Tensor, fmt: int) -> torch.Tensor:
    return q.view(_DTYPE[fmt]).to(torch.float64)


def recipe_update_ref(history: torch.Tensor, scale: torch.Tensor, fp8_max: float):
    """DelayedScaling(amax_history_len=len, amax_compute_algo="max", margin=0) update of fp32 [len, n] history and [n]
    scales -> (new history, new scale, new scale_inv); the arithmetic of TE 1.x's amax-and-scale update."""
    amax = torch.max(history, dim=0).values  # NaN propagates
    sf = torch.tensor(fp8_max, dtype=torch.float32) / amax
    sf = torch.where(amax > 0.0, sf, scale)
    sf = torch.where(torch.isfinite(amax), sf, scale)
    new_hist = torch.roll(history, -1, 0)
    new_hist[0].fill_(0.0)
    return new_hist, sf, torch.tensor(1.0, dtype=torch.float32) / sf


def _bits(vals, fmt, scale=1.0):
    return quantize_ref(torch.tensor(vals, dtype=torch.bfloat16), scale, fmt).tolist()


def test_quantizer_saturates_at_max():
    assert _bits([448.0, 480.0, 1e30, float("inf"), -float("inf"), -1000.0], E4M3) == [0x7E, 0x7E, 0x7E, 0x7E, 0xFE, 0xFE]
    assert _bits([57344.0, 61440.0, float("inf"), -1e9], E5M2) == [0x7B, 0x7B, 0x7B, 0xFB]
    # saturation applies to the scaled value
    assert _bits([2.0], E4M3, scale=1000.0) == [0x7E]


def test_quantizer_subnormals():
    # e4m3: smallest subnormal 2^-9 (bits 0x01), largest subnormal 7 * 2^-9 (0x07), smallest normal 2^-6 (0x08)
    assert _bits([2.0 ** -9, 7 * 2.0 ** -9, 2.0 ** -6, -(2.0 ** -9)], E4M3) == [0x01, 0x07, 0x08, 0x81]
    # e5m2: smallest subnormal 2^-16, smallest normal 2^-14
    assert _bits([2.0 ** -16, 3 * 2.0 ** -16, 2.0 ** -14], E5M2) == [0x01, 0x03, 0x04]
    # below half the smallest subnormal rounds to zero; exactly half is a tie -> even (zero)
    assert _bits([2.0 ** -11, 2.0 ** -10], E4M3) == [0x00, 0x00]


def test_quantizer_ties_to_even():
    # e4m3 around 1.0: spacing 1/8.  1 + 1/16 is halfway between 1.0 (0x38, even) and 1.125 (0x39) -> 0x38;
    # 1.125 + 1/16 is halfway between 0x39 and 1.25 (0x3A, even) -> 0x3A
    assert _bits([1.0 + 1 / 16, 1.125 + 1 / 16], E4M3) == [0x38, 0x3A]
    # e5m2 around 1.0: spacing 1/4
    assert _bits([1.0 + 1 / 8, 1.25 + 1 / 8], E5M2) == [0x3C, 0x3E]
    # the subnormal range ties to even too: 1.5 * 2^-9 -> 2 * 2^-9 (0x02), 2.5 * 2^-9 -> 0x02
    assert _bits([1.5 * 2.0 ** -9, 2.5 * 2.0 ** -9], E4M3) == [0x02, 0x02]


def test_recipe_update_reference():
    h = torch.zeros(16, 4)
    h[0] = torch.tensor([2.0, 0.0, float("inf"), float("nan")])
    h[5, 0] = 4.0
    s = torch.full((4,), 3.0)
    nh, ns, nsi = recipe_update_ref(h, s, 448.0)
    assert ns.tolist() == [112.0, 3.0, 3.0, 3.0]  # 448 / max(2, 4); zero, inf and NaN keep the scale
    assert torch.equal(nsi, 1.0 / ns)
    assert nh[0].tolist() == [0.0] * 4 and nh[4, 0].item() == 4.0 and nh[15, 0].item() == 2.0


def _cfg(**kw):
    from dolomite_engine_b200.hf_models.config import GPTDolomiteConfig

    base = dict(vocab_size=512, n_positions=256, n_embd=256, n_layer=2, n_head=4, num_key_value_heads=4, n_inner=512,
                activation_function="swiglu", normalization_function="rmsnorm", position_embedding_type="rope",
                add_bias=False, tie_word_embeddings=True)
    base.update(kw)
    kv = base["num_key_value_heads"]
    base.setdefault("attention_head_type", "mha" if kv == base["n_head"] else ("mqa" if kv == 1 else "gqa"))
    return GPTDolomiteConfig(**base)


def _moe_cfg(E):
    from dolomite_engine_b200.hf_models.config import MoEDolomiteConfig

    return MoEDolomiteConfig(vocab_size=512, n_positions=256, n_embd=256, n_layer=1, n_head=4, num_key_value_heads=4,
                             n_inner=512, activation_function="swiglu", normalization_function="rmsnorm",
                             position_embedding_type="rope", add_bias=False, num_experts=E, num_experts_per_tok=2,
                             attention_head_type="mha")


_BLOCK = ("attn.c_attn.weight", "attn.c_proj.weight", "mlp.c_fc.weight", "mlp.c_proj.weight")


def _block_names(n_layer):
    return [f"transformer.h.{i}.{s}" for i in range(n_layer) for s in _BLOCK]


def test_selection_tied_dense():
    from dolomite_engine_b200.fp8 import fp8_weight_names

    assert fp8_weight_names(_cfg()) == _block_names(2)  # the tied head is F.linear on wte: BF16


def test_selection_untied_gqa_and_c1():
    from dolomite_engine_b200.fp8 import fp8_weight_names
    from dolomite_engine_b200.hf_models.config import CommonConfig

    assert fp8_weight_names(_cfg(num_key_value_heads=2, tie_word_embeddings=False)) == _block_names(2) + ["lm_head.weight"]
    import yaml

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "configs", "c1_tiny.yml")) as f:
        pc = yaml.safe_load(f)["model_args"]["pretrained_config"]
    cfg = _cfg(**{k: v for k, v in pc.items() if k != "model_type"})
    names = fp8_weight_names(cfg)
    assert isinstance(cfg, CommonConfig) and set(_block_names(cfg.n_layer)) <= set(names)
    assert ("lm_head.weight" in names) == (not cfg.tie_word_embeddings)


def test_selection_skips_dimensions_not_multiple_of_16():
    from dolomite_engine_b200.fp8 import fp8_weight_names

    # bigcode shape (LayerNorm, GELU, biases, MQA, learned positions), with an MLP width that is not a multiple of 16
    cfg = _cfg(normalization_function="layernorm", activation_function="gelu_pytorch_tanh", add_bias=True,
               num_key_value_heads=1, position_embedding_type="learned_absolute", n_inner=1000)
    names = fp8_weight_names(cfg)
    assert "transformer.h.0.attn.c_attn.weight" in names and "transformer.h.0.attn.c_proj.weight" in names
    assert "transformer.h.0.mlp.c_fc.weight" not in names and "transformer.h.0.mlp.c_proj.weight" not in names
    assert fp8_weight_names(_cfg(normalization_function="layernorm", activation_function="gelu_pytorch_tanh",
                                 add_bias=True, num_key_value_heads=1)) == _block_names(2)


@pytest.mark.parametrize("E", [8, 32])
def test_selection_moe(E):
    from dolomite_engine_b200.fp8 import fp8_weight_names

    names = fp8_weight_names(_moe_cfg(E))
    # experts are ParameterizedExperts (not nn.Linear): BF16; the router gate is FP8 only when E % 16 == 0
    assert names[:2] == ["transformer.h.0.attn.c_attn.weight", "transformer.h.0.attn.c_proj.weight"]
    assert ("transformer.h.0.mlp.gate.weight" in names) == (E % 16 == 0)
    assert not any(".mlp.c_" in n for n in names)


def test_argument_surface():
    from dolomite_engine_b200.arguments import MixedPrecisionArgs

    a = MixedPrecisionArgs(dtype="fp8", fp8_backend="nvte")
    assert a.dtype == "fp8" and a.fp8_backend == "nvte"
    assert MixedPrecisionArgs(dtype="float8", fp8_backend="nvte").dtype == "fp8"
    with pytest.raises(NotImplementedError, match="msamp"):
        MixedPrecisionArgs(dtype="fp8", fp8_backend="msamp")
    with pytest.raises(ValueError, match="fp8_backend"):
        MixedPrecisionArgs(dtype="fp8")
    with pytest.raises(ValueError, match="fp8 dtype"):
        MixedPrecisionArgs(dtype="bf16", fp8_backend="nvte")
    assert MixedPrecisionArgs(dtype="bf16").fp8_backend is None


def test_recipe_state_roundtrip():
    from dolomite_engine_b200.fp8 import Fp8Recipe

    names = _block_names(2)
    r = Fp8Recipe(names, device="cpu")
    assert r.fwd_history.shape == (16, 2 * len(names)) and r.bwd_history.shape == (16, len(names))
    assert torch.all(r.fwd_scale == 1) and torch.all(r.bwd_scale_inv == 1) and torch.all(r.fwd_history == 0)
    r.fwd_scale[3] = 7.0
    r.bwd_history[0, 1] = 2.5
    sd = r.state_dict()
    r2 = Fp8Recipe(names, device="cpu")
    r2.load_state_dict(sd)
    assert r2.fwd_scale[3].item() == 7.0 and r2.bwd_history[0, 1].item() == 2.5
    with pytest.raises(ValueError):
        Fp8Recipe(names[:2], device="cpu").load_state_dict(sd)


def test_sass_has_fp8_tensor_core_mma():
    """the FP8 GEMM is wgmma with e4m3 / e5m2 operands: the sm_90a SASS names that form QGMMA (HGMMA is the 16-bit one)"""
    from dolomite_engine_b200 import _lib, build

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    build.build()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    for kind in ("E4M3.E4M3", "E5M2.E4M3"):
        assert f"GMMA.64x128x32.F32.{kind}" in sass, kind
