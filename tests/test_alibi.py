"""CPU: ALiBi host logic and oracle against the reference fixtures (tools/pin_alibi.py), the configurations the engine
accepts, and the SASS of the ALiBi attention kernels."""

import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import alibi_oracle as A
import oracle.dolomite_oracle as O
from dolomite_engine_b200.alibi import alibi_slopes
from dolomite_engine_b200.engine import check_supported
from dolomite_engine_b200.hf_models.config import GPTDolomiteConfig

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
HEADS = [1, 2, 3, 5, 6, 8, 12, 20, 24, 32, 40, 48, 64]
BIAS_STRIDE = 61
_BASE = dict(vocab_size=512, n_positions=256, n_embd=128, n_layer=2, n_inner=256, activation_function="swiglu",
             position_embedding_type="alibi", add_bias=False)
MODELS = {
    "mha_eager_nomask": (dict(n_head=8, attention_head_type="mha"), "eager"),
    "gqa_eager_left": (dict(n_head=8, num_key_value_heads=2, attention_head_type="gqa"), "eager"),
    "mqa_sdpa_mask": (dict(n_head=8, attention_head_type="mqa"), "sdpa"),
    "mha_sdpa_nomask": (dict(n_head=8, attention_head_type="mha"), "sdpa"),
}


@pytest.fixture(scope="module")
def fx():
    return np.load(os.path.join(GOLDEN, "alibi.npz"))


@pytest.mark.parametrize("n", HEADS)
def test_slopes_are_bit_identical_to_the_reference(fx, n):
    s = alibi_slopes(n)
    assert s.dtype == torch.float32
    assert np.array_equal(s.numpy(), fx[f"slopes_{n}"])


@pytest.mark.parametrize("case", ["nomask", "left", "right", "short"])
@pytest.mark.parametrize("n", [5, 32])
def test_bias_is_bit_identical_to_the_reference(fx, case, n):
    mask = fx[f"mask_{case}"] if f"mask_{case}" in fx.files else None
    stride = 1 if case == "short" else BIAS_STRIDE
    L = 37 if case == "short" else 8192
    B = 3 if case == "short" else (2 if mask is None else 4)
    kpos = A.key_positions(mask, B, L)
    for bf16, key in ((False, "bias32"), (True, "bias16")):
        b = A.alibi_bias(alibi_slopes(n), kpos, bf16)[..., ::stride]
        assert np.array_equal(b.numpy(), fx[f"{key}_{case}_{n}"]), key


def _oracle_padded(kw, impl, tokens, mask):
    cfg = O.OracleConfig(**kw)
    params = O.init_params(cfg, seed=42)
    B, S = tokens.shape
    m = np.ones((B, S), dtype=bool) if mask is None else mask.astype(bool)
    ids = tokens[m]
    cu = np.concatenate([[0], np.cumsum(m.sum(1))]).astype(np.int32)
    pos = np.concatenate([np.arange(n) for n in m.sum(1)])
    p = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    if impl == "eager" or mask is not None:
        with A.install(alibi_slopes(cfg.n_head), bias_bf16=False):
            logits = O.forward_logits(p, cfg, ids, pos, cu)
    else:
        logits = O.forward_logits(p, cfg, ids, pos, cu)
    labels = np.full(ids.shape, -100, dtype=np.int64)
    for d in range(B):
        labels[cu[d] : cu[d + 1] - 1] = ids[cu[d] + 1 : cu[d + 1]]
    loss = torch.nn.functional.cross_entropy(logits, torch.as_tensor(labels), ignore_index=-100)
    loss.backward()
    return loss.detach(), logits.detach(), {k: v.grad for k, v in p.items()}


@pytest.mark.parametrize("name", sorted(MODELS))
def test_oracle_matches_the_reference_models(name):
    """eager: the existing pins (logits 4e-7, gradients 2e-9); SDPA sums in another order (measured 1.4e-6 / 2.2e-8)"""
    kw, impl = MODELS[name]
    f = np.load(os.path.join(GOLDEN, f"alibi_model_{name}.npz"))
    loss, logits, grads = _oracle_padded({**_BASE, **kw}, impl, f["tokens"], f["mask"] if "mask" in f.files else None)
    tol_l, tol_g = (4e-7, 2e-9) if impl == "eager" else (2e-6, 5e-8)
    assert abs(loss.item() - float(f["loss"])) <= 1e-5
    assert (logits - torch.from_numpy(f["logits"])).abs().max().item() <= tol_l
    for key in f.files:
        if key.startswith("grad:"):
            g = grads[key[5:]].flatten()[::16]
            assert (g - torch.from_numpy(f[key])).abs().max().item() <= tol_g, key


def _cfg(**kw):
    return GPTDolomiteConfig(**{**_BASE, "n_head": 8, "attention_head_type": "mha", **kw})


@pytest.mark.parametrize("impl", ["eager", "sdpa"])
def test_check_supported_accepts_padded_eager_and_sdpa(impl):
    check_supported(_cfg(), attention_implementation=impl, use_padding_free_transformer=False)


@pytest.mark.parametrize("impl,padding_free", [("flash_attention_2", False), ("flash_attention_2", True), ("eager", True),
                                               ("sdpa", True)])
def test_check_supported_rejects_flash_and_padding_free(impl, padding_free):
    with pytest.raises(NotImplementedError, match="alibi"):
        check_supported(_cfg(), attention_implementation=impl, use_padding_free_transformer=padding_free)
    with pytest.raises(NotImplementedError):
        check_supported(_cfg())


def test_engine_keeps_slopes_and_leaves_the_state_dict_alone():
    from dolomite_engine_b200.engine import DolomiteEngine

    eng = DolomiteEngine(_cfg(), "cpu", seed=1, attention_implementation="eager", use_padding_free_transformer=False)
    assert torch.equal(eng.alibi_slopes, alibi_slopes(8))
    nope = DolomiteEngine(_cfg(position_embedding_type="nope"), "cpu", seed=1)
    assert nope.alibi_slopes is None
    assert sorted(eng.state_dict()) == sorted(nope.state_dict())
    with pytest.raises(NotImplementedError):
        DolomiteEngine(_cfg(), "cpu", seed=1)


def test_model_constructor_passes_its_settings():
    from dolomite_engine_b200.hf_models.modeling import GPTDolomiteForCausalLM

    for impl, pf in (("flash_attention_2", False), ("eager", True)):
        with pytest.raises(NotImplementedError, match="alibi"):
            GPTDolomiteForCausalLM(_cfg(), attn_implementation=impl, use_padding_free_transformer=pf, device="cpu")
    m = GPTDolomiteForCausalLM(_cfg(), attn_implementation="sdpa", use_padding_free_transformer=False, device="cpu")
    assert m._alibi_pass(True) and not m._alibi_pass(False)
    m = GPTDolomiteForCausalLM(_cfg(), attn_implementation="eager", use_padding_free_transformer=False, device="cpu")
    assert m._alibi_pass(True) and m._alibi_pass(False)


def _ops(body):
    return re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9.]*)", body)


def test_alibi_kernels_keep_the_tensor_core_path_and_add_no_local_memory():
    """every ALIBI instance uses HGMMA / UTMALDG where its plain kernel does; it has no local memory unless its plain
    kernel has (the head_dim 128 dK/dV kernel already spills a few registers)"""
    from dolomite_engine_b200 import _lib, build

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    build.build()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    funcs = {}
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split("\n", 1)[0].strip()
        m = re.search(r"(attn_(?:fwd|bwd|dq|decode)_kernel)ILi(\d+)ELb([01])E", name)
        if m:
            funcs[(m.group(1), int(m.group(2)), m.group(3) == "1")] = _ops(body)
    assert len(funcs) == 4 * 6 * 2, sorted(funcs)
    for (kern, hd, alibi), ops in funcs.items():
        if not alibi:
            continue
        base = funcs[(kern, hd, False)]
        for op in ("HGMMA.64x", "UTMALDG"):
            has = lambda o: any(x.startswith(op) for x in o)  # noqa: E731
            assert has(ops) == has(base), (kern, hd, op)
        local = lambda o: any(x.startswith(("LDL", "STL")) for x in o)  # noqa: E731
        assert not local(ops) or local(base), (kern, hd)
