"""GPU: vocabularies that are not a multiple of 8.  The bf16 GEMM at every extent tail, the cross-entropy kernel on rows whose
last 16-byte vector is partial, and models with odd vocabularies against the reference fixtures of tools/pin_vocab.py,
with the bars of test_gpu_model.py: loss within 1e-3 relative, logits as test_gpu_model compares the bf16 engine with
the fp32 oracle, every gradient within rel-L2 3e-2."""

import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle.dolomite_oracle as O
from test_vocab import EOS, GOLDEN, MODELS, _fixture_params, _packed_inputs, _padded_inputs, subsample

pytestmark = pytest.mark.gpu


def _k():
    from dolomite_engine_b200 import kernels

    return kernels


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _ld(cols, dtype):
    per = 16 // torch.empty((), dtype=dtype).element_size()
    return -(-cols // per) * per


def _stored(rows, cols, dtype, gen, fill=float("nan"), extra=0):
    """[rows, cols] random view of a [rows, 16-byte-rounded cols + extra] buffer whose spare columns hold `fill`"""
    buf = torch.full((rows, _ld(cols, dtype) + extra), fill, dtype=dtype, device="cuda")
    buf[:, :cols] = (torch.randn(rows, cols, generator=gen) * 0.5).to(dtype).cuda()
    return buf, buf[:, :cols]


# ---------------------------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------------------------
# every tail 0..7 of M, N and K appears; the last shapes are the head GEMMs of an odd vocabulary at a small T
SHAPES = [(128 + a, 256 + b, 64 + c) for a, b, c in zip(range(8), [3, 5, 7, 0, 2, 4, 6, 1], [5, 2, 7, 4, 1, 6, 3, 0])]
SHAPES += [(1, 9, 1), (7, 1, 9), (200, 2053, 128), (2053, 128, 200), (256, 130, 2051)]
SENTINEL = -512.0


def _check_d_padding(dbuf, N):
    """A TMA store writes the 16-byte segment holding column N - 1 whole: its columns after N - 1 may receive 0.
    Every column after that segment is untouched."""
    seg = _ld(N, dbuf.dtype)
    tail = dbuf[:, N:seg]
    assert bool(((tail == SENTINEL) | (tail == 0)).all()), "the last 16-byte segment of a row received data"
    assert bool((dbuf[:, seg:] == SENTINEL).all()), "a column after the last 16-byte segment of D was written"


def _gemm_case(M, N, K, a_mn, b_mn, f32, with_c, with_bias, tile_n, splitk=False):
    Km = _k()
    gen = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    _, a = _stored(K, M, torch.bfloat16, gen) if a_mn else _stored(M, K, torch.bfloat16, gen)
    _, b = _stored(K, N, torch.bfloat16, gen) if b_mn else _stored(N, K, torch.bfloat16, gen)
    A = (a.t() if a_mn else a).float()
    B = (b.t() if b_mn else b).float()
    dt = torch.float32 if f32 else torch.bfloat16
    dbuf, d = _stored(M, N, dt, gen, fill=SENTINEL, extra=8)
    c0 = d.clone().float()
    bias = (torch.randn(N, generator=gen) * 0.5).bfloat16().cuda() if with_bias else None
    alpha, beta = 0.75, (0.5 if with_c else 0.0)
    ref = alpha * (A @ B.t() + (bias.float() if with_bias else 0.0))
    if with_c or splitk:
        ref = ref + (1.0 if splitk else beta) * c0
    old = Km.get_option("gemm_tile_n")
    Km.set_option("gemm_tile_n", tile_n)
    try:
        if splitk:
            Km.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out=d, c=d, alpha=alpha, beta=1.0,
                    flags=Km.GEMM_SPLITK_ACCUMULATE)
        else:
            Km.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out=d, c=d if with_c else None, alpha=alpha, beta=beta, bias=bias)
        torch.cuda.synchronize()
    finally:
        Km.set_option("gemm_tile_n", old)
    got = d.float()
    assert torch.isfinite(got).all(), "a padding column (NaN) was read as data"
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item() + 1e-6
    assert err <= (2e-5 if f32 else 8e-3) * scale * (4 if splitk else 1), (err, scale)
    _check_d_padding(dbuf, N)


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("tile_n", [128, 256])
def test_gemm_any_extent_bf16_d(M, N, K, a_mn, b_mn, tile_n):
    _gemm_case(M, N, K, a_mn, b_mn, False, with_c=False, with_bias=True, tile_n=tile_n)
    _gemm_case(M, N, K, a_mn, b_mn, False, with_c=True, with_bias=False, tile_n=tile_n)


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True)])
@pytest.mark.parametrize("tile_n", [128, 256])
def test_gemm_any_extent_f32_d(M, N, K, a_mn, b_mn, tile_n):
    _gemm_case(M, N, K, a_mn, b_mn, True, with_c=False, with_bias=False, tile_n=tile_n)
    _gemm_case(M, N, K, a_mn, b_mn, True, with_c=True, with_bias=True, tile_n=tile_n)


@pytest.mark.parametrize("M,N,K", [(2053, 128, 1031), (129, 263, 4099), (37, 2051, 8195)])
def test_gemm_any_extent_split_k_accumulate(M, N, K):
    _gemm_case(M, N, K, True, True, True, with_c=True, with_bias=False, tile_n=128, splitk=True)


def test_gemm_wgrad_multi_any_extent():
    """the block weight-gradient launch with odd M and N (fp32 D, both operands MN-major)"""
    Km = _k()
    gen = torch.Generator().manual_seed(5)
    T = 203
    probs, refs = [], []
    for M, N in [(2053, 128), (131, 77), (8, 9)]:
        _, dy = _stored(T, M, torch.bfloat16, gen)
        _, x = _stored(T, N, torch.bfloat16, gen)
        dbuf, dw = _stored(M, N, torch.float32, gen, fill=SENTINEL, extra=8)
        refs.append((dbuf, N, 0.5 * dy.float().t() @ x.float()))
        probs.append((dy, x, dw, 0.5, False))
    Km.gemm_wgrad_multi(probs)
    for dbuf, N, ref in refs:
        got = dbuf[:, :N]
        assert (got - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
        _check_d_padding(dbuf, N)


# ---------------------------------------------------------------------------------------------------------------------
# cross entropy
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [1, 7, 9, 2051, 2056, 36871, 50257, 128259])
@pytest.mark.parametrize("in_place", [False, True])
def test_cross_entropy_any_vocabulary(V, in_place):
    """single-CTA widths (V <= 49152 and even ones up to it), the 2-CTA cluster (36871: an odd width of the 24-vector
    single-CTA range, 50257) and the 4-CTA cluster (128259); padding columns hold NaN"""
    Km = _k()
    T = 67
    gen = torch.Generator().manual_seed(V)
    buf, x = _stored(T, V, torch.bfloat16, gen)
    buf[:, :V] *= 8
    labels = torch.randint(0, V, (T,), generator=gen)
    labels[3] = V - 1
    labels[5] = -100
    labels[T - 1] = -100
    labels = labels.cuda()
    logit_scale, grad_scale = 0.625, 1.5
    xf = x.float().clone().requires_grad_(True)
    want = F.cross_entropy(xf * logit_scale, labels, ignore_index=-100)
    (want * grad_scale).backward()
    if in_place:
        loss, loss_tok, dl = Km.cross_entropy_fwd_bwd(x, labels, ignore_index=-100, logit_scale=logit_scale,
                                                      grad_scale=grad_scale)
    else:
        dbuf = torch.full_like(buf, float("nan"))
        dl = dbuf[:, :V]
        loss, loss_tok, _ = Km.cross_entropy_fwd_bwd(x, labels, ignore_index=-100, logit_scale=logit_scale,
                                                     grad_scale=grad_scale, dlogits=dl)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all() and torch.isfinite(loss_tok).all()
    assert abs(loss.item() - want.item()) <= 1e-4 * abs(want.item()) + 1e-6, (loss.item(), want.item())
    g = dl.float()
    assert torch.isfinite(g).all()
    ref = xf.grad.cuda()
    assert (g - ref).abs().max().item() <= 1e-2 * ref.abs().max().item() + 1e-7
    assert bool((g[5] == 0).all()) and bool((g[T - 1] == 0).all())
    if not in_place and V % 8:
        # the partial vector's spare lanes get 0; the columns after it are not touched
        last = (V + 7) // 8 * 8
        assert bool((dbuf[:, V:last] == 0).all())


def test_cross_entropy_rows_chunks_match_one_call():
    """the fused head's per-chunk calls (count / rows / mean) give the one-call result at an odd V"""
    Km = _k()
    V, T = 2053, 96
    gen = torch.Generator().manual_seed(1)
    buf, x = _stored(T, V, torch.bfloat16, gen)
    labels = torch.randint(0, V, (T,), generator=gen).cuda()
    loss, _, dl = Km.cross_entropy_fwd_bwd(buf.clone()[:, :V], labels)
    scratch = Km.cross_entropy_count(labels)
    loss_tok = torch.empty(T, device="cuda")
    y = buf.clone()[:, :V]
    for r0 in range(0, T, 40):
        Km.cross_entropy_rows(y[r0 : r0 + 40], labels[r0 : r0 + 40], loss_tok[r0 : r0 + 40], scratch)
    assert torch.equal(Km.cross_entropy_mean(loss_tok, scratch), loss)
    assert torch.equal(y, dl)


# ---------------------------------------------------------------------------------------------------------------------
# models against the reference fixtures
# ---------------------------------------------------------------------------------------------------------------------
def _model(name, padding_free=True, params=None):
    from dolomite_engine_b200.hf_models import (GPTDolomiteConfig, GPTDolomiteForCausalLM, MoEDolomiteConfig,
                                                MoEDolomiteForCausalLM)

    kw = dict(MODELS[name])
    moe = kw.get("num_experts", 0) > 0
    kw.setdefault("normalization_function", "rmsnorm")
    kw.setdefault("position_embedding_type", "rope")
    cfg = (MoEDolomiteConfig if moe else GPTDolomiteConfig)(resid_pdrop=0, embd_pdrop=0, attn_pdrop=0, eos_token_id=EOS, **kw)
    cls = MoEDolomiteForCausalLM if moe else GPTDolomiteForCausalLM
    model = cls(cfg, seed=None, use_padding_free_transformer=padding_free,
                **({} if padding_free else {"attn_implementation": "sdpa"}))
    if params is not None:
        model.load_state_dict(params)
    return model


def _check_logits(got, want):
    assert got.shape == want.shape
    close = torch.isclose(got, want, rtol=5e-3, atol=5e-3).float().mean().item()
    assert close > 0.99 and rel_l2(got, want) < 1e-2 and (got - want).abs().max().item() < 4e-2, close


def _check_grads(model, fx, batch):
    bad = []
    for pname, unit, _ in model.engine.named_views():
        g = subsample(unit.gviews[pname])
        assert torch.isfinite(g).all(), pname
        e = rel_l2(g, torch.from_numpy(fx[f"{batch}_grad:{pname}"]))
        if e > 3e-2:
            bad.append((pname, round(e, 4)))
    assert not bad, bad


@pytest.mark.parametrize("name", list(MODELS))
def test_packed_batch_matches_reference(name):
    """padding-free pretraining batch: the fused head + loss (chunk buffer of odd width) and the logits-mode head"""
    fx = np.load(os.path.join(GOLDEN, f"model_vocab_{name}.npz"))
    cfg = O.OracleConfig(**MODELS[name])
    model = _model(name, params=_fixture_params(cfg, fx))
    model.assume_unit_loss_grad = True
    ids, pos, cu, labels = _packed_inputs(fx)
    args = (torch.from_numpy(ids).cuda(), torch.from_numpy(pos).cuda(), torch.from_numpy(cu).cuda(), int(np.diff(cu).max()))
    model.engine.zero_grad()
    loss = model.forward_pretraining_loss(*args, torch.from_numpy(labels).cuda())
    loss.backward()
    want = float(fx["packed_loss"])
    assert abs(loss.item() - want) / want < 1e-3
    _check_grads(model, fx, "packed")
    with torch.no_grad():
        out = model(input_ids=args[0], position_ids=args[1], cu_seqlens=args[2], max_seqlen=args[3])
    logits = out.logits
    assert logits.shape == (ids.size, cfg.vocab_size) and logits.is_contiguous()
    assert logits.view(-1, cfg.vocab_size).shape[0] == ids.size
    _check_logits(logits.float().cpu()[::8], torch.from_numpy(fx["packed_logits"]))


@pytest.mark.parametrize("name", list(MODELS))
def test_padded_batch_matches_reference(name):
    """[B, S] batch with right and left padding: logits [B, S, V] and the unfused loss backward (upstream gradient
    applied on the device to the odd-width dlogits buffer)"""
    fx = np.load(os.path.join(GOLDEN, f"model_vocab_{name}.npz"))
    cfg = O.OracleConfig(**MODELS[name])
    model = _model(name, padding_free=False, params=_fixture_params(cfg, fx))
    tokens = torch.from_numpy(fx["padded_tokens"]).cuda()
    mask = torch.from_numpy(fx["padded_mask"]).cuda()
    model.engine.zero_grad()
    out = model(input_ids=tokens, attention_mask=mask, labels=tokens)
    out.loss.backward()
    want = float(fx["padded_loss"])
    assert abs(out.loss.item() - want) / want < 1e-3
    _check_grads(model, fx, "padded")
    with torch.no_grad():
        logits = model(input_ids=tokens, attention_mask=mask).logits
    assert logits.shape == (*tokens.shape, cfg.vocab_size)
    real = logits[mask.bool()].float().cpu()
    _check_logits(real[::8], torch.from_numpy(fx["padded_logits"]))


def test_logits_mode_autograd_matches_fused_loss():
    """an external loss on the [T, V] logits (dlogits staged into 16-byte rows) gives the fused path's gradients"""
    name = "bigcode_2053"
    fx = np.load(os.path.join(GOLDEN, f"model_vocab_{name}.npz"))
    cfg = O.OracleConfig(**MODELS[name])
    params = _fixture_params(cfg, fx)
    ids, pos, cu, labels = _packed_inputs(fx)
    args = (torch.from_numpy(ids).cuda(), torch.from_numpy(pos).cuda(), torch.from_numpy(cu).cuda(), int(np.diff(cu).max()))
    lab = torch.from_numpy(labels).cuda()
    fused = _model(name, params=params)
    fused.assume_unit_loss_grad = True
    fused.engine.zero_grad()
    loss_f = fused.forward_pretraining_loss(*args, lab)
    loss_f.backward()
    ext = _model(name, params=params)
    ext.engine.zero_grad()
    logits = ext(input_ids=args[0], position_ids=args[1], cu_seqlens=args[2], max_seqlen=args[3]).logits
    assert logits.shape[-1] == cfg.vocab_size and logits.requires_grad
    loss_e = F.cross_entropy(logits.float().view(-1, cfg.vocab_size), lab)
    loss_e.backward()
    assert abs(loss_e.item() - loss_f.item()) <= 1e-3 * loss_f.item()
    g_ext = {pname: unit.gviews[pname] for pname, unit, _ in ext.engine.named_views()}
    for pname, unit, _ in fused.engine.named_views():
        assert rel_l2(g_ext[pname], unit.gviews[pname]) < 1e-2, pname


def test_training_steps_are_bit_identical_from_run_to_run():
    from test_gpu_fp8 import _batch, _grads, _step

    from dolomite_engine_b200.engine import DolomiteEngine
    from test_fp8 import _cfg

    runs = []
    for _ in range(2):
        eng = DolomiteEngine(_cfg(vocab_size=2053, tie_word_embeddings=False), "cuda", seed=42)
        losses = [_step(eng, _batch(2053, seed=s), False, lr=0.05) for s in range(2)]
        runs.append((losses, _grads(eng)))
    (l1, g1), (l2, g2) = runs
    assert l1 == l2
    assert all(torch.equal(g1[n], g2[n]) for n in g1)


@pytest.mark.parametrize("name", ["gqa_rope_2051", "bigcode_2053"])
def test_generation_cached_equals_uncached_and_stays_in_vocabulary(name):
    cfg = O.OracleConfig(**MODELS[name])
    params = O.init_params(cfg, seed=42)
    V = cfg.vocab_size
    # make the last vocabulary entry (in the partial 16-byte vector of a logits row) a likely token
    head = "transformer.wte.weight" if cfg.tie_word_embeddings else "lm_head.weight"
    params[head][V - 1] *= 40
    model = _model(name, params=params)
    gen = torch.Generator().manual_seed(0)
    ids = torch.randint(0, V, (3, 12), generator=gen)
    mask = torch.ones_like(ids)
    mask[1, :4] = 0  # left padded
    a = model.generate(input_ids=ids, attention_mask=mask, max_new_tokens=10, eos_token_id=-1, use_cache=True)
    b = model.generate(input_ids=ids, attention_mask=mask, max_new_tokens=10, eos_token_id=-1, use_cache=False)
    if not torch.equal(a, b):
        # the decode kernel and the full forward round differently: they may part only at a near tie of the argmax
        from dolomite_engine_b200.hf_models.generation import last_token_logits

        r, t = [int(i) for i in (a != b).nonzero()[0]]
        m = torch.cat([mask[r : r + 1], torch.ones(1, t - mask.shape[1], dtype=mask.dtype)], 1)
        top2 = last_token_logits(model, b[r : r + 1, :t].cpu(), m)[0].topk(2).values
        assert float(top2[0] - top2[1]) < 0.05, (r, t, top2.tolist())
    assert int(a.max()) < V and int(b.max()) < V
    s = model.generate(input_ids=ids, attention_mask=mask, max_new_tokens=10, eos_token_id=-1, do_sample=True,
                       temperature=2.0, generator=torch.Generator(device="cuda").manual_seed(1))
    assert int(s.max()) < V and int(s.min()) >= 0


def test_granite_checkpoint_with_vocab_49155_roundtrips_through_training(tmp_path):
    """a Granite-style HF checkpoint (vocab_size 49155): import -> one training step -> export -> re-import"""
    import transformers

    from dolomite_engine_b200.hf_models import AutoModelForCausalLM, export_to_huggingface, import_from_huggingface

    torch.manual_seed(0)
    hf_cfg = transformers.GraniteConfig(vocab_size=49155, hidden_size=128, intermediate_size=256, num_hidden_layers=2,
                                        num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=256,
                                        embedding_multiplier=12.0, residual_multiplier=0.22, logits_scaling=8.0,
                                        attention_multiplier=0.0625, tie_word_embeddings=True)
    transformers.GraniteForCausalLM(hf_cfg).save_pretrained(tmp_path / "hf", safe_serialization=True)
    import_from_huggingface(str(tmp_path / "hf"), str(tmp_path / "dolo"))
    model = AutoModelForCausalLM.from_pretrained(str(tmp_path / "dolo"))
    assert model.config.vocab_size == 49155
    model.assume_unit_loss_grad = True
    gen = torch.Generator().manual_seed(2)
    rows = [torch.randint(0, 49155, (n,), generator=gen).tolist() for n in (37, 50)]
    rows[0][-1] = 49154
    model.engine.zero_grad()
    loss = model(input_ids=rows, labels=rows).loss
    loss.backward()
    assert torch.isfinite(loss)
    eng = model.engine
    for u in eng.units:
        u.master.data.add_(u.master.grad, alpha=-0.1)
    eng.refresh_compute_from_master()
    trained = {k: v.clone() for k, v in model.state_dict().items()}
    model.save_pretrained(str(tmp_path / "trained"))
    export_to_huggingface(str(tmp_path / "trained"), str(tmp_path / "hf2"), "granite")
    import_from_huggingface(str(tmp_path / "hf2"), str(tmp_path / "dolo2"))
    again = AutoModelForCausalLM.from_pretrained(str(tmp_path / "dolo2")).state_dict()
    assert sorted(again) == sorted(trained)
    for k, v in trained.items():
        assert torch.equal(again[k].cpu(), v.cpu()), k
