"""NEFTune noise and added special tokens on the GPU.

The reference draws NEFTune's uniform noise from torch's Philox stream, which no independent kernel reproduces; parity is
stated as in tests/test_gpu_dropout.py: (a) the noise is a documented function of (pass seed, element index) that
tests/neft_oracle.py restates bit for bit -- checked element by element here; (b) with that noise installed, the oracle's
loss and every gradient match the GPU's; (c) evaluation and generation are untouched; (d) the noise stream is reproducible
and resumable.  Added tokens: the resized model trains against the oracle, generates, and survives save and load."""

import numpy as np
import pytest
import torch

import neft_oracle as N
import oracle.dolomite_oracle as O
from special_tokens_util import ADDED_TOKENS, build_tokenizer

pytestmark = pytest.mark.gpu


def K():
    from dolomite_engine_b200 import kernels

    return kernels


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


@pytest.mark.parametrize("T", [1, 7, 4096, 16384])
@pytest.mark.parametrize("H", [64, 2056, 4096])
def test_embedding_neft_is_bit_identical_to_the_oracle(T, H):
    V = 1003
    g = torch.Generator().manual_seed(T * 7 + H)
    wte = (torch.randn(V, H, generator=g) * 0.02).to(torch.bfloat16)
    ids = torch.randint(0, V, (T,), generator=g)
    ids[0] = V - 1
    mags = [K().neft_mag(5.0, T * H), K().neft_mag(15.0, 7 * H), 0.37, 3e-4]
    wte_d, ids_d = wte.cuda(), ids.cuda()
    for i, mag in enumerate(mags[: 4 if T * H <= 4096 * 4096 else 2]):
        keys = K().dropout_keys(1000 + i, N.NEFT_SITE)
        got = K().embedding_fwd_neft(ids_d, wte_d, keys, mag).cpu()
        want = N.embed(wte, ids, keys, mag)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (T, H, mag)


def test_repeated_calls_are_identical_and_a_new_pass_is_a_new_stream():
    V, T, H = 517, 3000, 1024
    g = torch.Generator().manual_seed(5)
    wte = (torch.randn(V, H, generator=g) * 0.02).to(torch.bfloat16).cuda()
    ids = torch.randint(0, V, (T,), generator=g).cuda()
    mag = K().neft_mag(5.0, T * H)
    a = K().embedding_fwd_neft(ids, wte, K().dropout_keys(9, N.NEFT_SITE), mag)
    b = K().embedding_fwd_neft(ids, wte, K().dropout_keys(9, N.NEFT_SITE), mag)
    c = K().embedding_fwd_neft(ids, wte, K().dropout_keys(10, N.NEFT_SITE), mag)
    plain = K().embedding_fwd(ids, wte)
    assert torch.equal(a, b)
    assert (a != c).float().mean().item() > 0.5 and (a != plain).float().mean().item() > 0.5
    # the noise is bounded by the bf16 bounds, up to the final bf16 rounding of the sum
    assert (a.float() - plain.float()).abs().max().item() <= 1.01 * mag + 2 ** -8 * plain.float().abs().max().item()


CONFIGS = {
    "rope_memb_mup": dict(vocab_size=1003, n_positions=512, n_embd=320, n_layer=2, n_head=4, n_inner=640,
                          attention_head_type="mha", add_bias=True, m_emb=12.0, m_residual=0.22, m_width=2.0),
    "bigcode_untied": dict(vocab_size=1003, n_positions=512, n_embd=256, n_layer=2, n_head=4, n_inner=1024,
                           attention_head_type="mqa", add_bias=True, position_embedding_type="learned_absolute",
                           normalization_function="layernorm", activation_function="gelu_pytorch_tanh", m_emb=3.0,
                           tie_word_embeddings=False),
}
ALPHA = 15.0


def _build(name, padding_free=True, neft=True, params=None):
    from dolomite_engine_b200.hf_models import GPTDolomiteConfig, GPTDolomiteForCausalLM

    kw = dict(CONFIGS[name])
    ocfg = O.OracleConfig(**kw)
    if params is None:
        params = O.init_params(ocfg, seed=42)
        g = torch.Generator().manual_seed(7)
        for k_ in params:
            if k_.endswith(".bias"):
                params[k_] = torch.randn(params[k_].shape, generator=g) * 0.02
    d = dict(position_embedding_type="rope", normalization_function="rmsnorm", activation_function="swiglu", eos_token_id=7,
             resid_pdrop=0, embd_pdrop=0, attn_pdrop=0)
    d.update(kw)
    model = GPTDolomiteForCausalLM(GPTDolomiteConfig(**d), seed=None, use_padding_free_transformer=padding_free,
                                   attn_implementation="flash_attention_2" if padding_free else "sdpa")
    model.load_state_dict(params)
    model.assume_unit_loss_grad = True
    if neft:
        model.engine.neft_alpha = ALPHA
    return model, ocfg, params


def _lists(V, seed=3):
    rng = np.random.default_rng(seed)
    lens = [61, 130, 17, 90]
    ids = [rng.integers(0, V, n).tolist() for n in lens]
    labels = [[t if j > 3 else -100 for j, t in enumerate(row)] for row in ids]
    return ids, labels


def _oracle_loss(params, ocfg, ids, labels, v):
    b = O.convert_padding_free_lists_to_tensors(ids, labels=labels)
    logits = N.forward_logits(params, ocfg, b["input_ids"], b["position_ids"], b["cu_seqlens"], v)
    shift = O.finetune_shift_labels(b["labels"], b["cu_seqlens"])
    return torch.nn.functional.cross_entropy(logits[:-1].float(), torch.as_tensor(shift, dtype=torch.long), ignore_index=-100)


def _padded(ids, labels, S=136):
    B = len(ids)
    x = torch.zeros(B, S, dtype=torch.long)
    lab = torch.full((B, S), -100, dtype=torch.long)
    mask = torch.zeros(B, S, dtype=torch.long)
    for r, (row, lr) in enumerate(zip(ids, labels)):
        x[r, : len(row)] = torch.tensor(row)
        lab[r, : len(row)] = torch.tensor(lr)
        mask[r, : len(row)] = 1
    return x, mask, lab


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("layout", ["packed", "padded"])
def test_model_with_neftune_matches_the_oracle_with_the_same_noise(name, layout):
    model, ocfg, params = _build(name, padding_free=layout == "packed")
    ids, labels = _lists(ocfg.vocab_size)
    eng = model.engine
    eng.dropout_seed, eng._dropout_passes = 31337, 0
    model.train()
    eng.zero_grad()
    H, T_real = ocfg.n_embd, sum(len(r) for r in ids)
    if layout == "packed":
        loss = model(input_ids=ids, labels=labels).loss
        numel = T_real * H  # the reference's wte sees the flat token list
    else:
        x, mask, lab = _padded(ids, labels)
        loss = model(input_ids=x, attention_mask=mask, labels=lab).loss
        numel = x.numel() * H  # ... or the padded [B, S] batch, padding included
    assert eng._saved["dropout_seed"] == 31337
    loss.backward()
    torch.cuda.synchronize()
    mag = K().neft_mag(ALPHA, numel)
    assert mag == (ALPHA / torch.sqrt(torch.tensor(numel))).item()
    v = torch.from_numpy(N.noise(K().dropout_keys(31337, N.NEFT_SITE), T_real * H, mag)).view(T_real, H)
    p_req = {k: t.clone().requires_grad_(True) for k, t in params.items()}
    ref = _oracle_loss(p_req, ocfg, ids, labels, v)
    ref.backward()
    p_ev = {k: t.clone().requires_grad_(True) for k, t in params.items()}
    ref_clean = _oracle_loss(p_ev, ocfg, ids, labels, None)
    ref_clean.backward()
    assert abs(loss.item() - ref.item()) / ref.item() < 1.5e-3, (loss.item(), ref.item(), ref_clean.item())
    moved = 0
    for n, u, _ in eng.named_views():
        r = p_req[n].grad
        if r is None or r.norm() == 0:
            continue
        assert rel_l2(u.gviews[n], r) < 4e-2, (n, rel_l2(u.gviews[n], r))
        moved += int(rel_l2(p_ev[n].grad, r) > 0.1)
    assert moved >= 3  # the noise moved the gradients far beyond the tolerance: the comparison is not vacuous
    # logits of the noisy training forward (no labels) against the oracle's
    with torch.no_grad():
        eng.dropout_seed, eng._dropout_passes = 31337, 0
        if layout == "packed":
            logits = model(input_ids=ids).logits
            want = N.forward_logits(params, ocfg, *[O.convert_padding_free_lists_to_tensors(ids)[k]
                                                    for k in ("input_ids", "position_ids", "cu_seqlens")], v)
            assert rel_l2(logits, want) < 1e-2


@pytest.mark.parametrize("name", list(CONFIGS))
def test_evaluation_and_generation_are_those_of_the_model_without_neftune(name):
    model, ocfg, params = _build(name, padding_free=False)
    plain, _, _ = _build(name, padding_free=False, neft=False, params=params)
    ids, labels = _lists(ocfg.vocab_size)
    x, mask, lab = _padded(ids, labels)
    for m in (model, plain):
        m.eval()
    with torch.no_grad():
        a = model(input_ids=x, attention_mask=mask).logits
        b = plain(input_ids=x, attention_mask=mask).logits
        la = model(input_ids=x, attention_mask=mask, labels=lab).loss
        lb = plain(input_ids=x, attention_mask=mask, labels=lab).loss
    assert torch.equal(a, b) and torch.equal(la, lb)
    prompt = x[:, :16]
    ga = model.generate(input_ids=prompt, max_new_tokens=12)
    gb = plain.generate(input_ids=prompt, max_new_tokens=12)
    assert torch.equal(ga, gb)
    # a training pass of the same model does add noise
    model.train()
    with torch.no_grad():
        c = model(input_ids=x, attention_mask=mask).logits
    assert rel_l2(c, a) > 1e-3


def _passes(model, ids, labels, n):
    """n training passes (forward + backward) -> [(loss, gradients)]"""
    out = []
    for _ in range(n):
        model.engine.zero_grad()
        loss = model(input_ids=ids, labels=labels).loss
        loss.backward()
        torch.cuda.synchronize()
        out.append((loss.item(), [u.master.grad.clone() for u in model.engine.units]))
    return out


def _same(a, b) -> bool:
    return a[0] == b[0] and all(torch.equal(x, y) for x, y in zip(a[1], b[1]))


def test_passes_are_reproducible_and_a_resumed_run_follows_the_uninterrupted_one():
    """each pass draws new noise (seed + passes so far); two runs give the same bits, and a run restarted from the saved
    (seed, passes) state -- what checkpoints store -- continues the same noise stream"""
    ids, labels = _lists(1003)
    runs = []
    for _ in range(2):
        model, _, params = _build("rope_memb_mup")
        model.engine.dropout_seed, model.engine._dropout_passes = 77, 0
        model.train()
        runs.append(_passes(model, ids, labels, 3))
    assert all(_same(a, b) for a, b in zip(*runs))
    assert runs[0][0][0] != runs[0][1][0] != runs[0][2][0]
    resumed, _, _ = _build("rope_memb_mup", params=params)
    resumed.engine.dropout_seed, resumed.engine._dropout_passes = 77, 2
    resumed.train()
    assert _same(_passes(resumed, ids, labels, 1)[0], runs[0][2])


@pytest.mark.parametrize("vocab_size,tied", [(1000, True), (1000, False), (1013, False)])
def test_model_with_added_tokens_trains_generates_and_roundtrips(tmp_path, vocab_size, tied):
    """V -> len(tokenizer) + 3: grows 1000 -> 1003, or shrinks a padded 1013 -> 1003"""
    from dolomite_engine_b200.hf_models import AutoModelForCausalLM
    from dolomite_engine_b200.model_wrapper import ModelWrapperForFinetuning

    build_tokenizer(str(tmp_path), 1000)
    pc = dict(model_type="gpt_dolomite", vocab_size=vocab_size, n_positions=512, n_embd=256, n_layer=2, n_head=4, n_inner=512,
              attention_head_type="gqa", num_key_value_heads=2, add_bias=False, activation_function="swiglu",
              position_embedding_type="rope", normalization_function="rmsnorm", resid_pdrop=0, embd_pdrop=0, attn_pdrop=0,
              eos_token_id=999, tie_word_embeddings=tied)
    torch.manual_seed(0)
    w = ModelWrapperForFinetuning(pretrained_config=pc, use_padding_free_transformer=True, random_seed=3,
                                  tokenizer_name=str(tmp_path / "tok_1000"), additional_special_tokens=list(ADDED_TOKENS),
                                  neft_alpha=5.0)
    assert w.config.vocab_size == 1003 and len(w.tokenizer) == 1003
    text = ["<|system|> t1 t2 <|user|> t3 t4 t5 <|assistant|> t6", "<|user|> t9 t10 <|assistant|> t11 t12 t13"]
    ids = [w.tokenizer(s, add_special_tokens=False)["input_ids"] for s in text]
    assert {1000, 1001, 1002} <= set(ids[0])
    ids = [r * 6 for r in ids]
    labels = [list(r) for r in ids]
    params = {k: t.float().cpu() for k, t in w.model.state_dict().items()}
    ocfg = O.OracleConfig(**{k: v for k, v in pc.items() if k not in ("model_type", "resid_pdrop", "embd_pdrop", "attn_pdrop",
                                                                    "eos_token_id")} | {"vocab_size": 1003})
    w.eval()  # the oracle comparison without noise; training mode adds it
    w.model.engine.zero_grad()
    loss = w({"input_ids": ids, "labels": labels})
    loss.backward()
    torch.cuda.synchronize()
    p_req = {k: t.clone().requires_grad_(True) for k, t in params.items()}
    ref = _oracle_loss(p_req, ocfg, ids, labels, None)
    ref.backward()
    assert abs(loss.item() - ref.item()) / ref.item() < 1.5e-3
    for n, u, _ in w.model.engine.named_views():
        if p_req[n].grad is not None and p_req[n].grad.norm() > 0:
            assert rel_l2(u.gviews[n], p_req[n].grad) < 4e-2, n
    # the added tokens' rows receive gradient
    gw = w.model.engine.units[0].gviews["transformer.wte.weight"]
    assert gw[1000:1003].abs().sum().item() > 0
    # generation over the new vocabulary: greedy decoding is the step-wise argmax, over all 1003 columns
    path = str(tmp_path / "saved")
    w.save_pretrained(path)
    m2 = AutoModelForCausalLM.from_pretrained(path, use_padding_free_transformer=False, attn_implementation="sdpa")
    m2.eval()
    with torch.no_grad():
        prompt = torch.tensor([ids[0][:10]])
        out = m2.generate(input_ids=prompt, max_new_tokens=6)
        seq = prompt.cuda()
        for _ in range(6):
            lg = m2(input_ids=seq).logits
            assert lg.shape[-1] == 1003
            seq = torch.cat([seq, lg[:, -1].argmax(-1, keepdim=True)], 1)
    assert torch.equal(out, seq)
    sd2 = m2.state_dict()
    for k, t in w.model.state_dict().items():
        assert torch.equal(sd2[k], t), k
