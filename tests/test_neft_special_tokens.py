"""CPU: NEFTune (`research_args.neft_alpha`) and added special tokens (`tokenizer_args.additional_special_tokens`).

- get_model forwards both options (model_wrapper/__init__.py:35-38 of the reference);
- the noise bound is torch's own host expression, and the noise restatement (tests/neft_oracle.py) has the stated support,
  moments and distribution, with independent streams per pass and per site;
- the vocabulary resize equals the reference's `resize_token_embeddings` (tests/golden/special_tokens.npz, written by
  tools/pin_special_tokens.py), through the wrapper too, and a sharded model resizes to the layout of one built at the new size.
"""

import math
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import neft_oracle as N
import oracle.dolomite_oracle as O
from special_tokens_util import ADDED_TOKENS, build_tokenizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "special_tokens.npz")
PC = dict(model_type="gpt_dolomite", n_embd=32, n_head=2, n_layer=1, n_inner=64, attention_head_type="mha", add_bias=False,
          activation_function="swiglu", position_embedding_type="rope", normalization_function="rmsnorm", resid_pdrop=0,
          embd_pdrop=0, attn_pdrop=0, eos_token_id=299, bos_token_id=299, pad_token_id=299)


def _args(tmp_path, tokenizer_dir, vocab_size=300, tied=True, neft_alpha=5.0, tokens=ADDED_TOKENS):
    from dolomite_engine_b200.arguments import get_args_from_dict

    pc = dict(PC, vocab_size=vocab_size, tie_word_embeddings=tied)
    return get_args_from_dict({
        "model_args": {"model_class": "AutoModelForCausalLM", "pretrained_config": pc, "use_padding_free_transformer": True},
        "tuning_args": {"tuning_method": "full_finetuning"},
        "tokenizer_args": {"tokenizer_name": tokenizer_dir, "additional_special_tokens": list(tokens) if tokens else None},
        "research_args": {"neft_alpha": neft_alpha},
        "datasets": [{"class_name": "JSONLinesDataset", "data_name": "s", "class_args": {"data_path": "x"}}],
        "training_parameters": {"num_training_steps": 1, "micro_batch_size": 2, "eval_during_training": False},
        "save_args": {"save_path": str(tmp_path), "save_interval": 1}, "random_args": {"seed": 5},
        "mixed_precision_args": {"dtype": "bf16"}})


def test_get_model_forwards_neft_alpha_and_the_added_tokens(tmp_path):
    from dolomite_engine_b200.model_wrapper import get_model

    build_tokenizer(str(tmp_path), 300)
    w = get_model(_args(tmp_path, str(tmp_path / "tok_300")), device=torch.device("cpu"))
    assert w.model.engine.neft_alpha == 5.0 and w.model.engine.uses_pass_seed and not w.model.engine.has_dropout
    assert len(w.tokenizer) == 303 and w.config.vocab_size == 303 and w.model.config.vocab_size == 303
    assert w.model.engine.units[0].views["transformer.wte.weight"].shape == (303, 32)
    ids = w.tokenizer("t3 <|user|> t5 <|assistant|>", add_special_tokens=False)["input_ids"]
    assert ids == [3, 301, 5, 302]
    # the expanded tokenizer and the new size travel with save_pretrained
    w.save_pretrained(str(tmp_path / "saved"))
    from transformers import AutoTokenizer

    from dolomite_engine_b200.hf_models.config import CommonConfig

    assert len(AutoTokenizer.from_pretrained(str(tmp_path / "saved"))) == 303
    assert CommonConfig.from_pretrained(str(tmp_path / "saved")).vocab_size == 303
    # neither option: nothing changes
    w0 = get_model(_args(tmp_path, str(tmp_path / "tok_300"), neft_alpha=None, tokens=None), device=torch.device("cpu"))
    assert w0.model.engine.neft_alpha is None and not w0.model.engine.uses_pass_seed and w0.config.vocab_size == 300


def test_added_tokens_need_a_local_tokenizer(tmp_path):
    from dolomite_engine_b200.model_wrapper import get_model

    with pytest.raises(ValueError, match="additional_special_tokens"):
        get_model(_args(tmp_path, str(tmp_path / "missing")), device=torch.device("cpu"))


def test_tokens_already_in_the_tokenizer_leave_the_model_alone(tmp_path):
    from dolomite_engine_b200.model_wrapper import get_model

    build_tokenizer(str(tmp_path), 300)
    w = get_model(_args(tmp_path, str(tmp_path / "tok_300"), vocab_size=304, tokens=("<|endoftext|>",)),
                  device=torch.device("cpu"))
    assert len(w.tokenizer) == 300 and w.config.vocab_size == 304


def test_noise_bound_is_torchs_host_expression():
    """mag = alpha / torch.sqrt(torch.tensor(numel)), fp32, bit for bit -- including numel above 2^24, where numel rounds"""
    from dolomite_engine_b200.kernels import neft_mag

    rng = np.random.default_rng(0)
    numels = [1, 7 * 64, 4096 * 4096, 2 ** 24 + 1, 2 ** 24 + 3, 16384 * 4096, 3 * 2 ** 30 + 5]
    numels += rng.integers(1, 2 ** 24, 300).tolist() + rng.integers(2 ** 24, 2 ** 36, 300).tolist()
    for alpha in (5.0, 10.0, 15.0, 0.1, 1.3):
        for n in numels:
            want = (alpha / torch.sqrt(torch.tensor(int(n)))).item()
            assert neft_mag(alpha, int(n)) == want, (alpha, n)
            assert np.float32(want) == want


@pytest.mark.parametrize("mag", [5 / math.sqrt(16384 * 4096), 10 / math.sqrt(7 * 2056), 0.37, 1e-5])
def test_noise_support_moments_and_distribution(mag):
    """2^24 samples: v in [from, to) (a value equal to `to` becomes `from`), mean 0, variance mag^2 / 3, and the KS distance to
    U(-mag, mag) within what bf16 quantisation and sampling allow"""
    n = 1 << 24
    keys = O.DropoutOracle(1234).keys(N.NEFT_SITE)
    v = N.noise(keys, n, mag).astype(np.float64)
    frm, to, _ = N.bounds(mag)
    assert v.min() >= frm and v.max() < to
    m = float(np.float32(mag))
    var = m * m / 3
    # sampling bars: 6 standard errors; bf16 rounding of v shifts no moment by more than its half-ulp bias bound
    half_ulp = 2.0 ** (math.floor(math.log2(m)) - 8)
    assert abs(v.mean()) < 6 * math.sqrt(var / n) + half_ulp
    assert abs(v.var() / var - 1) < 6 * math.sqrt(0.8 / n) + 4 * half_ulp / m
    # KS on the bf16 support: the CDF of U(-mag, mag) at each distinct value against the empirical one
    vals, counts = np.unique(v, return_counts=True)
    emp = np.cumsum(counts) / n
    cdf = np.clip((vals - (-m)) / (2 * m), 0, 1)
    ks = np.max(np.abs(emp - cdf))
    # the largest bf16 gap in [-mag, mag) is 2^-7 relative: the CDF step across it bounds the quantisation part
    assert ks < 2.0 ** -8 + 1.63 / math.sqrt(n), ks


def test_passes_and_sites_give_independent_streams():
    n = 1 << 20
    u = {}
    for seed, site in [(7, N.NEFT_SITE), (8, N.NEFT_SITE), (7, 0), (7, 5)]:
        u[(seed, site)] = N.uniform_u(O.DropoutOracle(seed).keys(site), n).astype(np.float64)
    base = u[(7, N.NEFT_SITE)]
    for k, other in u.items():
        if k == (7, N.NEFT_SITE):
            continue
        assert not np.array_equal(base, other)
        assert abs(np.corrcoef(base, other)[0, 1]) < 6 / math.sqrt(n), k
    # the noise site is none of the dropout sites of a 64-layer model
    dropout_keys = {O.DropoutOracle(7).keys(s) for s in [0] + [4 * i + j for i in range(64) for j in (1, 2, 3)]}
    assert O.DropoutOracle(7).keys(N.NEFT_SITE) not in dropout_keys


@pytest.mark.parametrize("case", ["grow_tied", "grow_untied", "shrink_tied", "shrink_untied"])
def test_resize_matches_the_reference(case):
    from dolomite_engine_b200.hf_models.utils import resize_vocab_state

    z = np.load(GOLDEN)
    V, V_tok, V_new, tied, H, seed = z[f"{case}_meta"].tolist()
    sd = {"transformer.wte.weight": torch.from_numpy(z[f"{case}_wte"]), "transformer.ln_f.weight": torch.ones(H)}
    if not tied:
        sd["lm_head.weight"] = torch.from_numpy(z[f"{case}_lm_head"])
    torch.manual_seed(seed)
    out = resize_vocab_state(sd, V_new)
    after = torch.rand(8)
    assert torch.equal(after, torch.from_numpy(z[f"{case}_after"]))  # the generator consumed what the reference consumed
    n = min(V, V_new)
    for name, key in [("transformer.wte.weight", "wte")] + ([] if tied else [("lm_head.weight", "lm_head")]):
        got, want = out[name], torch.from_numpy(z[f"{case}_new_{key}"])
        assert got.shape == (V_new, H) and got.dtype == torch.float32
        assert torch.equal(got[:n], sd[name][:n])  # old rows unchanged
        assert torch.equal(got, want), case  # new rows bit-identical
    assert ("lm_head.weight" in out) == (not tied) and out["transformer.ln_f.weight"] is sd["transformer.ln_f.weight"]


@pytest.mark.parametrize("tied,vocab_size", [(True, 300), (False, 300), (False, 308)])
def test_wrapper_resizes_the_model_it_builds(tmp_path, tied, vocab_size):
    """the wrapper's resize is resize_vocab_state of the model built at the old size, drawn from the global generator"""
    from dolomite_engine_b200.hf_models.utils import resize_vocab_state
    from dolomite_engine_b200.model_wrapper import get_model

    build_tokenizer(str(tmp_path), 300)
    tok = str(tmp_path / "tok_300")
    old = get_model(_args(tmp_path, tok, vocab_size, tied, tokens=None), device=torch.device("cpu")).model.state_dict()
    torch.manual_seed(77)
    w = get_model(_args(tmp_path, tok, vocab_size, tied), device=torch.device("cpu"))
    after = torch.rand(4)
    torch.manual_seed(77)
    want = resize_vocab_state(old, 303)
    assert torch.equal(after, torch.rand(4))
    got = w.model.state_dict()
    assert set(got) == set(want)
    for k in got:
        assert torch.equal(got[k], want[k]), k


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _sharded_worker(rank, world, port, q):
    import torch.distributed as dist

    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dolomite_engine_b200.hf_models import GPTDolomiteConfig, GPTDolomiteForCausalLM

        torch.manual_seed(21)
        cfg = GPTDolomiteConfig(**{k: v for k, v in PC.items() if k != "model_type"}, vocab_size=300, tie_word_embeddings=False)
        m = GPTDolomiteForCausalLM(cfg, device=torch.device("cpu"), world_size=world, rank=rank, seed=3, resize_vocab_to=303)
        # numpy arrays travel by value; torch tensors would be shared through file descriptors that die with this process
        q.put((rank, [u.master.detach().numpy().copy() for u in m.engine.units], m.engine.units[0].padded, cfg.vocab_size))
    finally:
        dist.destroy_process_group()


def test_sharded_resize_has_the_layout_of_a_model_built_at_the_new_size():
    """gloo, world size 2: each rank resizes the full root before taking its shard; the gathered root equals the one-rank
    resize, and its flat layout is that of a model built with vocab_size = 303"""
    from dolomite_engine_b200.engine import FlatUnit, _root_specs
    from dolomite_engine_b200.hf_models import GPTDolomiteConfig, GPTDolomiteForCausalLM

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in range(2)]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    results.sort(key=lambda r: r[0])
    torch.manual_seed(21)
    cfg = GPTDolomiteConfig(**{k: v for k, v in PC.items() if k != "model_type"}, vocab_size=300, tie_word_embeddings=False)
    one = GPTDolomiteForCausalLM(cfg, device=torch.device("cpu"), seed=3, resize_vocab_to=303)
    built = FlatUnit("root", _root_specs(GPTDolomiteConfig(**{k: v for k, v in PC.items() if k != "model_type"},
                                                           vocab_size=303, tie_word_embeddings=False)), 2, 0)
    assert all(r[2] == built.padded and r[3] == 303 for r in results)
    for i, u in enumerate(one.engine.units):
        full = torch.from_numpy(np.concatenate([results[0][1][i], results[1][1][i]]))
        assert torch.equal(full[: u.numel], u.master.detach()[: u.numel]), u.name


def test_checkpoints_carry_the_noise_stream_of_a_neftune_model(tmp_path):
    """a NEFTune model without dropout saves and restores (pass seed, passes so far), so a resumed run continues the noise"""
    from test_checkpointing import _args as ckpt_args
    from test_checkpointing import _build

    from dolomite_engine_b200 import checkpointing as C

    path = str(tmp_path / "ckpt")
    engine, model, opt, sched = _build(1, 0, seed=1)
    assert not engine.has_dropout and not engine.uses_pass_seed
    engine.neft_alpha, engine.dropout_seed, engine._dropout_passes = 5.0, 4242, 17
    C.save_checkpoint(ckpt_args(path), model, opt, sched, None, None, 3, metadata={})
    engine2, model2, opt2, sched2 = _build(1, 0, seed=2)
    engine2.neft_alpha = 5.0
    C.load_checkpoint_for_training(ckpt_args(path, load=True), model2, opt2, sched2, None)
    assert (engine2.dropout_seed, engine2._dropout_passes) == (4242, 17)
    engine2.training = True
    engine2._begin_dropout_pass()
    assert engine2._dropout_now == 4242 + 17
