"""GPU: every FP8 linear of a real training step, element by element, against its own quantised operands.

The fp8 GEMM and cast kernels have their own suites (test_gpu_gemm_elementwise.py, test_gpu_fp8.py).  This file pins how
the engine wires them together for each FP8 linear: which slot's scale each cast uses, which e4m3 weight copy the dgrad
reads, which alpha / c / beta / bias the epilogue gets, and which amax slot every cast folds into.

Each case builds an engine as test_gpu_fp8.py does, runs two warm-up steps (every slot then has a scale of its own, not 1)
and snapshots the recipe.  Spies on `_linear` and `_linear_bwd_fp8` record, at call time, the input, the bf16 weight,
bias, c, alpha, beta, the output gradient, the dgrad's `dx_add`, and the result.  From the snapshot scales and the slot
layout of fp8.py (input 2 i, weight 2 i + 1, gradient i) the test quantises every operand itself (test_fp8.quantize_ref)
and checks, per call:

- fprop  y  = alpha ((q(x) sxi)(q(w) swi)^T + b) + beta c            fast accumulation over the whole contraction
- dgrad  dx = q5(bf16(alpha dy)) sgi . q(w) swi [+ dx_add]            split accumulation
- wgrad  gw = sum over the accumulation window of q5(bf16(alpha dy))^T sgi . q(x) sxi, per element, where the window
  starts at zero_grad (lazily cleared buffers are overwritten by their first weight-gradient GEMM, the head's chunks and
  later micro-steps accumulate)

each against an fp64 reference with the per-element bars of test_gpu_gemm_elementwise.py.  Those bars bound every addend
of every tensor-core step at once, so they are far above what one operand quantised with another slot's scale moves an
output (up to a whole fp8 step per element, mostly averaging out over the contraction).  Each call is therefore also
replayed through the same GEMM entry point from the operands quantised here: the engine's result must come back bit for
bit, which pins the quantised operands, the scale inverses, the epilogue arguments and the accumulation mode exactly.

Exact checks (`torch.equal`): the linears that ran FP8 are fp8_weight_names(cfg) and every other linear took the bf16
path; the fp8 GEMM launches of the step are exactly the spied ones; after each micro-step the amax history and the
scales equal one DelayedScaling update of the snapshot whose current amaxes are max|x| over every input the linear saw
(all head chunks, both forwards of a recomputed block), max|w| and max|bf16(alpha dy)|.
"""

import pytest
import torch

from test_fp8 import E4M3, E5M2, FP8_MAX, dequantize_ref, quantize_ref, recipe_update_ref
from test_gpu_fp8 import _engine_and_oracle
from test_gpu_gemm_elementwise import U32, _acc_bar, _finish_bar, _fp8_steps

pytestmark = pytest.mark.gpu

# largest err / bar per (case, linear kind, pass), printed at the end of the module
WORST: dict = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    from dolomite_engine_b200 import build

    build.build()
    yield
    for (case, kind, pas), r in sorted(WORST.items()):
        print(f"ERRBAR {case:28s} {kind:12s} {pas:6s}: {r:.3e}")


def _kernels():
    from dolomite_engine_b200 import kernels

    return kernels



# hand-set scales (factor on the delayed-scaling value): (slot kind, linear, factor)
HANDSET_GQA = (
    ("input", "transformer.h.0.attn.c_attn.weight", 16.0),  # inputs saturate at 448
    ("weight", "transformer.h.1.mlp.c_fc.weight", 1 / 16),  # small weights become e4m3 subnormals
    ("grad", "transformer.h.1.attn.c_proj.weight", 8.0),  # large gradients saturate at 57344
    ("grad", "lm_head.weight", 1 / 16),
    ("grad", "transformer.h.0.mlp.c_fc.weight", 1 / 16),
)
HANDSET_MOE = (
    ("input", "transformer.h.1.mlp.gate.weight", 16.0),
    ("weight", "transformer.h.0.mlp.gate.weight", 1 / 16),
    ("grad", "transformer.h.0.mlp.gate.weight", 1 / 16),  # the router's dlogits: the widest range of the step
    ("grad", "transformer.h.1.attn.c_attn.weight", 4.0),
)

# name -> (model of test_gpu_fp8._oracle_cfgs, document lengths, options)
#   head: "fused" (loss and head backward chunk by chunk, >= 3 chunks with a partial last one), "unfused" (logits, then
#   backward(dlogits=...)); ckpt: checkpoint_every; micro: micro-steps without zero_grad between them; overlap: weight
#   gradients on the side stream; aux: router_aux=True; handset: recipe scales set off their delayed-scaling values;
#   later_chunk_max: the batch puts the head's largest |x| outside its first chunk (checked), so that the input amax
#   needs the casts of the later chunks
CASES = {
    "gqa_untied_fused": ("gqa_untied", (300, 212, 144), dict(head="fused", later_chunk_max=True)),
    "gqa_untied_unfused": ("gqa_untied", (300, 212, 144), dict(head="unfused")),
    "gqa_untied_ckpt": ("gqa_untied", (400, 256), dict(head="fused", ckpt=1)),
    "gqa_untied_accum": ("gqa_untied", (300, 212, 144), dict(head="fused", micro=2)),
    "gqa_untied_handset": ("gqa_untied", (300, 212, 144), dict(head="fused", handset=HANDSET_GQA)),
    "bigcode": ("bigcode", (256, 200, 152), dict()),
    "bigcode_mixed": ("bigcode_mixed", (256, 200, 152), dict()),
    "bigcode_mixed_accum_overlap": ("bigcode_mixed", (256, 240, 64), dict(micro=2, overlap=True)),
    "moe32": ("moe32", (240, 176, 96), dict()),
    "moe32_aux": ("moe32", (240, 176, 96), dict(aux=True)),
    "moe32_aux_ckpt": ("moe32", (320, 192), dict(aux=True, ckpt=1)),
    "moe32_aux_handset": ("moe32", (240, 176, 96), dict(aux=True, handset=HANDSET_MOE)),
}


def _kind(name):
    return name.split(".", 3)[-1].removesuffix(".weight") if name.startswith("transformer.h.") else name.removesuffix(".weight")


def _batch(V, docs, seed):
    g = torch.Generator().manual_seed(seed)
    T = sum(docs)
    assert T % 16 == 0  # the FP8 step's token stream (the row count of the transposed wgrad operands)
    ids = torch.randint(0, V, (T,), generator=g)
    labels = torch.randint(0, V, (T,), generator=g)
    pos = torch.cat([torch.arange(n) for n in docs])
    cu = torch.tensor([0] + list(torch.tensor(docs).cumsum(0)), dtype=torch.int32)
    return ids.cuda(), pos.cuda(), cu.cuda(), max(docs), labels.cuda()


def _micro_step(eng, opts, batch):
    from dolomite_engine_b200.fp8 import fp8_autocast

    ids, pos, cu, ms, labels = batch
    with fp8_autocast(eng):
        if opts.get("head") == "unfused":
            logits, _ = eng.forward(ids, pos, cu, ms)
        else:
            eng.forward(ids, pos, cu, ms, labels=labels, fuse_head_loss=True, router_aux=bool(opts.get("aux")),
                        coef=0.01 if opts.get("aux") else 0.0)
    if opts.get("head") == "unfused":
        lg = logits.float()
        dl = (torch.softmax(lg, -1) - torch.nn.functional.one_hot(labels, lg.shape[1]).float()) / lg.shape[0]
        eng.backward(dlogits=dl.bfloat16())
    else:
        eng.backward()


class _Spy:
    """records every FP8 fprop / backward call and every bf16 linear of the engine, and counts the fp8 GEMM launches"""

    def __init__(self, eng):
        self.eng = eng
        self.fwd, self.bwd, self.bf16 = [], [], []
        self.n_gemm_fp8 = 0
        self.n_wgrad_problems = 0

    def __enter__(self):
        eng, K = self.eng, _kernels()
        lin, bwd = eng._linear, eng._linear_bwd_fp8
        self._gemm_fp8, self._wgrad = K.gemm_fp8, K.gemm_fp8_wgrad_multi

        def linear(unit, wname, x, bname=None, *, c=None, alpha=1.0, beta=0.0, out=None, flags=None):
            if not eng._is_fp8(wname):
                self.bf16.append(wname)
                return lin(unit, wname, x, bname, c=c, alpha=alpha, beta=beta, out=out, flags=flags)
            b = unit.views.get(bname) if bname is not None else None
            rec = dict(name=wname, x=x.clone(), w=unit.views[wname].clone(), b=None if b is None else b.clone(),
                       c=None if c is None else c.clone(), alpha=alpha, beta=beta)
            y = lin(unit, wname, x, bname, c=c, alpha=alpha, beta=beta, out=out, flags=flags)
            rec["y"] = y.clone()  # at once: the fused head's cross entropy overwrites it in place
            self.fwd.append(rec)
            return y

        def linear_bwd_fp8(unit, wname, bname, x, dy, alpha=1.0, need_dx=True, dx_out=None, dx_add=None):
            rec = dict(name=wname, x=x.clone(), dy=dy.clone(), alpha=alpha, need_dx=need_dx, w=unit.views[wname].clone(),
                       dx_add=None if dx_add is None else dx_add.clone())
            dx = bwd(unit, wname, bname, x, dy, alpha, need_dx, dx_out, dx_add)
            rec["dx"] = None if dx is None else dx.clone()
            self.bwd.append(rec)
            return dx

        def gemm_fp8(*a, **k):
            self.n_gemm_fp8 += 1
            return self._gemm_fp8(*a, **k)

        def gemm_fp8_wgrad_multi(problems, *a, **k):
            self.n_wgrad_problems += len(problems)
            return self._wgrad(problems, *a, **k)

        eng._linear, eng._linear_bwd_fp8 = linear, linear_bwd_fp8
        K.gemm_fp8, K.gemm_fp8_wgrad_multi = gemm_fp8, gemm_fp8_wgrad_multi
        return self

    def __exit__(self, *exc):
        K = _kernels()
        del self.eng._linear, self.eng._linear_bwd_fp8
        K.gemm_fp8, K.gemm_fp8_wgrad_multi = self._gemm_fp8, self._wgrad


def _recipe(eng):
    return {k: getattr(eng.fp8, k).clone() for k in eng.fp8._KEYS}


def _set_handset(eng, handset):
    """scales off their delayed-scaling values for the `handset` slots; scale_inv stays the fp32 inverse of the scale"""
    r = eng.fp8
    for kind, name, f in handset:
        i = r.index[name]
        scale, inv, j = (r.bwd_scale, r.bwd_scale_inv, i) if kind == "grad" else (
            r.fwd_scale, r.fwd_scale_inv, 2 * i + (kind == "weight"))
        scale[j] = scale[j] * f
        inv[j] = 1.0 / scale[j]


class _Ref:
    """the snapshot scales of one micro-step and the reference quantisation with them (CPU casts, as test_fp8 restates)"""

    def __init__(self, eng, snap):
        self.index = eng.fp8.index
        self.snap = snap

    def slot(self, name, kind):
        i = self.index[name]
        if kind == "grad":
            return self.snap["bwd_scale"][i : i + 1], self.snap["bwd_scale_inv"][i : i + 1]
        j = 2 * i + (kind == "weight")
        return self.snap["fwd_scale"][j : j + 1], self.snap["fwd_scale_inv"][j : j + 1]

    def quantize(self, t, name, kind):
        """-> (fp8 bits on the device, their fp64 values times scale_inv, scale_inv device scalar)"""
        s, si = self.slot(name, kind)
        fmt = E5M2 if kind == "grad" else E4M3
        q = quantize_ref(t.cpu(), s.item(), fmt)
        return q.cuda(), (dequantize_ref(q, fmt) * si.item()).cuda(), si


def _dy_cast_operand(rec):
    """te.Linear's output gradient: that of its own output, bf16(alpha dy)"""
    return rec["dy"] if rec["alpha"] == 1.0 else (rec["dy"].float() * rec["alpha"]).bfloat16()


def _check(case, name, pas, got, ref, bar):
    assert bool(torch.isfinite(got).all()), (name, pas)
    err = (got.double() - ref).abs()
    key = (case, _kind(name), pas)
    WORST[key] = max(WORST.get(key, 0.0), (err / (bar + 1e-30)).max().item())
    assert bool((err <= bar + 1e-30).all()), f"{pas} of {name} off its fp64 bar: err/bar {WORST[key]:.3g}"


def _check_fprop(case, ref, rec):
    K = _kernels()
    name, alpha, beta = rec["name"], rec["alpha"], rec["beta"]
    qx, vx, xsi = ref.quantize(rec["x"], name, "input")
    qw, vw, wsi = ref.quantize(rec["w"], name, "weight")
    b = 0.0 if rec["b"] is None else rec["b"].double()
    c = 0.0 if rec["c"] is None else rec["c"].double()
    want = alpha * (vx @ vw.t() + b) + beta * c
    mag = vx.abs() @ vw.abs().t()
    mag_out = abs(alpha) * (mag + (b.abs() if rec["b"] is not None else 0.0)) + abs(beta) * (
        c.abs() if rec["c"] is not None else 0.0)
    bar32 = abs(alpha) * _acc_bar("fp8", _fp8_steps(dict(split=False), qx.shape[1]), mag) + 4 * U32 * mag_out
    _check(case, name, "fprop", rec["y"], want, _finish_bar(bar32, want, rec["y"].dtype))
    again = K.gemm_fp8(qx, E4M3, xsi, qw, E4M3, wsi, bias=rec["b"], c=rec["c"], alpha=alpha, beta=beta,
                       out_dtype=rec["y"].dtype)
    assert torch.equal(again, rec["y"]), f"fprop of {name} is not the GEMM of its operands quantised with its slots' scales"


def _check_dgrad(case, ref, rec):
    K = _kernels()
    name = rec["name"]
    qdy, vdy, gsi = ref.quantize(_dy_cast_operand(rec), name, "grad")
    qw, vw, wsi = ref.quantize(rec["w"], name, "weight")
    add = rec["dx_add"]
    want = vdy @ vw + (0.0 if add is None else add.double())
    mag = vdy.abs() @ vw.abs()
    mag_out = mag + (0.0 if add is None else add.double().abs())
    bar32 = _acc_bar("fp8", _fp8_steps(dict(split=True), qdy.shape[1]), mag) + 4 * U32 * mag_out
    _check(case, name, "dgrad", rec["dx"], want, _finish_bar(bar32, want, rec["dx"].dtype))
    wt = qw.t().contiguous()
    if add is None:
        again = K.gemm_fp8(qdy, E5M2, gsi, wt, E4M3, wsi, split_accumulate=True)
    else:
        again = add.clone()
        K.gemm_fp8(qdy, E5M2, gsi, wt, E4M3, wsi, out=again, c=again, beta=1.0, split_accumulate=True)
    assert torch.equal(again, rec["dx"]), f"dgrad of {name} is not the GEMM of its operands quantised with its slots' scales"


def _check_wgrad(case, ref, name, recs, base, got):
    """recs: the backward calls of `name` in this micro-step, in order; base: the gradient after the previous micro-step of
    the window (None: the window starts here, the buffer holds whatever the last step left)"""
    K = _kernels()
    want = torch.zeros(got.shape, dtype=torch.float64, device="cuda") if base is None else base.double()
    bar = torch.zeros_like(want)
    mags = torch.zeros_like(want) if base is None else base.double().abs()
    again = torch.full(got.shape, float("nan"), dtype=torch.float32, device="cuda") if base is None else base.clone()
    for n, rec in enumerate(recs):
        qdy, vdy, gsi = ref.quantize(_dy_cast_operand(rec), name, "grad")
        qx, vx, xsi = ref.quantize(rec["x"], name, "input")
        want += vdy.t() @ vx
        mag = vdy.abs().t() @ vx.abs()
        mags += mag
        bar += _acc_bar("fp8", _fp8_steps(dict(split=True), qdy.shape[0]), mag) + 4 * U32 * mag
        K.gemm_fp8_wgrad_multi([(qdy.t().contiguous(), gsi, qx.t().contiguous(), xsi, again, 1.0,
                                 base is not None or n > 0)])
    bar += len(recs) * U32 * mags  # one fp32 add per call onto the running sum
    _check(case, name, "wgrad", got, want, bar)
    assert torch.equal(again, got), f"wgrad of {name} is not the sum of its calls' GEMMs over the window"


def _expected_linears(cfg, eng):
    """every weight that goes through `_linear` in a training step (MoE experts use the grouped GEMMs)"""
    names = []
    for i in range(cfg.n_layer):
        p = f"transformer.h.{i}."
        names += [p + "attn.c_attn.weight", p + "attn.c_proj.weight"]
        names += [p + "mlp.gate.weight"] if eng.is_moe else [p + "mlp.c_fc.weight", p + "mlp.c_proj.weight"]
    names.append("transformer.wte.weight" if cfg.tie_word_embeddings else "lm_head.weight")
    return names


def _q_stats(t, fmt, scale):
    """(saturated, subnormal, flushed to zero) elements of t quantised with `scale`"""
    q = quantize_ref(t.cpu(), scale, fmt)
    mag = q & 0x7F
    mant_bits = 3 if fmt == E4M3 else 2
    sat = int((mag == (0x7E if fmt == E4M3 else 0x7B)).sum())
    sub = int(((mag >> mant_bits) == 0).logical_and(mag != 0).sum())
    flushed = int(((mag == 0) & (t.cpu() != 0)).sum())
    return sat, sub, flushed


@pytest.mark.parametrize("case", list(CASES))
def test_fp8_linears_of_a_step(case):
    from dolomite_engine_b200.fp8 import fp8_weight_names

    model, docs, opts = CASES[case]
    eng, ocfg, params = _engine_and_oracle(model)
    cfg = eng.cfg
    batch = _batch(ocfg.vocab_size, docs, seed=len(case))
    T = sum(docs)
    n_chunks = 1
    if opts.get("head") == "fused":
        eng.head_chunk_bytes = 2 * cfg.vocab_size * 224
        rows = eng._head_chunk_rows(T, cfg.vocab_size, eng.head_chunk_bytes, 16)
        n_chunks = -(-T // rows)
        assert n_chunks >= 3 and T % rows != 0, (T, rows)
    if opts.get("later_chunk_max"):
        # token 0 embeds as one large coordinate and occurs only in the head's last chunk: ln_f's output there has
        # |x| near sqrt(n_embd), above every row of the other chunks, so the head's input amax needs the last chunk's cast
        params["transformer.wte.weight"][0] = 0.0
        params["transformer.wte.weight"][0, 0] = 1.0
        eng.load_state_dict(params)
        ids = batch[0]
        ids[ids == 0] = 1
        ids[T - 40 :: 13] = 0
    eng.checkpoint_every = opts.get("ckpt")
    eng.overlap_wgrads = bool(opts.get("overlap"))
    for _ in range(2):  # warm-up: every slot gets a delayed-scaling scale of its own
        eng.zero_grad()
        _micro_step(eng, opts, batch)
    r = eng.fp8
    assert bool((r.fwd_scale != 1).all()) and bool((r.bwd_scale != 1).all())
    if opts.get("handset"):
        _set_handset(eng, opts["handset"])
    names = fp8_weight_names(cfg)
    assert r.names == names
    weights = {n: (u, s) for n, u, s in eng.named_views() if n in r}

    eng.zero_grad()
    base = None  # the accumulation window starts here
    for m in range(opts.get("micro", 1)):
        snap = _recipe(eng)
        ref = _Ref(eng, snap)
        with _Spy(eng) as spy:
            _micro_step(eng, opts, batch)
        torch.cuda.synchronize()

        # which linears ran FP8, how often, and no fp8 GEMM outside the spied calls
        expected = _expected_linears(cfg, eng)
        assert sorted({rec["name"] for rec in spy.fwd}) == sorted(names)
        assert sorted({rec["name"] for rec in spy.bwd}) == sorted(names)
        assert sorted(set(spy.bf16)) == sorted(set(expected) - set(names))
        for n in names:
            head = not n.startswith("transformer.h.")
            i = None if head else int(n.split(".")[2])
            n_fwd = n_chunks if head else (2 if eng._is_checkpointed(i) else 1)
            assert sum(rec["name"] == n for rec in spy.fwd) == n_fwd, n
            assert sum(rec["name"] == n for rec in spy.bwd) == (n_chunks if head else 1), n
        assert spy.n_gemm_fp8 == len(spy.fwd) + sum(rec["need_dx"] for rec in spy.bwd)
        assert spy.n_wgrad_problems == len(spy.bwd)
        if eng.is_moe:  # the router's dgrad adds onto the expert path's dx
            assert all((rec["dx_add"] is not None) == rec["name"].endswith("mlp.gate.weight") for rec in spy.bwd)

        # per element: fprop, dgrad, wgrad
        for rec in spy.fwd:
            _check_fprop(case, ref, rec)
        for rec in spy.bwd:
            _check_dgrad(case, ref, rec)
        grads = {}
        for n in names:
            u, _ = weights[n]
            grads[n] = u.gviews[n].clone()
            _check_wgrad(case, ref, n, [rec for rec in spy.bwd if rec["name"] == n], None if base is None else base[n],
                         grads[n])
        base = grads

        # amaxes: what every cast saw, then one DelayedScaling update of the snapshot
        n = len(names)
        amax_f = torch.zeros(2 * n, dtype=torch.float32)
        amax_b = torch.zeros(n, dtype=torch.float32)
        for rec in spy.fwd:
            i = r.index[rec["name"]]
            amax_f[2 * i] = torch.maximum(amax_f[2 * i], rec["x"].float().abs().max().cpu())
            amax_f[2 * i + 1] = torch.maximum(amax_f[2 * i + 1], rec["w"].float().abs().max().cpu())
        for rec in spy.bwd:
            i = r.index[rec["name"]]
            amax_b[i] = torch.maximum(amax_b[i], _dy_cast_operand(rec).float().abs().max().cpu())
        if opts.get("later_chunk_max"):
            chunks = [rec["x"].float().abs().max().item() for rec in spy.fwd if rec["name"] == "lm_head.weight"]
            assert max(chunks[1:]) > chunks[0], chunks
        for hist, scale, amax, fmt in (("fwd_history", "fwd_scale", amax_f, E4M3), ("bwd_history", "bwd_scale", amax_b, E5M2)):
            h0 = snap[hist].cpu()
            assert bool((h0[0] == 0).all())  # the previous update cleared the current row
            h0[0] = amax
            want_h, want_s, want_si = recipe_update_ref(h0, snap[scale].cpu(), FP8_MAX[fmt])
            assert torch.equal(getattr(r, hist).cpu(), want_h), f"{hist}: the amaxes the casts recorded"
            assert torch.equal(getattr(r, scale).cpu(), want_s), scale
            assert torch.equal(getattr(r, scale + "_inv").cpu(), want_si), scale + "_inv"

        if opts.get("handset") and m == 0:
            # the hand-set slots reach the formats' edges, and the engine matched the reference there (above)
            for kind, name, f in opts["handset"]:
                s, _ = ref.slot(name, kind)
                if kind == "input":
                    stats = [_q_stats(rec["x"], E4M3, s.item()) for rec in spy.fwd if rec["name"] == name]
                elif kind == "weight":
                    stats = [_q_stats(rec["w"], E4M3, s.item()) for rec in spy.fwd if rec["name"] == name]
                else:
                    stats = [_q_stats(_dy_cast_operand(rec), E5M2, s.item()) for rec in spy.bwd if rec["name"] == name]
                sat, sub, flushed = (sum(x[k] for x in stats) for k in range(3))
                print(f"{case} {kind} slot of {name} x{f:g}: saturated {sat}, subnormal {sub}, flushed to zero {flushed}")
                if kind == "input" or f > 1:
                    assert sat > 0, (kind, name)
                if kind == "weight":
                    assert sub > 0, (kind, name)
