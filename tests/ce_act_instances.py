"""Which template instance of the cross-entropy and MLP activation kernels a call runs: a Python statement of the host's
choice in csrc/elementwise.cu, and named cases that reach every instance.  No torch import, so the CPU test of the built
library (test_ce_act_instances.py) can check the table against the instances the compiler emitted.

Cross entropy (dolomite_b200_cross_entropy_rows): nv1 = ceil(ceil(V / 8) / 256) vectors per thread with the whole row in
one 256-thread CTA picks ce_rows_kernel<NV, SPLIT, TAIL>, TAIL = V % 8 != 0.

Activations (visit_act, launch_act_fwd, launch_act_bwd_form): one functor per id (CELU and ELU share EluT<0>);
act_fwd_kernel<Op, form> for the plain and GLU forms of every functor and the sigmoid-GLU form of Sigmoid;
act_bwd_kernel<Op, glu> without and act_bwd_bias_kernel<Op, glu> with a bias-gradient buffer (dense or segmented).
"""

KCE_THREADS = 256  # kCeThreads of elementwise.cu


def ce_instance(V: int) -> str:
    """the ce_rows_kernel<NV, SPLIT, TAIL> the host runs for a vocabulary of V columns (None: refused)"""
    v8 = (V + 7) // 8
    nv1 = (v8 + KCE_THREADS - 1) // KCE_THREADS
    tail = "true" if V % 8 else "false"
    for limit, nv, split in ((4, 4, 1), (8, 8, 1), (16, 16, 1)):
        if nv1 <= limit:
            return f"ce_rows_kernel<{nv}, {split}, {tail}>"
    if nv1 <= 24 and V % 8 == 0:
        return "ce_rows_kernel<24, 1, false>"
    for limit, nv, split in ((32, 16, 2), (48, 12, 4), (64, 16, 4)):
        if nv1 <= limit:
            return f"ce_rows_kernel<{nv}, {split}, {tail}>"
    return None


def ce_split(V: int) -> int:
    return int(ce_instance(V).split(", ")[1])


# instance -> the vocabularies of its cases (the first is the instance's main case in the GPU tests)
CE_CASES = {
    "ce_rows_kernel<4, 1, false>": [2056, 2048, 8],
    "ce_rows_kernel<4, 1, true>": [2051, 1, 7, 9],
    "ce_rows_kernel<8, 1, false>": [16384, 8200],
    "ce_rows_kernel<8, 1, true>": [16383, 8193],
    "ce_rows_kernel<16, 1, false>": [32768, 16392],
    "ce_rows_kernel<16, 1, true>": [32767, 16385],
    "ce_rows_kernel<24, 1, false>": [49152, 32776],
    "ce_rows_kernel<16, 2, false>": [65536, 49160],
    "ce_rows_kernel<16, 2, true>": [49153, 36871, 50257],
    "ce_rows_kernel<12, 4, false>": [98304, 65544],
    "ce_rows_kernel<12, 4, true>": [98303, 65537],
    "ce_rows_kernel<16, 4, false>": [131072, 98312],
    "ce_rows_kernel<16, 4, true>": [128259, 98305],
}
CE_OTHER = {"ce_count_kernel", "ce_mean_kernel"}

# ---------------------------------------------------------------------------------------------------------------------
# activations: ids of include/dolomite_b200.h (enum DOLO_ACT_*), restated so that this file needs no package import
# ---------------------------------------------------------------------------------------------------------------------
ACT_NAMES = ["celu", "elu", "gelu", "gelu_tanh", "selu", "hardshrink", "hardsigmoid", "hardswish", "hardtanh", "laplace",
             "leaky_relu", "log_sigmoid", "mish", "relu", "relu2", "relu6", "sigmoid", "silu", "softplus", "softshrink",
             "softsign", "tanh", "tanhshrink"]
ACT_IDS = {n: i for i, n in enumerate(ACT_NAMES)}
PLAIN, GLU, SIGMOID_GLU = 0, 1, 2
FORM_NAMES = {PLAIN: "plain", GLU: "glu", SIGMOID_GLU: "sigmoid_glu"}

# visit_act: id -> functor (the names the compiler emits under act::)
FUNCTOR = {
    "celu": "EluT<0>", "elu": "EluT<0>", "gelu": "Gelu", "gelu_tanh": "GeluTanh", "selu": "EluT<1>",
    "hardshrink": "HardShrink", "hardsigmoid": "HardSigmoid", "hardswish": "HardSwish", "hardtanh": "HardTanh",
    "laplace": "Laplace", "leaky_relu": "LeakyRelu", "log_sigmoid": "LogSigmoid", "mish": "Mish", "relu": "Relu",
    "relu2": "Relu2", "relu6": "Relu6", "sigmoid": "Sigmoid", "silu": "Silu", "softplus": "Softplus",
    "softshrink": "SoftShrink", "softsign": "SoftSign", "tanh": "Tanh", "tanhshrink": "TanhShrink",
}

ENTRY_POINTS = ("act_fwd", "act_bwd", "act_bwd_bias", "act_bwd_segmented")


def forms_of(act_id: int) -> list[int]:
    """the forms check_act accepts for an activation id"""
    return [PLAIN, GLU] + ([SIGMOID_GLU] if act_id == ACT_IDS["sigmoid"] else [])


def act_instance(act_id: int, form: int, entry: str) -> str:
    """the kernel instance a call of `entry` runs: act_fwd(id, form), act_bwd without / with a bias-gradient buffer,
    act_bwd_segmented (always with one)"""
    op = FUNCTOR[ACT_NAMES[act_id]]
    if entry == "act_fwd":
        return f"act_fwd_kernel<{op}, {form}>"
    glu = "false" if form == PLAIN else "true"
    kern = "act_bwd_kernel" if entry == "act_bwd" else "act_bwd_bias_kernel"
    return f"{kern}<{op}, {glu}>"


# one named case per (id, form, entry point): every id and form is run through every entry point, so each functor
# instance has a case for each of the ids that share it
ACT_CASES = {
    f"{ACT_NAMES[i]}/{FORM_NAMES[f]}/{e}": (i, f, e) for i in range(len(ACT_NAMES)) for f in forms_of(i)
    for e in ENTRY_POINTS
}


def act_instances() -> set:
    return {act_instance(*c) for c in ACT_CASES.values()}
