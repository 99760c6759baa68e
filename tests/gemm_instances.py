"""The cases of tests/test_gpu_gemm_elementwise.py and the template instances of the GEMM kernels they reach.

No torch import, so the CPU test of the built library (test_gemm_sass.py) can check that the instances the compiler
emitted are exactly the keys of INSTANCES: a new instance without a case fails there.  Each case also names the instance
it is meant to reach, and instance_of() restates the host's choice of kernel (gemm.cu: gemm_impl picks the tile width,
dispatch / dispatch_fp8 the template arguments), so the CPU test also checks that every case lands where it claims.

Every case runs twice on the GPU: with random inputs against per-element fp64 bars, and with exact-arithmetic inputs
against the fp64 result rounded once to D's type, bit for bit.

Instance names follow the demangled template arguments as integers: gemm_bf16_kernel<A_MN, B_MN, TN> and
gemm_fp8_kernel<FA, FB, SPLIT> (format 0 = e4m3, 1 = e5m2).
"""

E4M3, E5M2 = 0, 1
FP8_PAIRS = [(E4M3, E4M3), (E4M3, E5M2), (E5M2, E4M3), (E5M2, E5M2)]
LAYOUTS = [(False, False), (False, True), (True, False), (True, True)]  # (A MN-major, B MN-major)

# entry points that always run the 128-wide tile, whatever gemm_tile_n forces (their tile tables are per 128 x 128 tile)
TILE128_ONLY = ("gemm_splitk", "grouped_m", "grouped_m_gather", "grouped_k")
BF16_ENTRIES = ("gemm", "wgrad_multi") + TILE128_ONLY
FP8_ENTRIES = ("gemm_fp8", "fp8_wgrad_multi")


def bf16_instance(a_mn: bool, b_mn: bool, tn: int) -> str:
    return f"gemm_bf16_kernel<{int(a_mn)}, {int(b_mn)}, {tn}>"


def fp8_instance(fa: int, fb: int, split: bool) -> str:
    return f"gemm_fp8_kernel<{fa}, {fb}, {int(split)}>"


def instance_of(case: dict) -> str:
    """the host's dispatch restated: fp8 launches take the formats and the split flag; bf16 launches take the layout and
    tile 128 for the grouped, gather-on-load and split-K modes, else the forced gemm_tile_n (the cases always force one)"""
    if case["entry"] in FP8_ENTRIES:
        return fp8_instance(case["fa"], case["fb"], case["split"])
    a_mn, b_mn = case["layout"]
    if case["entry"] in ("grouped_m", "grouped_m_gather"):
        a_mn = False  # the grouped rows of A are K-major
    if case["entry"] == "grouped_k":
        a_mn = b_mn = True  # both are the [rows, features] activations
    tn = 128 if case["entry"] in TILE128_ONLY else case["tile_n"]
    return bf16_instance(a_mn, b_mn, tn)


# dense shapes (M, N, K): M % 128 in {1, 63, 64, 65, 127}; N in {1, 8, 136, 264} and N % 256 in {8, 136}; K in {1, 8, 40},
# K % 64 in {8, 56} and one K >= 4096 whose operands exceed 24 MB (the L2 eviction hints); one shape with several times
# more tiles than SMs at both widths
DENSE_SHAPES = [
    (193, 264, 40), (127, 136, 72), (129, 1, 120), (63, 8, 8), (320, 392, 1), (255, 520, 184),
    (4033, 2440, 72), (65, 264, 56),
]
HINT_SHAPE = (2049, 1288, 4104)


def _dense_cases() -> dict:
    cases = {}
    i = 0
    for layout in LAYOUTS:
        for tn in (128, 256):
            for j in range(2):
                M, N, K = DENSE_SHAPES[i % len(DENSE_SHAPES)]
                i += 1
                name = f"gemm-{'TF'[layout[0] ^ 1]}{'TF'[layout[1] ^ 1]}-{tn}-{M}x{N}x{K}"
                cases[name] = dict(entry="gemm", layout=layout, tile_n=tn, shape=(M, N, K), seed=i,
                                   instance=bf16_instance(*layout, tn))
    for tn in (128, 256):  # the long contraction with L2 eviction hints: the forward layout and the weight gradient's
        for layout in ((False, False), (True, True)):
            M, N, K = HINT_SHAPE
            name = f"gemm-hints-{'TF'[layout[0] ^ 1]}{'TF'[layout[1] ^ 1]}-{tn}-{M}x{N}x{K}"
            cases[name] = dict(entry="gemm", layout=layout, tile_n=tn, shape=HINT_SHAPE, seed=50 + tn + layout[0],
                               instance=bf16_instance(*layout, tn))
    return cases


def _splitk_cases() -> dict:
    # K = 2056 (33 k-blocks: 4 splits of 128-wide tiles) and 1096 (18 k-blocks: 2 splits); C == D, beta = 1, fp32 D
    grid = [((True, True), (200, 136, 2056)), ((False, False), (65, 264, 1096)), ((False, True), (191, 8, 2056))]
    return {f"splitk-{'TF'[l[0] ^ 1]}{'TF'[l[1] ^ 1]}-{s[0]}x{s[1]}x{s[2]}":
            dict(entry="gemm_splitk", layout=l, tile_n=256, shape=s, seed=70 + i, instance=bf16_instance(*l, 128))
            for i, (l, s) in enumerate(grid)}


def _wgrad_multi_cases() -> dict:
    # (tokens K, [(M, N)] of up to four weight gradients), every other problem accumulating
    problems = [(264, 200), (136, 520), (72, 8), (193, 136)]
    return {f"wgrad_multi-{tn}": dict(entry="wgrad_multi", layout=(True, True), tile_n=tn, K={128: 328, 256: 376}[tn],
                                      problems=problems, seed=80 + tn, instance=bf16_instance(True, True, tn))
            for tn in (128, 256)}


# MoE shapes (T tokens, E experts, top-k, K, N); expert 1 receives no tokens, and with the K-grouped cases' seeds some
# expert's rows reach the last 64-row k-block of its segment (segments are padded to 256 rows)
MOE_SHAPES = [(200, 3, 2, 72, 136), (1000, 5, 2, 120, 264)]


def _grouped_cases() -> dict:
    cases = {}
    for i, (T, E, k, Kd, N) in enumerate(MOE_SHAPES):
        for bias in (False, True):
            for b_mn in (False, True):
                cases[f"grouped_m-F{'TF'[b_mn ^ 1]}-{'bias' if bias else 'plain'}-{T}x{E}x{Kd}x{N}"] = dict(
                    entry="grouped_m", layout=(False, b_mn), tile_n=256, moe=(T, E, k, Kd, N), bias=bias, seed=90 + 4 * i + 2 * bias + b_mn,
                    instance=bf16_instance(False, b_mn, 128))
            cases[f"grouped_m_gather-FF-{'bias' if bias else 'plain'}-{T}x{E}x{Kd}x{N}"] = dict(
                entry="grouped_m_gather", layout=(False, False), tile_n=256, moe=(T, E, k, Kd, N), bias=bias, seed=110 + 2 * i + bias,
                instance=bf16_instance(False, False, 128))
        # K-grouped expert weight gradient dW[e] [N, Kd] (+)= dY_e^T X_e: overwrite and accumulate
        for beta in (0.0, 1.0):
            cases[f"grouped_k-TT-beta{beta:g}-{T}x{E}x{N}x{Kd}"] = dict(
                entry="grouped_k", layout=(True, True), tile_n=256, moe=(T, E, k, Kd, N), beta=beta, seed=124 + 2 * i + int(beta),
                instance=bf16_instance(True, True, 128))
    return cases


# fp8 shapes: K % 16 == 0 and N % 16 == 0; K = 16 (one k32 step, half of it zero-filled), 144 (one full k-block and a
# partial one) and 240 (a last k-block whose fourth k32 step holds data); one has more tiles than SMs
FP8_SHAPES = [(200, 272, 144), (65, 16, 16), (1031, 2064, 144), (127, 144, 240)]


def _fp8_cases() -> dict:
    cases = {}
    i = 0
    for fa, fb in FP8_PAIRS:
        for split in (False, True):
            M, N, K = FP8_SHAPES[i % len(FP8_SHAPES)]
            cases[f"gemm_fp8-{fa}{fb}-{'split' if split else 'fast'}-{M}x{N}x{K}"] = dict(
                entry="gemm_fp8", fa=fa, fb=fb, split=split, shape=(M, N, K), seed=130 + i, instance=fp8_instance(fa, fb, split))
            i += 1
    for fa, fb, split in ((E5M2, E4M3, True), (E5M2, E4M3, False), (E4M3, E4M3, True)):
        cases[f"fp8_wgrad_multi-{fa}{fb}-{'split' if split else 'fast'}"] = dict(
            entry="fp8_wgrad_multi", fa=fa, fb=fb, split=split, K=368, problems=[(200, 272), (128, 16), (65, 144)],
            seed=150 + i, instance=fp8_instance(fa, fb, split))
        i += 1
    return cases


CASES = {**_dense_cases(), **_splitk_cases(), **_wgrad_multi_cases(), **_grouped_cases(), **_fp8_cases()}


def _instances() -> dict:
    inst: dict = {}
    for name, c in CASES.items():
        inst.setdefault(c["instance"], []).append(name)
    return inst


# instance -> the cases that run it
INSTANCES = _instances()
